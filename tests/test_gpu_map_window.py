"""Large maps: the map window (include/mcl3dl_b200.h, "Map window").

A map whose whole likelihood lattice is refused, or exceeds MCL3DL_MAP_MAX_CELLS, is staged windowed: the search
structures cover only a box around the particles and are rebuilt when the particles leave it.  Every search returns the
exact nearest neighbour within its radius, so each record must equal, byte for byte, the record of an engine that staged
the whole map (or, for a map too large for that, only the part around the particles).

- a forced window on the warehouse scene (a small cap), particles moved across the map: every map-reading call and a
  resident cycle, for the KD caster with the likelihood model and for the likelihood model alone;
- copies of the warehouse 1.5 km apart, whose whole lattice is far above 2^31 cells: tracking at each copy, on one and
  on two device contexts;
- map updates inside and outside the window, and an append that takes a whole-staged map over the cap;
- the refusals (particles spread beyond the cap, measure_device, field mode, global localisation) and non-finite inputs.
"""
import numpy as np
import pytest

from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu

F = np.float32
CAP = 4_000_000  # cells: a few metres of the warehouse around the particles (the whole map has ~25 M)
N_P, N_LIK, N_BEAM = 384, 96, 12
REACH = 3.0


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


def make_engine(eng_mod, monkeypatch, cap=None, devices=(0,)):
    if cap is None:
        monkeypatch.delenv("MCL3DL_MAP_MAX_CELLS", raising=False)
    else:
        monkeypatch.setenv("MCL3DL_MAP_MAX_CELLS", str(cap))
    e = eng_mod.Engine(devices)
    monkeypatch.delenv("MCL3DL_MAP_MAX_CELLS", raising=False)
    return e


def params(eng_mod, caster):
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    if caster is None:
        return lik, None
    beam = eng_mod.beam_params_from_reference(num_points_default=N_BEAM, dda_grid_size=0.2,
                                              use_raycast_using_dda=0)
    return lik, beam


@pytest.fixture(scope="module")
def warehouse():
    mp, info = synth.warehouse_map(400_000, seed=7)
    return mp, info


def stop(mp, pos, yaw, seed):
    """Particles, scans and origins of a tracking step at (pos, yaw)."""
    q = synth.quat_from_rpy(np.array([[0.0, 0.0, yaw]]))[0]
    lik = synth.make_scan(mp, pos, q, N_LIK, 0.5, REACH, seed=seed)
    beam = synth.make_scan(mp, pos, q, N_BEAM, 0.5, REACH, n_origins=2, seed=seed + 1)
    parts = synth.tracking_particles(N_P, pos, (0.0, 0.0, yaw), seed=seed + 2)
    return {"particles": parts, "lik": lik, "beam": beam, "origins": synth.sensor_origins(2, seed=seed + 3), "pos": pos,
            "yaw": yaw}


def records(e, s, with_beam=True):
    """Every map-reading call of the host API at one stop, as bytes."""
    P = s["particles"]
    beam = s["beam"] if with_beam else None
    out = [e.measure(P, s["lik"], beam, s["origins"]).tobytes()]
    prior = np.random.default_rng(5).uniform(0.1, 1.0, len(P)).astype(F)
    post, summ, rec = e.measure_update(P, s["lik"], beam, s["origins"], prior, want_records=True)
    out += [post.tobytes(), repr(sorted(summ.items())), rec.tobytes()]
    if with_beam:
        out.append(e.beam_status(P[:32], s["beam"], s["origins"]).tobytes())
        out.append(e.beam_cast(P[0], s["beam"], s["origins"]).tobytes())
    pts_q = np.concatenate([s["lik"], s["beam"]])
    out += [a.tobytes() for a in e.match_output(P[:1], pts_q, 0.1, 0.5, 20.0, 0.2)]
    return out


def resident_cycle(e, s, with_beam=True, seed=3):
    """init -> predict -> scan_prepare -> measure_update_prepared -> estimate -> resample, as bytes."""
    from mcl_3dl_b200 import engine as em
    mean6 = np.array([s["pos"][0], s["pos"][1], s["pos"][2], 0.0, 0.0, s["yaw"]], F)
    e.particles_init(N_P, mean6, seed, sigma=np.array([0.2, 0.2, 0.05, 0.02, 0.02, 0.1], F))
    a = synth.make_poses(np.zeros((1, 3)), synth.quat_from_rpy(np.zeros((1, 3))))
    b = synth.make_poses(np.array([[0.2, 0.05, 0.0]]), synth.quat_from_rpy(np.array([[0.0, 0.0, 0.03]])))
    e.particles_predict(a, b, 0.1, 10.0, 10.0)
    sp = em.ScanParams(downsample=(0.0, 0.0, 0.0), lik_num_points=64, beam_num_points=8 if with_beam else 0)
    sp.lik_clip_far = REACH
    sp.beam_clip_far = REACH
    e.scan_prepare(np.concatenate([s["lik"], s["beam"]]), sp)
    summ = e.particles_measure_update_prepared(s["origins"])
    est = e.particles_estimate()
    e.particles_resample((0.05, 0.05, 0.05), (0.01, 0.01, 0.02), 0.0, seed + 1)
    return [repr(sorted(summ.items())), repr({k: (v.tobytes() if hasattr(v, "tobytes") else v) for k, v in est.items()})] + \
        [x.tobytes() for x in e.particles_get()]


def path(info, n):
    L = info["L"]
    xs = np.linspace(0.15 * L, 0.85 * L, n)
    return [np.array([x, 0.5 * L + 0.3 * np.sin(i), 0.6]) for i, x in enumerate(xs)]


@pytest.mark.parametrize("caster", ["kd", None])
def test_forced_window_equals_whole_staging(eng_mod, monkeypatch, warehouse, caster):
    mp, info = warehouse
    lik, beam = params(eng_mod, caster)
    whole = make_engine(eng_mod, monkeypatch)
    win = make_engine(eng_mod, monkeypatch, CAP)
    for e in (whole, win):
        e.set_map(mp, lik, beam)
    assert not whole.map_window_info()["windowed"]
    wi = win.map_window_info()
    assert wi["windowed"] and not wi["staged"] and wi["rebuilds"] == 0
    with_beam = caster is not None
    for i, pos in enumerate(path(info, 5)):
        s = stop(mp, pos, 0.4 * i, seed=100 + 10 * i)
        assert records(win, s, with_beam) == records(whole, s, with_beam), i
        assert resident_cycle(win, s, with_beam) == resident_cycle(whole, s, with_beam), i
        # both engines select the same likelihood kernel: the NN field is staged in both
        assert whole.nn_field_info()["bytes"] > 0 and win.nn_field_info()["bytes"] > 0
    wi = win.map_window_info()
    assert wi["staged"] and wi["rebuilds"] >= 2, wi
    dims = wi["dims"]
    assert dims[0] * dims[1] * dims[2] <= CAP
    assert tuple(win.map_info().nn_dims) == dims
    assert win.map_get()[0].tobytes() == whole.map_get()[0].tobytes()
    whole.close()
    win.close()


def copies(mp, offsets):
    parts = []
    for ox, oy in offsets:
        c = mp.copy()
        c["x"] = (c["x"].astype(np.float64) + ox).astype(F)
        c["y"] = (c["y"].astype(np.float64) + oy).astype(F)
        parts.append(c)
    return parts


OFFSETS = [(0.0, 0.0), (1500.0, 0.0), (0.0, 1500.0), (1500.0, 1500.0)]


@pytest.fixture(scope="module")
def campus():
    mp, info = synth.warehouse_map(60_000, seed=9)
    parts = copies(mp, OFFSETS)
    return np.concatenate(parts), parts, info


@pytest.mark.parametrize("devices", [(0,), (0, 0)])
def test_map_the_whole_lattice_refuses(eng_mod, monkeypatch, campus, devices):
    big, parts, info = campus
    lik, beam = params(eng_mod, "kd")
    e = make_engine(eng_mod, monkeypatch, devices=devices)
    e.set_map(big, lik, beam)  # the whole lattice: far above 2^31 cells
    assert e.map_window_info()["windowed"]
    L = info["L"]
    # one engine for the local copies, so that its resident set draws from the same Philox calls as e's
    local = make_engine(eng_mod, monkeypatch)
    for k, (ox, oy) in enumerate(OFFSETS):
        local.set_map(parts[k], lik, beam)  # that copy alone: the other copies are 1.5 km away
        pos = np.array([ox + 0.5 * L, oy + 0.5 * L, 0.6])
        s = stop(parts[k], pos, 0.3 * k, seed=300 + k)
        P = s["particles"]
        # each context computes its block of the particles as a one-device engine computes that block
        G = len(devices)
        blocks = [(len(P) * d // G, len(P) * (d + 1) // G) for d in range(G)]
        want = b"".join(local.measure(P[lo:hi], s["lik"], s["beam"], s["origins"]).tobytes() for lo, hi in blocks)
        assert e.measure(P, s["lik"], s["beam"], s["origins"]).tobytes() == want, k
        want = b"".join(local.beam_status(P[lo:hi], s["beam"], s["origins"]).tobytes() for lo, hi in blocks)
        assert e.beam_status(P, s["beam"], s["origins"]).tobytes() == want, k
        if len(devices) == 1:
            assert records(e, s) == records(local, s), k
            assert resident_cycle(e, s) == resident_cycle(local, s), k
    local.close()
    assert e.map_window_info()["rebuilds"] >= len(OFFSETS)
    e.close()


def patch_at(center, n=400, seed=0):
    rng = np.random.default_rng(seed)
    xyz = np.asarray(center) + rng.uniform(-0.6, 0.6, (n, 3))
    return synth.make_points(xyz.astype(F))


def test_map_updates(eng_mod, monkeypatch, warehouse):
    mp, info = warehouse
    lik, beam = params(eng_mod, "kd")
    L = info["L"]
    win = make_engine(eng_mod, monkeypatch, CAP)
    win.set_map(mp, lik, beam)
    here = stop(mp, np.array([0.3 * L, 0.5 * L, 0.6]), 0.2, seed=500)
    win.measure(here["particles"], here["lik"], here["beam"], here["origins"])
    n0 = win.map_window_info()["rebuilds"]
    # a patch inside the window: rebuilt once, records of a whole staging of the merged map
    inside = patch_at((0.3 * L + 1.5, 0.5 * L, 0.8), seed=1)
    win.map_append(inside)
    merged = np.concatenate([mp, inside])
    whole = make_engine(eng_mod, monkeypatch)
    whole.set_map(merged, lik, beam)
    assert records(win, here) == records(whole, here)
    assert win.map_window_info()["rebuilds"] == n0 + 1
    # a patch outside the window: nothing rebuilt; a later visit sees it
    far = (0.85 * L, 0.5 * L, 0.8)
    outside = patch_at(far, seed=2)
    win.map_append(outside)
    merged = np.concatenate([merged, outside])
    whole.set_map(merged, lik, beam)
    assert records(win, here) == records(whole, here)
    assert win.map_window_info()["rebuilds"] == n0 + 1
    there = stop(mp, np.array([0.85 * L - 1.0, 0.5 * L, 0.6]), 0.0, seed=510)
    assert records(win, there) == records(whole, there)
    assert win.map_get()[0].tobytes() == merged.tobytes()
    whole.close()
    win.close()
    # an append that takes a whole-staged map over the cap: windowed, not refused
    small = mp[(mp["x"] < 0.4 * L) & (mp["y"] < 0.4 * L)]
    e = make_engine(eng_mod, monkeypatch, CAP)
    e.set_map(small, lik, beam)
    assert not e.map_window_info()["windowed"]
    e.map_append(patch_at((L - 1.0, L - 1.0, 5.0), seed=3))
    assert e.map_window_info()["windowed"]
    whole = make_engine(eng_mod, monkeypatch)
    whole.set_map(np.concatenate([small, patch_at((L - 1.0, L - 1.0, 5.0), seed=3)]), lik, beam)
    s = stop(small, np.array([0.2 * L, 0.2 * L, 0.6]), 0.0, seed=520)
    assert records(e, s) == records(whole, s)
    e.close()
    whole.close()


def test_refusals_and_non_finite_inputs(eng_mod, monkeypatch, warehouse):
    import torch
    mp, info = warehouse
    lik, beam = params(eng_mod, "kd")
    L = info["L"]
    win = make_engine(eng_mod, monkeypatch, CAP)
    whole = make_engine(eng_mod, monkeypatch)
    for e in (win, whole):
        e.set_map(mp, lik, beam)
    s = stop(mp, np.array([0.5 * L, 0.5 * L, 0.6]), 0.7, seed=700)
    # NaN particles and NaN scan points: left out of the box, records of the whole staging
    P = s["particles"].copy()
    P["px"][3] = np.nan
    P["qw"][5] = np.nan
    P["py"][7] = np.inf
    lk = s["lik"].copy()
    lk["x"][2] = np.nan
    lk["z"][4] = np.inf
    bm = s["beam"].copy()
    bm["y"][1] = np.nan
    t = dict(s, particles=P, lik=lk, beam=bm)
    assert records(win, t) == records(whole, t)
    # particles spread beyond the cap: refused, window and resident set unchanged
    mean6 = np.array([0.5 * L, 0.5 * L, 0.6, 0.0, 0.0, 0.0], F)
    win.particles_init(N_P, mean6, 1, sigma=np.array([0.2, 0.2, 0.05, 0.02, 0.02, 0.1], F))
    win.particles_measure_update(s["lik"], s["beam"], s["origins"])
    before_w, before_p = win.map_window_info(), [a.tobytes() for a in win.particles_get()]
    spread = synth.spread_particles(N_P, info, seed=4)
    with pytest.raises(eng_mod.EngineError) as ei:
        win.measure(spread, s["lik"], s["beam"], s["origins"])
    assert ei.value.code == -5
    st = np.zeros(N_P, dtype=synth.STATE)
    st["pos"] = np.stack([spread["px"], spread["py"], spread["pz"]], 1)
    st["rot"] = np.stack([spread[k] for k in ("qx", "qy", "qz", "qw")], 1)
    win.particles_set(st, np.full(N_P, 1.0 / N_P, F))
    mid = [a.tobytes() for a in win.particles_get()]
    with pytest.raises(eng_mod.EngineError) as ei:
        win.particles_measure_update(s["lik"], s["beam"], s["origins"])
    assert ei.value.code == -5
    assert [a.tobytes() for a in win.particles_get()] == mid
    assert win.map_window_info() == before_w
    assert mid != before_p
    # measure_device, field mode and global localisation on a windowed map
    dev = torch.device("cuda:0")
    d_poses = torch.from_numpy(s["particles"].view(np.uint8).copy()).to(dev)
    d_lik = torch.from_numpy(s["lik"].view(np.uint8).copy()).to(dev)
    d_out = torch.zeros(N_P * 24, dtype=torch.uint8, device=dev)
    with pytest.raises(eng_mod.EngineError) as ei:
        win.measure_device(d_poses.data_ptr(), N_P, d_lik.data_ptr(), N_LIK, None, 0, None, 0, d_out.data_ptr())
    assert ei.value.code == -5
    with pytest.raises(eng_mod.EngineError) as ei:
        win.field_mode(True)
    assert ei.value.code == -5
    with pytest.raises(eng_mod.EngineError) as ei:
        win.global_localization(None, grid=0.5)
    assert ei.value.code == -5
    # the engine still serves tracking afterwards
    assert records(win, s) == records(whole, s)
    win.close()
    whole.close()


def test_appends_in_a_row_before_the_next_call(eng_mod, monkeypatch, warehouse):
    """An append with a point inside the window, then one with none, and no call that reads the map in between: the
    window must still be rebuilt with the first patch's points."""
    mp, info = warehouse
    lik, beam = params(eng_mod, "kd")
    L = info["L"]
    win = make_engine(eng_mod, monkeypatch, CAP)
    win.set_map(mp, lik, beam)
    here = stop(mp, np.array([0.4 * L, 0.5 * L, 0.6]), 0.5, seed=800)
    win.measure(here["particles"], here["lik"], here["beam"], here["origins"])
    n0 = win.map_window_info()["rebuilds"]
    inside = patch_at((0.4 * L + 1.0, 0.5 * L + 0.5, 0.8), seed=11)
    outside = patch_at((0.9 * L, 0.1 * L, 0.8), seed=12)
    win.map_append(inside)
    win.map_append(outside)
    whole = make_engine(eng_mod, monkeypatch)
    whole.set_map(np.concatenate([mp, inside, outside]), lik, beam)
    assert records(win, here) == records(whole, here)
    assert win.map_window_info()["rebuilds"] == n0 + 1
    whole.close()
    win.close()


def test_restaging_a_different_windowed_map(eng_mod, monkeypatch, warehouse):
    """set_map of a second windowed map with no point inside the first map's window: nothing of the first map's
    window may serve it.  The second map is smaller and lies 200 m away, so indices of the first would run past it."""
    mp, info = warehouse
    lik, beam = params(eng_mod, "kd")
    L = info["L"]
    win = make_engine(eng_mod, monkeypatch, 1_500_000)  # below the second map's whole lattice as well
    win.set_map(mp, lik, beam)
    here = stop(mp, np.array([0.5 * L, 0.5 * L, 0.6]), 0.1, seed=900)
    win.measure(here["particles"], here["lik"], here["beam"], here["origins"])
    assert win.map_window_info()["rebuilds"] == 1
    second = mp[: len(mp) * 3 // 4].copy()
    second["x"] = (second["x"].astype(np.float64) + 200.0).astype(F)
    # other parameters as well: the new window must be laid out for them
    lik2 = eng_mod.LikParams(match_dist_min=0.22, dist_weight=(1, 1, 4.5))
    win.set_map(second, lik2, beam)
    wi = win.map_window_info()
    assert wi["windowed"] and not wi["staged"] and wi["rebuilds"] == 0
    whole = make_engine(eng_mod, monkeypatch)
    whole.set_map(second, lik2, beam)
    # the same particles, now far from every map point, and then a stop on the second map
    assert records(win, here) == records(whole, here)
    there = stop(second, np.array([200.0 + 0.5 * L, 0.5 * L, 0.6]), 0.2, seed=910)
    assert records(win, there) == records(whole, there)
    assert resident_cycle(win, there) == resident_cycle(whole, there)
    assert win.map_window_info()["rebuilds"] >= 1
    whole.close()
    win.close()


def test_two_contexts_on_a_forced_window(eng_mod, monkeypatch, warehouse):
    """Engine((0, 0)): both contexts' window checks are enqueued before either is read; measure_update's weight total
    spans both.  Every host call equals a two-context engine that staged the whole map."""
    mp, info = warehouse
    lik, beam = params(eng_mod, "kd")
    whole = make_engine(eng_mod, monkeypatch, devices=(0, 0))
    win = make_engine(eng_mod, monkeypatch, CAP, devices=(0, 0))
    for e in (whole, win):
        e.set_map(mp, lik, beam)
    for i, pos in enumerate(path(info, 3)):
        s = stop(mp, pos, 0.3 * i, seed=1000 + 10 * i)
        P = s["particles"]
        assert win.measure(P, s["lik"], s["beam"], s["origins"]).tobytes() == \
            whole.measure(P, s["lik"], s["beam"], s["origins"]).tobytes(), i
        prior = np.random.default_rng(i).uniform(0.1, 1.0, len(P)).astype(F)
        a = win.measure_update(P, s["lik"], s["beam"], s["origins"], prior, want_records=True)
        b = whole.measure_update(P, s["lik"], s["beam"], s["origins"], prior, want_records=True)
        assert a[0].tobytes() == b[0].tobytes() and a[1] == b[1] and a[2].tobytes() == b[2].tobytes(), i
        assert win.beam_status(P, s["beam"], s["origins"]).tobytes() == \
            whole.beam_status(P, s["beam"], s["origins"]).tobytes(), i
    assert win.map_window_info()["rebuilds"] >= 2
    whole.close()
    win.close()
