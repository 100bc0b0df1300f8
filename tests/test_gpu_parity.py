"""GPU parity: the CUDA engine, called through the C ABI, against the CPU oracle and the committed
golden outputs of the reference's own sources.  Everything here needs an H100 (`-m gpu`).

Bars (BASELINE.json north_star): beam HIT/SHORT/LONG tallies and per-ray BeamStatus bit-exact;
match counts bit-exact; likelihood scores within 1e-4 relative (the per-particle float sum is
reduced in a different order than the reference's sequential loop).
"""
import os

import numpy as np
import pytest

from conftest import golden
from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu

LIK_RTOL = 1e-4


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(params=["tuned", "group"])
def eng(eng_mod, request, monkeypatch):
    """Both likelihood paths (csrc/kernels.cuh): `tuned` stages the NN field (lik_kernel_nf_pm / lik_kernel_nf);
    `group` stages none (MCL3DL_NNF=0, as for a field above MCL3DL_NNF_MAX_MB): lik_kernel_wi, a group of TPP lanes per
    particle searching the CSR windows.  The beam kernels are the same in both."""
    if request.param == "group":
        monkeypatch.setenv("MCL3DL_NNF", "0")
    else:
        monkeypatch.delenv("MCL3DL_NNF", raising=False)
    e = eng_mod.Engine((0,))
    yield e
    e.close()


@pytest.fixture
def eng_mod_engine_tuned(eng_mod, monkeypatch):
    monkeypatch.delenv("MCL3DL_NNF", raising=False)
    e = eng_mod.Engine((0,))
    yield e
    e.close()


@pytest.fixture(scope="module")
def cc():
    from oracle import cpu_checker
    cpu_checker.build("port")
    return cpu_checker


def check_records(got, want, n_beam):
    for f in ("match_cnt", "n_short", "n_hit", "n_long"):
        assert np.array_equal(got[f], want[f]), f
    assert np.array_equal(got["score_beam"], want["score_beam"])
    assert np.allclose(got["score_like"], want["score_like"], rtol=LIK_RTOL, atol=1e-6)
    assert ((got["n_short"] + got["n_hit"] + got["n_long"]) <= n_beam).all()


# ------------------------------------------------------------------ committed reference outputs
@pytest.mark.parametrize("name", ["room_iso", "room_aniso", "room_spread", "room_kd_iso", "room_kd_aniso"])
def test_golden_rooms(eng_mod, eng, name):
    g = golden(name + ".npz")
    n_beam, flm, short_only = [int(v) for v in g["beam_cfg"]]
    lik = eng_mod.LikParams(dist_weight=tuple(float(v) for v in g["dist_weight"]))
    beam = eng_mod.beam_params_from_reference(num_points_default=n_beam, filter_label_max=flm,
                                              add_penalty_short_only_mode=bool(short_only),
                                              dda_grid_size=float(g["dda_grid"]),
                                              use_raycast_using_dda=bool(int(g["use_dda"])))
    eng.set_map(g["map"], lik, beam)
    res = eng.measure(g["particles"], g["lik"], g["beam"], g["origins"])
    check_records(res, g["result"], n_beam)
    assert np.array_equal(eng.beam_status(g["particles"], g["beam"], g["origins"]), g["status"])


def test_golden_beam_likelihood_world(eng_mod, eng):
    """World + sweep of test/src/test_beam_likelihood.cpp:81-210, both raycasters."""
    g = golden("beam_likelihood_world.npz")
    pc_map, pc, xs = synth.make_points(g["map"]), synth.make_points(g["scan"]), g["xs"]
    k = 0
    for method, mode in ((1, 0), (1, 1), (0, 0), (0, 1)):
        for hr in g["hit_ranges"]:
            beam = eng_mod.beam_params_from_reference(map_grid=(0.1, 0.1, 0.1), num_points_default=len(pc) + 2,
                                                      beam_likelihood_min=0.2, hit_range=float(hr),
                                                      add_penalty_short_only_mode=(mode == 1), dda_grid_size=0.1,
                                                      use_raycast_using_dda=(method == 1))
            # the KD-tree caster searches the likelihood grid: it needs the (default, isotropic) lik params too
            eng.set_map(pc_map, eng_mod.LikParams() if method == 0 else None, beam, stamp=100 + k)
            # every x is its own update in the reference test: origin = pose position, identity rotation
            for i, x in enumerate(xs):
                r = eng.measure(synth.make_poses([[x, 0, 0]], [[0, 0, 0, 1]]), None, pc,
                                np.array([[x, 0, 0]], np.float32))
                assert r["score_beam"][0] == g["likelihood"][k, i], (method, mode, hr, i)
            ident = synth.make_poses([[0, 0, 0]], [[0, 0, 0, 1]])
            st = np.array([eng.beam_status(ident, synth.make_points([[x, 0, 0]]), np.zeros((1, 3), np.float32))[0, 0]
                           for x in xs])
            assert np.array_equal(st, g["status"][k]), (method, mode, hr)
            k += 1


# ------------------------------------------------------------------ seeded scenes vs the oracle
def run_both(eng_mod, eng, cc, s, w, n_beam_default, dda_grid=0.2, flm=0xFFFFFFFF, short_only=True, hit_range=0.3,
             use_dda=True):
    port = cc.CpuChecker("port")
    lik_c = cc.lik_params(dist_weight=w)
    braw = cc.beam_raw(num_points_default=n_beam_default, dda_grid_size=dda_grid, filter_label_max=flm,
                       add_penalty_short_only_mode=short_only, hit_range=hit_range, use_raycast_using_dda=use_dda)
    cpu = port.create(s["map"], lik_c, braw, 20.0, 0.4)
    lik = eng_mod.LikParams(dist_weight=w)
    beam = eng_mod.beam_params_from_reference(num_points_default=n_beam_default, dda_grid_size=dda_grid,
                                              filter_label_max=flm, add_penalty_short_only_mode=short_only,
                                              hit_range=hit_range, use_raycast_using_dda=use_dda)
    assert beam.as_tuple() == cpu.beam_params().as_tuple()
    eng.set_map(s["map"], lik, beam, stamp=int(np.random.default_rng().integers(1, 2 ** 40)))
    return cpu


@pytest.mark.parametrize("seed,w,spread,P,n_lik,n_beam", [
    (11, (1, 1, 1), False, 64, 96, 3),      # BASELINE config 1: the reference's default operating point
    (12, (1, 1, 5), False, 64, 96, 3),      # ... with the node's anisotropic metric (parameters.cpp:108-111)
    (13, (1, 1, 5), True, 333, 257, 65),    # ragged sizes, spread particles (many outside / LONG rays)
    (14, (1, 1, 5), False, 1000, 33, 200),  # more rays than likelihood points
    (15, (2, 1, 3), False, 97, 1, 1),       # single-point scans
])
def test_scene_vs_oracle(eng_mod, eng, cc, seed, w, spread, P, n_lik, n_beam):
    s = synth.scene(50_000, P, n_lik, n_beam, spread=spread, seed=seed)
    cpu = run_both(eng_mod, eng, cc, s, w, n_beam, dda_grid=0.2 if seed % 2 else 0.1,
                   flm=1 if seed == 13 else 0xFFFFFFFF, short_only=seed != 14)
    want = cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    got = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    check_records(got, want, n_beam)
    assert np.array_equal(eng.beam_status(s["particles"], s["beam"], s["origins"]),
                          cpu.beam_status(s["particles"], s["beam"], s["origins"]))
    if not spread:
        assert want["match_cnt"].sum() > 0 and want["n_hit"].sum() + want["n_short"].sum() > 0


@pytest.mark.parametrize("seed,w,spread,P,n_beam,flm", [
    (61, (1, 1, 5), False, 64, 3, 0xFFFFFFFF),   # the node's defaults: KD-tree caster, 3 rays
    (62, (1, 1, 1), False, 200, 48, 1),          # label filter + TOTAL_REFLECTION paths
    (63, (1, 1, 5), True, 129, 33, 0xFFFFFFFF),  # spread particles
])
def test_kdtree_raycaster_vs_oracle(eng_mod, eng, cc, seed, w, spread, P, n_beam, flm):
    """RaycastUsingKDTree (raycasts/raycast_using_kdtree.h), the reference's default raycaster (parameters.h:109)."""
    s = synth.scene(50_000, P, 64, n_beam, spread=spread, seed=seed)
    cpu = run_both(eng_mod, eng, cc, s, w, n_beam, flm=flm, short_only=seed != 62, use_dda=False)
    want = cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    got = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    check_records(got, want, n_beam)
    st_want = cpu.beam_status(s["particles"], s["beam"], s["origins"])
    assert np.array_equal(eng.beam_status(s["particles"], s["beam"], s["origins"]), st_want)
    if seed == 62:
        assert (st_want == 3).sum() > 0 and (st_want == 1).sum() > 0 and (st_want == 0).sum() > 0


def test_edge_cases(eng_mod, eng, cc):
    s = synth.scene(20_000, 40, 64, 16, seed=21)
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 5), 16)
    P = s["particles"]
    # empty scans -> LidarMeasurementResult(1, 0) for that model (likelihood.cpp:111-114, beam.cpp:130-133)
    r = eng.measure(P, None, None, s["origins"])
    assert (r["score_like"] == 1).all() and (r["match_cnt"] == 0).all() and (r["score_beam"] == 1).all()
    r = eng.measure(P, s["lik"], None, None)
    w = cpu.measure(P, s["lik"], None, s["origins"])
    assert (r["score_beam"] == 1).all() and np.array_equal(r["match_cnt"], w["match_cnt"])
    r = eng.measure(P, None, s["beam"], s["origins"])
    w = cpu.measure(P, None, s["beam"], s["origins"])
    assert (r["score_like"] == 1).all() and np.array_equal(r["score_beam"], w["score_beam"])
    # zero particles
    assert len(eng.measure(P[:0], s["lik"], s["beam"], s["origins"])) == 0
    # one particle, particle far outside the map (every ray LONG: begin outside the AABB, raycast_using_dda.h:70-75)
    far = synth.make_poses([[1e4, 1e4, 1e4]], [[0, 0, 0, 1]])
    r = eng.measure(far, s["lik"], s["beam"], s["origins"])
    assert r["n_long"][0] == 16 and r["match_cnt"][0] == 0 and r["score_like"][0] == 0
    # beam label out of the origins range is rejected, not read out of bounds
    bad = s["beam"].copy()
    bad["label"][3] = 7
    with pytest.raises(eng_mod.EngineError) as ei:
        eng.measure(P, s["lik"], bad, s["origins"])
    assert ei.value.code == -1
    # non-unit and negated quaternions behave like the reference (normalised for points, raw for origins)
    Q = P.copy()
    for f in ("qx", "qy", "qz", "qw"):
        Q[f] *= np.float32(-1.7)
    check_records(eng.measure(Q, s["lik"], s["beam"], s["origins"]), cpu.measure(Q, s["lik"], s["beam"], s["origins"]), 16)


def test_errors_without_map(eng_mod):
    e = eng_mod.Engine((0,))
    with pytest.raises(eng_mod.EngineError) as ei:
        e.measure(synth.make_poses([[0, 0, 0]], [[0, 0, 0, 1]]), synth.make_points([[1, 0, 0]]), None, None)
    assert ei.value.code == -2
    e.close()


def test_large_scan_unstaged_path(eng_mod, eng, cc):
    """More scan points than fit the shared-memory tile (> 200 KiB): the direct-from-global variant."""
    s = synth.scene(30_000, 6, 13_500, 13_000, seed=31)
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 5), 64)
    check_records(eng.measure(s["particles"], s["lik"], s["beam"], s["origins"]),
                  cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"]), 13_000)


def test_set_params_and_restage(eng_mod, eng, cc):
    s = synth.scene(20_000, 32, 64, 32, seed=41)
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 5), 32)
    a = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    # scalar refresh without restaging (refreshParameters)
    lik2 = eng_mod.LikParams(match_weight=2.5, match_dist_flat=0.1, dist_weight=(1, 1, 5))
    eng.set_params(lik2, None)
    b = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    assert np.array_equal(a["n_hit"], b["n_hit"]) and not np.array_equal(a["score_like"], b["score_like"])
    port = cc.CpuChecker("port")
    cpu2 = port.create(s["map"], cc.lik_params(2.5, 0.2, 0.1, (1, 1, 5)), cc.beam_raw(num_points_default=32), 20.0, 0.4)
    check_records(b, cpu2.measure(s["particles"], s["lik"], s["beam"], s["origins"]), 32)
    # changing the radius needs a restage
    with pytest.raises(eng_mod.EngineError):
        eng.set_params(eng_mod.LikParams(match_dist_min=0.3, dist_weight=(1, 1, 5)), None)


# ------------------------------------------------------------------ full-size properties (BASELINE configs 2 and 3)
@pytest.fixture(scope="module")
def big_scene():
    return synth.scene(1_000_000, 4096, 512, 256, seed=51)


def test_full_size_properties(eng_mod, eng, cc, big_scene):
    s = big_scene
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=256, dda_grid_size=0.2)
    eng.set_map(s["map"], lik, beam)
    P = s["particles"]
    full = eng.measure(P[:1024], s["lik"], None, None)            # config 2: 1024 x 512 likelihood
    beam_full = eng.measure(P, None, s["beam"], s["origins"])     # config 3: 4096 x 256 beam DDA
    # (1) permutation equivariance over particles, bit-exact (deterministic reductions)
    perm = np.random.default_rng(5).permutation(1024)
    assert np.array_equal(eng.measure(P[:1024][perm], s["lik"], None, None), full[perm])
    # (2) scan additivity: counts add exactly, scores to rounding
    a = eng.measure(P[:1024], s["lik"][:200], None, None)
    b = eng.measure(P[:1024], s["lik"][200:], None, None)
    assert np.array_equal(a["match_cnt"] + b["match_cnt"], full["match_cnt"])
    assert np.allclose(a["score_like"] + b["score_like"], full["score_like"], rtol=1e-5, atol=1e-5)
    # (3) every ray is classified exactly once; beam tallies add over a split of the rays
    assert ((beam_full["n_short"] + beam_full["n_hit"] + beam_full["n_long"]) == 256).all()
    h1 = eng.measure(P, None, s["beam"][:100], s["origins"])
    h2 = eng.measure(P, None, s["beam"][100:], s["origins"])
    for f in ("n_short", "n_hit", "n_long"):
        assert np.array_equal(h1[f] + h2[f], beam_full[f])
    # (4) duplicated particles give identical records; idempotence of repeated calls
    dup = np.concatenate([P[:7], P[:7]])
    d = eng.measure(dup, s["lik"], s["beam"], s["origins"])
    assert np.array_equal(d[:7], d[7:])
    assert np.array_equal(eng.measure(P[:1024], s["lik"], None, None), full)
    # (5) a strided sample of the full-size job against the oracle
    port = cc.CpuChecker("port")
    cpu = port.create(s["map"], cc.lik_params(dist_weight=(1, 1, 5)), cc.beam_raw(num_points_default=256), 20.0, 0.4)
    idx = np.arange(0, 4096, 128)
    want = cpu.measure(P[idx], s["lik"], s["beam"], s["origins"])
    got = eng.measure(P[idx], s["lik"], s["beam"], s["origins"])
    check_records(got, want, 256)
    assert np.array_equal(got["n_hit"], beam_full["n_hit"][idx])


def test_device_resident_entry_matches_host_entry(eng_mod, eng, big_scene):
    import torch
    s = big_scene
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=256, dda_grid_size=0.2)
    eng.set_map(s["map"], lik, beam)
    P = s["particles"][:777]
    want = eng.measure(P, s["lik"], s["beam"], s["origins"])
    dev = torch.device("cuda:0")

    def up(a):
        return torch.from_numpy(np.frombuffer(np.ascontiguousarray(a).tobytes(), dtype=np.uint8).copy()).to(dev)
    d_p, d_l, d_b = up(P), up(s["lik"]), up(s["beam"])
    d_o = torch.from_numpy(np.ascontiguousarray(s["origins"], dtype=np.float32)).to(dev)
    d_out = torch.zeros(len(P) * 24, dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    eng.measure_device(d_p.data_ptr(), len(P), d_l.data_ptr(), len(s["lik"]), d_b.data_ptr(), len(s["beam"]),
                       d_o.data_ptr(), len(s["origins"]), d_out.data_ptr(), st)
    torch.cuda.synchronize()
    got = np.frombuffer(d_out.cpu().numpy().tobytes(), dtype=synth.RESULT)
    assert np.array_equal(got, want)


def test_multi_device_engine_matches_single(eng_mod, big_scene):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = big_scene
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=256, dda_grid_size=0.2)
    e1, e2 = eng_mod.Engine((0,)), eng_mod.Engine((0, 1))
    e1.set_map(s["map"], lik, beam)
    e2.set_map(s["map"], lik, beam)
    P = s["particles"][:1001]
    assert np.array_equal(e1.measure(P, s["lik"], s["beam"], s["origins"]), e2.measure(P, s["lik"], s["beam"], s["origins"]))
    e1.close()
    e2.close()


# ------------------------------------------------------------------ BASELINE configs 4 and 5 against the oracle
def test_c4_shape_vs_oracle(eng_mod, eng_mod_engine_tuned, cc):
    """Config 4's shape: a 9.7 M-point map (0.1 m DDA lattice, 4e8 cells; 2.6e8-cell search grid), 16 384 tracking
    particles x (1024 likelihood points + 1024 beam rays).  The whole job runs on the GPU; a strided 256-particle sample
    is compared with the oracle, and the sample's records must equal the full job's rows."""
    eng = eng_mod_engine_tuned
    s = synth.scene(10_000_000, 16384, 1024, 1024, seed=7)
    assert len(s["map"]) > 9_000_000
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 5), 1024, dda_grid=0.1)
    info = eng.map_info()
    assert int(np.prod(np.array(list(info.dda_dims), dtype=np.int64))) > 3e8
    full = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    idx = np.arange(0, 16384, 64)
    want = cpu.measure(s["particles"][idx], s["lik"], s["beam"], s["origins"], n_threads=8)
    check_records(full[idx], want, 1024)
    # the sample run on its own: 256 particles get more threads per particle than 16 384 do, so the likelihood sums are
    # reduced in another order (scores to rounding, everything integer exactly)
    alone = eng.measure(s["particles"][idx], s["lik"], s["beam"], s["origins"])
    check_records(alone, want, 1024)
    for f in ("match_cnt", "n_short", "n_hit", "n_long", "score_beam"):
        assert np.array_equal(alone[f], full[idx][f]), f
    assert want["match_cnt"].sum() > 0 and want["n_hit"].sum() > 0


@pytest.mark.parametrize("n_lik,n_beam", [(64, 8), (8, 0)])
def test_c5_shape_vs_oracle(eng_mod, eng, cc, n_lik, n_beam):
    """Config 5's shape: 65 536 particles spread over the floor plan x 12 headings (global localisation,
    src/mcl_3dl.cpp:1039-1099) on the 1 M-point map; (8, 0) is the node's own point budget in that state
    (num_points_global = 8 likelihood points, 0 beam rays: src/lidar_measurement_model_likelihood.cpp:63-77,
    parameters.cpp:219-220,255-256).  A strided 512-particle sample against the oracle; the rest of the job through
    the sample's rows and the permutation property."""
    s = synth.scene(1_000_000, 65536, n_lik, n_beam, spread=True, seed=57)
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 5), max(n_beam, 1))
    full = eng.measure(s["particles"], s["lik"], s["beam"] if n_beam else None, s["origins"])
    idx = np.arange(0, 65536, 128)
    want = cpu.measure(s["particles"][idx], s["lik"], s["beam"] if n_beam else None, s["origins"], n_threads=8)
    check_records(full[idx], want, n_beam)
    assert want["match_cnt"].sum() > 0
    perm = np.random.default_rng(6).permutation(65536)
    assert np.array_equal(eng.measure(s["particles"][perm], s["lik"], s["beam"] if n_beam else None, s["origins"]), full[perm])


# ------------------------------------------------------------------ scope row f2: fused weight update
@pytest.mark.parametrize("P,seed,with_extra", [(64, 71, False), (1000, 72, True), (65536, 73, True)])
def test_fused_weight_update_vs_pf_measure(eng_mod, eng, cc, P, seed, with_extra):
    """mcl3dl_measure_update == pf::ParticleFilter::measure driven by the node's lambda (pf.h:252-279,
    mcl_3dl.cpp:402-426).  Tolerance 1e-4 relative on posteriors / entropy: the reference sums sequentially
    in float, the device sums in double with a fixed tree."""
    n_lik, n_beam = (96, 3) if P <= 1000 else (16, 2)
    s = synth.scene(50_000, P, n_lik, n_beam, seed=seed)
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 5), n_beam)
    rng = np.random.default_rng(seed)
    prior = rng.uniform(0.1, 1.0, P).astype(np.float32)
    prior /= prior.sum(dtype=np.float64).astype(np.float32)
    extra = rng.uniform(0.5, 1.0, P).astype(np.float32) if with_extra else None
    post, summ, rec = eng.measure_update(s["particles"], s["lik"], s["beam"], s["origins"], prior, extra, want_records=True)
    # the records of the fused path against the ORACLE (every particle, 65 536 included), then against the plain entry
    check_records(rec, cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"], n_threads=8), n_beam)
    want_rec = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    assert np.array_equal(rec, want_rec)
    like = (np.float32(1.0) * want_rec["score_beam"]).astype(np.float32)
    like = (like * want_rec["score_like"]).astype(np.float32)
    if extra is not None:
        like = (like * extra).astype(np.float32)
    port = cc.CpuChecker("port")
    ref_post, ref_ent, ref_kept = port.pf_update(prior, like)
    assert bool(summ["kept"]) == ref_kept and ref_kept
    assert np.allclose(post, ref_post, rtol=1e-4, atol=1e-12)
    assert abs(summ["entropy"] - ref_ent) <= 1e-4 * abs(ref_ent) + 1e-6
    q = want_rec["match_cnt"].astype(np.float32) / np.float32(n_lik)
    assert summ["match_ratio_min"] == min(np.float32(1.0), q.min()) and summ["match_ratio_max"] == max(np.float32(0.0), q.max())
    assert post[summ["max_index"]] == post.max()
    assert abs(float(post.sum(dtype=np.float64)) - 1.0) < 1e-4


def test_fused_weight_update_restores_when_no_particle_survives(eng_mod, eng, cc):
    s = synth.scene(20_000, 50, 32, 4, seed=81)
    run_both(eng_mod, eng, cc, s, (1, 1, 5), 4)
    far = s["particles"].copy()
    far["px"] += np.float32(1e4)  # nothing matches: score_like = 0 for every particle
    prior = np.full(50, 0.02, np.float32)
    post, summ, _ = eng.measure_update(far, s["lik"], s["beam"], s["origins"], prior)
    assert summ["kept"] == 0 and np.array_equal(post, prior) and summ["weight_sum"] == 0.0
    assert summ["match_ratio_max"] == 0.0


def test_multi_device_fused_update_matches_single(eng_mod, big_scene):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = big_scene
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=256, dda_grid_size=0.2)
    e1, e2 = eng_mod.Engine((0,)), eng_mod.Engine((0, 1))
    e1.set_map(s["map"], lik, beam)
    e2.set_map(s["map"], lik, beam)
    P = s["particles"][:1001]
    prior = np.random.default_rng(9).uniform(0.1, 1.0, len(P)).astype(np.float32)
    p1, s1, r1 = e1.measure_update(P, s["lik"], s["beam"], s["origins"], prior, want_records=True)
    p2, s2, r2 = e2.measure_update(P, s["lik"], s["beam"], s["origins"], prior, want_records=True)
    assert np.array_equal(r1, r2)
    assert np.allclose(p1, p2, rtol=1e-6) and s1["kept"] == s2["kept"] == 1
    assert abs(s1["entropy"] - s2["entropy"]) < 1e-5 and s1["max_index"] == s2["max_index"]
    assert s1["match_ratio_min"] == s2["match_ratio_min"] and s1["match_ratio_max"] == s2["match_ratio_max"]
    e1.close()
    e2.close()


def test_dense_cloud_overflows_the_window_table(eng_mod, eng, cc):
    """A raw (not voxel-filtered) cloud: thousands of points per search-grid cell, so the packed per-cell counts of
    the window table saturate and the kernel has to fall back to the CSR bounds; the DDA cells hold long point lists."""
    rng = np.random.default_rng(91)
    pts = rng.uniform(0.0, 1.0, (120_000, 3)).astype(np.float32)
    pts = np.vstack([pts, [[-0.5, -0.5, -0.5], [1.5, 1.5, 1.5]]]).astype(np.float32)
    s = {"map": synth.make_points(pts, (rng.random(len(pts)) < 0.3).astype(np.uint32) * 2)}
    P, n_lik, n_beam = 9, 24, 10
    s["particles"] = synth.make_poses(rng.uniform(0.3, 0.7, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.3, (P, 3))))
    s["lik"] = synth.make_points(rng.uniform(-0.7, 0.7, (n_lik, 3)))
    s["beam"] = synth.make_points(rng.uniform(-0.6, 0.6, (n_beam, 3)), rng.integers(0, 2, n_beam))
    s["origins"] = np.array([[0.0, 0.0, 0.05], [0.02, 0.0, 0.0]], np.float32)
    cpu = run_both(eng_mod, eng, cc, s, (1, 1, 1), n_beam, dda_grid=0.2, flm=1)
    want = cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    got = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    check_records(got, want, n_beam)
    assert want["match_cnt"].sum() > 0
    assert np.array_equal(eng.beam_status(s["particles"], s["beam"], s["origins"]),
                          cpu.beam_status(s["particles"], s["beam"], s["origins"]))


def test_wide_cells_of_the_nn_field(eng_mod, eng, cc):
    """A sparse volume cloud: some voxels keep 15..40 nearest-neighbour candidates (wide cells: byte counts in the side
    table), none more (no overflow cell, so the lean likelihood kernel without the window-search fallback runs)."""
    rng = np.random.default_rng(92)
    s = {"map": synth.make_points(rng.uniform(0.0, 1.0, (600, 3)).astype(np.float32))}
    P, n_lik = 64, 64
    s["particles"] = synth.make_poses(rng.uniform(0.3, 0.7, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.3, (P, 3))))
    s["lik"] = synth.make_points(rng.uniform(-0.7, 0.7, (n_lik, 3)))
    s["beam"] = synth.make_points(rng.uniform(-0.6, 0.6, (8, 3)))
    s["origins"] = np.zeros((1, 3), np.float32)
    for use_dda in (True, False):  # the KD-tree caster's marching search reads the same lists
        cpu = run_both(eng_mod, eng, cc, s, (1, 1, 1), 8, dda_grid=0.2, use_dda=use_dda)
        info = eng.nn_field_info()
        if os.environ.get("MCL3DL_NNF") != "0":  # (without the field the CSR windows are searched: none staged)
            assert info["bytes"] > 0 and info["wide_cells"] > 0
            assert not use_dda or info["overflow_cells"] == 0  # (the KD caster's larger search radius may overflow a few)
        want = cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"])
        got = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
        check_records(got, want, 8)
        assert want["match_cnt"].sum() > 0


@pytest.mark.parametrize("P", [64, 4096, 20000])
def test_page_locked_caller_arrays_are_transferred_in_place(eng_mod, eng_mod_engine_tuned, P):
    """Pose / record arrays from mcl3dl_host_alloc skip the staging copies (poses of >= 64 KB are DMA-ed from where they
    lie; the records are stored - by the kernels up to 8192 particles, by the D2H copy above - where the caller reads
    them): same bytes as the same call on ordinary memory, also after the block went back (ordinary path again)."""
    eng = eng_mod_engine_tuned
    s = synth.scene(40_000, P, 48, 8, seed=77)
    eng.set_map(s["map"], eng_mod.LikParams(dist_weight=(1, 1, 5)),
                eng_mod.beam_params_from_reference(num_points_default=8, dda_grid_size=0.2))
    want = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"]).copy()
    h_p = eng.host_array(P, synth.POSE)
    h_p[...] = s["particles"]
    h_o = eng.host_array(P, synth.RESULT)
    got = eng.measure(h_p, s["lik"], s["beam"], s["origins"], out=h_o)
    assert got.ctypes.data == h_o.ctypes.data            # no hidden copy on the Python side
    assert got.tobytes() == want.tobytes()
    # a slice of a block is still inside the block; results of a second call overwrite the first
    h_o[...] = np.zeros((), synth.RESULT)
    half = P // 2
    want2 = eng.measure(s["particles"][half:], s["lik"], s["beam"], s["origins"]).copy()  # (another P: other lane counts)
    got2 = eng.measure(h_p[half:], s["lik"], s["beam"], s["origins"], out=h_o[half:])
    assert got2.tobytes() == want2.tobytes() and not h_o[:half].tobytes().strip(b"\0")
    keep = h_p.copy()
    eng.host_free(h_p)
    eng.host_free(h_o)
    assert eng.measure(keep, s["lik"], s["beam"], s["origins"]).tobytes() == want.tobytes()


# ------------------------------------------------------------------ engine options
@pytest.mark.parametrize("use_dda", [True, False])
def test_options_change_no_record(eng_mod, monkeypatch, use_dda):
    """The near-field screens, the zero-copy record stores and the timing events are pure performance options:
    every combination returns the records of the plainest configuration byte for byte."""
    s = synth.scene(60_000, 300, 96, 24, seed=131)
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=24, dda_grid_size=0.2, use_raycast_using_dda=use_dda)

    def run(env, timing=False):
        for k in ("MCL3DL_NEAR_K", "MCL3DL_NEAR_KD_K", "MCL3DL_ZEROCOPY_OUT", "MCL3DL_TIMING", "MCL3DL_NNF",
                  "MCL3DL_BEAM", "MCL3DL_BEAM_DQ_PPL"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = eng_mod.Engine((0,))
        e.set_map(s["map"], lik, beam)
        if timing:
            e.collect_timing(True)
        out = e.measure(s["particles"], s["lik"], s["beam"], s["origins"]).copy()
        info, t = e.near_field_info(), e.last_timing()
        e.close()
        return out, info, t

    plain, info0, t0 = run({"MCL3DL_NEAR_K": "0", "MCL3DL_NEAR_KD_K": "0", "MCL3DL_ZEROCOPY_OUT": "0"})
    assert info0[0][0] == 0 and info0[1][0] == 0
    assert t0["lik_ms"] == 0.0 and t0["beam_ms"] == 0.0          # timing events are opt-in
    dflt, info1, _ = run({})
    assert dflt.tobytes() == plain.tobytes()
    assert info1[0][0] == 2 and info1[0][1] > 0 and (info1[1][0] == 1) == (not use_dda)
    timed, _, t1 = run({"MCL3DL_NEAR_K": "1", "MCL3DL_ZEROCOPY_OUT": "100"}, timing=True)   # 300 particles > 100: bulk D2H copy
    assert timed.tobytes() == plain.tobytes()
    assert t1["lik_ms"] > 0.0 and t1["beam_ms"] > 0.0 and t1["h2d_ms"] > 0.0
    def same(a, b):  # another likelihood kernel may sum a particle's likelihood terms in another order
        for f in ("match_cnt", "score_beam", "n_short", "n_hit", "n_long"):
            assert np.array_equal(a[f], b[f]), f
        assert np.allclose(a["score_like"], b["score_like"], rtol=2e-6, atol=1e-6)
    csr, _, _ = run({"MCL3DL_NNF": "0", "MCL3DL_NEAR_K": "3", "MCL3DL_NEAR_KD_K": "2"})  # the CSR-window kernel (no NN field)
    same(csr, plain)
    # both beam kernels (static CTA mapping / dynamic queue with several item sizes): integer tallies, so byte-identical
    for env in ({"MCL3DL_BEAM": "pl"}, {"MCL3DL_BEAM": "dq"}, {"MCL3DL_BEAM": "dq", "MCL3DL_BEAM_DQ_PPL": "1"},
                {"MCL3DL_BEAM": "dq", "MCL3DL_BEAM_DQ_PPL": "7"}):
        got, _, _ = run(env)
        assert got.tobytes() == dflt.tobytes(), env
