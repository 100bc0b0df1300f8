"""Global localisation and the resident set's resize on the device (include/mcl3dl_b200.h: mcl3dl_global_localization,
mcl3dl_particles_resize), held to the CPU checkers of oracle/gl_api.h byte for byte: the seeded set from the staged map,
from a host cloud and after map_append; the info counts; every other staged buffer untouched; the error codes; the resize
of non-uniform posteriors against the reference's own resizeParticle; the resized set behaving exactly like the same
set uploaded; and an end-to-end global localisation in a room, shrink rule included.  The VoxelGrid the checkers start
from is tests/hostsim/scan_hostsim.cpp's, which tests/test_gpu_scan_exact.py holds the device to."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from oracle import gl_checker as gc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "gl_hostsim.cpp")
PARITY = os.path.join(ROOT, "oracle", "_ref", "global_localization_parity_test")
IMU = (0.02, -0.03, 0.01, 0.9993)
W = (1.0, 1.0, 5.0)
INVALID_ARG, NO_MAP, TOO_LARGE = -1, -2, -5

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def E():
    from mcl_3dl_b200 import engine
    return engine


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("glhs") / "libglhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    L.hostsim_scan_voxel_grid.restype = C.c_long
    L.hostsim_scan_voxel_grid.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def port():
    gc.build("port")
    return gc.GlChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not gc.available("reference"):
        pytest.skip("oracle/_ref/libmcl3dl_gl_ref.so not built (needs a checkout of the reference at build time)")
    return gc.GlChecker("reference")


def voxel_grid(L, pts, grid):
    pts = np.ascontiguousarray(pts, dtype=synth.POINT)
    out = np.zeros(len(pts), dtype=synth.POINT)
    leaf = np.full(3, np.float32(grid), np.float32)
    m = L.hostsim_scan_voxel_grid(pts.ctypes.data_as(C.c_void_p), len(pts), leaf.ctypes.data_as(C.c_void_p),
                                  out.ctypes.data_as(C.c_void_p))
    return pts.copy() if m < 0 else out[:m]


def want_seed(hs, port, cloud, grid, div_yaw, w=W):
    ds = voxel_grid(hs, cloud, grid)
    s, p = port.gl_seed(ds, grid, div_yaw, IMU, w)
    return ds, s, p


@pytest.fixture(scope="module")
def warehouse():
    return synth.warehouse_map(200_000, seed=3)[0]


@pytest.mark.parametrize("grid,div_yaw", [(0.3, 12), (0.2, 13), (0.5, 1)])
def test_seed_equals_checker_map_and_host_cloud(E, hs, port, warehouse, grid, div_yaw):
    eng = E.Engine((0,))
    eng.set_map(warehouse, E.LikParams(dist_weight=W))
    ds, want_s, want_p = want_seed(hs, port, warehouse, grid, div_yaw)
    info = eng.global_localization(None, grid, div_yaw, IMU, W)
    got_s, got_p = eng.particles_get()
    assert got_s.tobytes() == want_s.tobytes() and got_p.tobytes() == want_p.tobytes()
    n_seeds = len(want_s) // div_yaw
    assert info["n_input"] == len(warehouse) and info["n_downsampled"] == len(ds)
    assert info["n_seeds"] == n_seeds and info["n_particles"] == len(want_s) and 0 < n_seeds < len(ds)
    assert np.float32(info["probability"]) == want_p[0] == np.float32(1.0 / np.float32(n_seeds))
    seeds = got_s["pos"][::div_yaw]
    assert np.array_equal(seeds.view(np.uint32), want_s["pos"][::div_yaw].view(np.uint32))
    # the same cloud from the host
    info2 = eng.global_localization(warehouse, grid, div_yaw, IMU, W)
    s2, p2 = eng.particles_get()
    assert s2.tobytes() == got_s.tobytes() and p2.tobytes() == got_p.tobytes()
    assert {k: v for k, v in info2.items() if k != "build_ms"} == {k: v for k, v in info.items() if k != "build_ms"}
    eng.close()


def test_seed_after_map_append(E, hs, port, warehouse):
    eng = E.Engine((0,))
    base, patch = warehouse[:150_000], warehouse[150_000:]
    eng.set_map(base, E.LikParams(dist_weight=W))
    eng.map_append(patch)
    _, want_s, want_p = want_seed(hs, port, np.concatenate([base, patch]), 0.3, 12)
    eng.global_localization(None, 0.3, 12, IMU, W)
    got_s, got_p = eng.particles_get()
    assert got_s.tobytes() == want_s.tobytes() and got_p.tobytes() == want_p.tobytes()
    eng.close()


def test_other_state_untouched(E):
    """The staged map's records, the prepared scans and the matched / unmatched output are byte-identical before and after."""
    s = synth.scene(60_000, 300, 64, 8, seed=31)
    eng = E.Engine((0,))
    eng.set_map(s["map"], E.LikParams(dist_weight=W), E.beam_params_from_reference(num_points_default=8))
    raw = np.tile(np.concatenate([s["lik"], s["beam"]]), 20)
    raw["x"] += np.random.default_rng(1).normal(0, 0.03, len(raw)).astype(np.float32)
    eng.scan_prepare(raw, E.ScanParams(lik_num_points=96, beam_num_points=6, seed=3))

    def snapshot():
        rec = eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])
        scans = [eng.scan_get(k).tobytes() for k in range(5)]
        m, u = eng.match_output(s["particles"][0])
        return rec.tobytes(), scans, m.tobytes(), u.tobytes()

    before = snapshot()
    eng.global_localization(None, 0.3, 12, IMU, W)
    assert snapshot() == before
    eng.close()


def test_error_codes(E, warehouse):
    eng = E.Engine((0,))
    with pytest.raises(E.EngineError) as e:
        eng.global_localization(None)
    assert e.value.code == NO_MAP
    eng.set_map(warehouse[:20_000], E.LikParams(dist_weight=W))
    st = np.zeros(10, synth.STATE)
    st["pos"][:, 0] = np.arange(10)
    eng.particles_set(st, np.full(10, 0.1, np.float32))
    for kw in ({"grid": 0.0}, {"grid": -0.3}, {"grid": float("nan")}, {"grid": float("inf")}, {"div_yaw": 0},
               {"dist_weight": (1, 1, 0)}):
        with pytest.raises(E.EngineError) as e:
            eng.global_localization(None, **kw)
        assert e.value.code == INVALID_ARG, kw
    # n_seeds * div_yaw >= 2^31: refused after the seeds are counted and before the set is touched
    with pytest.raises(E.EngineError) as e:
        eng.global_localization(None, 0.3, 2 ** 30, IMU, W)
    assert e.value.code == TOO_LARGE
    # an empty host cloud and a cloud with no survivor: OK, zero counts, the set unchanged
    assert eng.global_localization(np.zeros(0, synth.POINT))["n_particles"] == 0
    info = eng.global_localization(warehouse[:20_000], 0.3, 12, IMU, (1, 1, 0.5))
    assert info["n_seeds"] == 0 and info["n_particles"] == 0 and info["n_downsampled"] > 0
    s, p = eng.particles_get()
    assert s.tobytes() == st.tobytes() and np.all(p == np.float32(0.1))
    for num in (0, 2 ** 31):
        with pytest.raises(E.EngineError) as e:
            eng.particles_resize(num)
        assert e.value.code == INVALID_ARG
    eng.close()
    fresh = E.Engine((0,))
    with pytest.raises(E.EngineError) as e:
        fresh.particles_resize(5)  # no resident set
    assert e.value.code == INVALID_ARG
    fresh.close()


def posterior_set(E, eng, s, n_map_seed_grid=0.3):
    """The seeded set of the scene's map with the posteriors of one resident update (non-uniform, some underflow)."""
    eng.global_localization(None, n_map_seed_grid, 12, IMU, W)
    eng.particles_measure_update(s["lik"], s["beam"], s["origins"])
    return eng.particles_get()


def resize_matches(port, ref, states, probs, num, got):
    want = port.resize(states, probs, num)
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()
    # the reference's std::sort may reorder particles that tie in accum; elsewhere it must agree byte for byte
    r = ref.resize(states, probs, num)
    assert r[1].tobytes() == got[1].tobytes()
    a = got[0].view(np.uint8).reshape(num, -1)
    b = r[0].view(np.uint8).reshape(num, -1)
    bad = np.flatnonzero((a != b).any(axis=1))
    if len(bad):
        acc = np.cumsum(probs, dtype=np.float32)  # sequential, as the filter sums
        tied = np.flatnonzero(np.diff(acc) == 0) + 1
        tied_states = {states[i].tobytes() for i in np.concatenate([tied, tied - 1])}
        assert all(got[0][i].tobytes() in tied_states and r[0][i].tobytes() in tied_states for i in bad), bad[:10]
    print("resize %d -> %d: %d outputs differ from the reference, all on ties" % (len(states), num, len(bad)))


@pytest.mark.parametrize("n_map,factor", [(200_000, 0.75), (200_000, 1.3), (1_000_000, 0.75), (1_000_000, 1.1)])
def test_resize_equals_reference(E, port, ref, n_map, factor):
    s = synth.scene(n_map, 8, 96, 8, seed=5)
    eng = E.Engine((0,))
    eng.set_map(s["map"], E.LikParams(dist_weight=W), E.beam_params_from_reference(num_points_default=8))
    states, probs = posterior_set(E, eng, s)
    assert len(np.unique(probs)) > 100
    num = max(1, int(len(states) * factor))
    eng.particles_resize(num)
    got = eng.particles_get()
    assert len(got[0]) == num
    resize_matches(port, ref, states, probs, num, got)
    eng.close()


def test_resized_set_behaves_like_uploaded(E):
    s = synth.scene(200_000, 8, 96, 8, seed=6)
    lik, beam = E.LikParams(dist_weight=W), E.beam_params_from_reference(num_points_default=8)
    a, b = E.Engine((0,)), E.Engine((0,))
    a.set_map(s["map"], lik, beam)
    b.set_map(s["map"], lik, beam)
    a.global_localization(None, 0.3, 12, IMU, W)
    a.particles_measure_update(s["lik"], s["beam"], s["origins"])
    a.particles_resize(int(a._n_resident * 0.75))
    st, pr = a.particles_get()
    b.particles_set(st, pr)
    for eng in (a, b):
        eng.particles_measure_update(s["lik"], s["beam"], s["origins"])
    sa, sb = a.particles_get(), b.particles_get()
    assert sa[0].tobytes() == sb[0].tobytes() and sa[1].tobytes() == sb[1].tobytes()
    ea, eb = a.particles_estimate(None), b.particles_estimate(None)
    for k in ("mean_biased", "max_state", "cov"):
        assert np.asarray(ea[k]).tobytes() == np.asarray(eb[k]).tobytes(), k
    for eng in (a, b):
        eng.particles_resample((0.05, 0.05, 0.05), (0.05, 0.05, 0.05), 0.37, 99)
    ra, rb = a.particles_get(), b.particles_get()
    assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes()
    a.close()
    b.close()


def room_map(rng):
    """A 6 x 4 m floor with 2 m walls and two boxes against the walls (no symmetry), 0.05 m point pitch."""
    pts = []
    h = 0.05
    xs, ys, zs = np.arange(0, 6.0, h), np.arange(0, 4.0, h), np.arange(0, 2.0, h)
    X, Y = np.meshgrid(xs, ys)
    pts.append(np.stack([X.ravel(), Y.ravel(), np.zeros(X.size)], 1))
    for x0, y0, sx, sy, sz in ((4.6, 0.0, 1.4, 1.0, 1.0), (0.0, 2.8, 0.8, 1.2, 0.6)):
        for a in np.arange(0, sx + 1e-6, h):
            for z in np.arange(0, sz + 1e-6, h):
                pts.append([[x0 + a, y0, z], [x0 + a, y0 + sy, z]])
        for b in np.arange(0, sy + 1e-6, h):
            for z in np.arange(0, sz + 1e-6, h):
                pts.append([[x0, y0 + b, z], [x0 + sx, y0 + b, z]])
        A, B = np.meshgrid(np.arange(0, sx + 1e-6, h), np.arange(0, sy + 1e-6, h))
        pts.append(np.stack([x0 + A.ravel(), y0 + B.ravel(), np.full(A.size, sz)], 1))
    Z, Xw = np.meshgrid(zs, xs)
    pts.append(np.stack([Xw.ravel(), np.zeros(Xw.size), Z.ravel()], 1))
    pts.append(np.stack([Xw.ravel(), np.full(Xw.size, 4.0), Z.ravel()], 1))
    Z, Yw = np.meshgrid(zs, ys)
    pts.append(np.stack([np.zeros(Yw.size), Yw.ravel(), Z.ravel()], 1))
    pts.append(np.stack([np.full(Yw.size, 6.0), Yw.ravel(), Z.ravel()], 1))
    xyz = np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in pts])
    xyz += rng.normal(0, 0.005, xyz.shape)
    return synth.make_points(xyz.astype(np.float32))


def test_end_to_end_room(E):
    """Seed from the map, then resident cycles (scan_prepare, measure_update_prepared, estimate, resample, the node's
    shrink rule) with fixed seeds: the count follows max(int(P * 0.75), num_particles) exactly, and the estimate ends
    within 0.2 m / 0.2 rad of the truth."""
    rng = np.random.default_rng(0)
    mp = room_map(rng)
    truth_pos, truth_yaw = np.array([2.2, 1.6, 0.0]), 0.6
    truth_q = synth.quat_from_rpy(np.array([[0.0, 0.0, truth_yaw]]))[0]
    raw = synth.make_scan(mp, truth_pos, truth_q, 6000, 0.3, 10.0, sigma=0.01, seed=7)
    origins = np.zeros((1, 3), np.float32)
    eng = E.Engine((0,))
    eng.set_map(mp, E.LikParams(dist_weight=(1, 1, 1)), E.beam_params_from_reference(num_points_default=16))
    info = eng.global_localization(None, 0.3, 12, (0, 0, 0, 1), (1, 1, 1))
    num_particles = 256
    count = info["n_particles"]
    assert count > num_particles
    sp = E.ScanParams(downsample=(0.1, 0.1, 0.1), lik_clip=(0.3, 10.0, -2.0, 2.0), beam_clip=(0.3, 4.0, -2.0, 2.0),
                      lik_num_points=256, beam_num_points=16, seed=1)
    est = None
    frac = np.random.default_rng(5)
    for cycle in range(40):
        sp.seed = 1000 + cycle
        eng.scan_prepare(raw, sp)
        eng.particles_measure_update_prepared(origins)
        est = eng.particles_estimate(None if count > num_particles else est["mean_biased"], 1.0, 1.0)
        eng.particles_resample((0.05, 0.05, 0.05), (0.05, 0.05, 0.05), float(frac.uniform(0, 1)), 77)
        if count > num_particles:
            reduced = int(count * 0.75)
            count = reduced if reduced > num_particles else num_particles
            eng.particles_resize(count)
        st, _ = eng.particles_get()
        assert len(st) == count
    m = est["mean_biased"][0]
    q = np.array([m["qx"], m["qy"], m["qz"], m["qw"]], np.float64)
    q /= np.linalg.norm(q)
    yaw = np.arctan2(2 * (q[3] * q[2] + q[0] * q[1]), 1 - 2 * (q[1] ** 2 + q[2] ** 2))
    d = np.hypot(m["px"] - truth_pos[0], m["py"] - truth_pos[1])
    dyaw = abs((yaw - truth_yaw + np.pi) % (2 * np.pi) - np.pi)
    print("end to end: %d seeds, final %d particles, pos error %.3f m, yaw error %.3f rad" % (info["n_seeds"], count, d, dyaw))
    assert count == num_particles
    assert d < 0.2 and dyaw < 0.2, (d, dyaw)
    eng.close()


def test_adapter_parity():
    """The adapter's globalLocalizationResident + resizeResident against the service body and pf_->resizeParticle on the
    reference filter (oracle/global_localization_parity_test.cpp)."""
    if not os.path.exists(PARITY):
        pytest.skip("oracle/_ref/global_localization_parity_test not built (needs a checkout of the reference at build time)")
    for args in (["512", "12"], ["2000", "13"]):
        r = subprocess.run([PARITY] + args, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        assert "GLOBAL LOCALIZATION PARITY OK" in r.stdout
