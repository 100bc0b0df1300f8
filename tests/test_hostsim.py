"""The product's per-thread device functions, compiled for the HOST (tests/hostsim/) and checked against the oracle.

mcl_3dl_b200/csrc/device_math.cuh and device_funcs.cuh — the SE(3) transform, nn_dist2, nn_search_arg, cast_ray
(DDA), cast_ray_kd (KD-tree caster), ray_origin — are included verbatim by tests/hostsim/hostsim.cpp through a small
intrinsic shim, so an edit to any of them can be checked here without a GPU.  Sequential scan-order sums make even the
likelihood score bit-exact against the oracle.  (The warp-cooperative kernel code is covered by the -m gpu suite.)
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import golden
from mcl_3dl_b200 import engine, synth
from oracle import cpu_checker as cc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS = os.path.join(ROOT, "tests", "hostsim")
LIB = os.path.join(HS, "libhostsim.so")
DEPS = [os.path.join(HS, "hostsim.cpp"), os.path.join(HS, "pf_hostsim.cpp"), os.path.join(HS, "cuda_shim.h"),
        os.path.join(ROOT, "mcl_3dl_b200", "csrc", "pf_funcs.cuh"),
        os.path.join(ROOT, "mcl_3dl_b200", "csrc", "device_funcs.cuh"),
        os.path.join(ROOT, "mcl_3dl_b200", "csrc", "device_math.cuh"), os.path.join(ROOT, "include", "mcl3dl_b200.h")]


@pytest.fixture(scope="module")
def hostsim():
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
        r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", LIB,
                            os.path.join(HS, "hostsim.cpp"), os.path.join(HS, "pf_hostsim.cpp")], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    L = C.CDLL(LIB)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_measure_nf.argtypes = [vp, sz, vp, vp, C.c_float, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp, C.c_int, C.c_int, vp,
                                     C.c_int]

    def run(map_pts, lik, beam, poses, lik_pts, beam_pts, origins, near=(2, 1), work=False, field=1):
        """near = dilation of the (likelihood, KD-caster) near-field screens; 0 = the unscreened searches.
        field = 1: stage the NN field (per-voxel candidate lists) and search through it, as the engine does by default;
        0: the CSR window searches.  work: [nn index entries, nn pts, steps, occupied, tested, field candidates stored,
        field voxels with candidates, field overflow cells, field wide cells]."""
        map_pts = np.ascontiguousarray(map_pts, dtype=synth.POINT)
        poses = np.ascontiguousarray(poses, dtype=synth.POSE)
        lik_pts = np.ascontiguousarray(lik_pts if lik_pts is not None else np.zeros(0, synth.POINT), dtype=synth.POINT)
        beam_pts = np.ascontiguousarray(beam_pts if beam_pts is not None else np.zeros(0, synth.POINT), dtype=synth.POINT)
        origins = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(poses), dtype=synth.RESULT)
        st = np.zeros((len(poses), max(len(beam_pts), 1)), dtype=np.uint8)
        wk = np.zeros(9, dtype=np.uint64)
        p = lambda a: a.ctypes.data_as(vp) if a.size else None  # noqa: E731
        rc = L.hostsim_measure_nf(p(map_pts), len(map_pts), C.byref(lik) if lik is not None else None,
                                  C.byref(beam) if beam is not None else None, 1.0, p(poses), len(poses), p(lik_pts),
                                  len(lik_pts), p(beam_pts), len(beam_pts), p(origins), len(origins), p(out), p(st),
                                  near[0], near[1], p(wk), field)
        assert rc == 0
        if work:
            return out, st[:, :len(beam_pts)], wk
        return out, st[:, :len(beam_pts)]
    return run


@pytest.mark.parametrize("seed,w,spread,use_dda,flm", [
    (1, (1, 1, 1), False, True, 0xFFFFFFFF), (2, (1, 1, 5), False, True, 1), (3, (1, 1, 5), True, True, 0xFFFFFFFF),
    (4, (1, 1, 5), False, False, 0xFFFFFFFF), (5, (1, 1, 1), False, False, 1), (6, (2, 1, 3), True, False, 0xFFFFFFFF),
])
def test_device_functions_on_host_match_oracle(hostsim, port, seed, w, spread, use_dda, flm):
    s = synth.scene(30_000, 40, 48, 20, spread=spread, seed=seed)
    kw = dict(num_points_default=20, dda_grid_size=0.2 if seed % 2 else 0.1, filter_label_max=flm,
              add_penalty_short_only_mode=seed != 3, use_raycast_using_dda=use_dda)
    lik = engine.LikParams(dist_weight=w)
    beam = engine.beam_params_from_reference(**kw)
    cpu = port.create(s["map"], cc.lik_params(dist_weight=w), cc.beam_raw(**kw), 20.0, 0.4 if min(w) >= 1 else 1.0)
    want = cpu.measure(s["particles"], s["lik"], s["beam"], s["origins"])
    got, st = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"])
    for f in want.dtype.names:
        assert np.array_equal(got[f], want[f]), f   # score_like too: same sequential sum
    assert np.array_equal(st, cpu.beam_status(s["particles"], s["beam"], s["origins"]))


@pytest.mark.parametrize("name", ["room_iso", "room_aniso", "room_spread", "room_kd_iso", "room_kd_aniso"])
def test_device_functions_on_host_match_reference_goldens(hostsim, name):
    g = golden(name + ".npz")
    n_beam, flm, short_only = [int(v) for v in g["beam_cfg"]]
    lik = engine.LikParams(dist_weight=tuple(float(v) for v in g["dist_weight"]))
    beam = engine.beam_params_from_reference(num_points_default=n_beam, filter_label_max=flm,
                                             add_penalty_short_only_mode=bool(short_only),
                                             dda_grid_size=float(g["dda_grid"]),
                                             use_raycast_using_dda=bool(int(g["use_dda"])))
    got, st = hostsim(g["map"], lik, beam, g["particles"], g["lik"], g["beam"], g["origins"])
    for f in got.dtype.names:
        assert np.array_equal(got[f], g["result"][f]), f
    assert np.array_equal(st, g["status"])


@pytest.mark.parametrize("near", [(1, 1), (2, 2), (3, 1), (4, 3)])
@pytest.mark.parametrize("seed,w,spread,use_dda", [(11, (1, 1, 1), False, False), (12, (1, 1, 5), True, False),
                                                    (13, (2, 1, 3), False, True), (14, (1, 1, 5), True, True)])
def test_near_field_screens_change_no_result(hostsim, near, seed, w, spread, use_dda):
    """The near-field bits only skip searches that cannot succeed: records and per-ray status are identical with
    and without them, for several dilations, while the work counters drop."""
    s = synth.scene(30_000, 24, 40, 16, spread=spread, seed=seed)
    lik = engine.LikParams(dist_weight=w, match_dist_min=0.2 if seed % 2 else 0.35)
    beam = engine.beam_params_from_reference(num_points_default=16, use_raycast_using_dda=use_dda)
    ref, st_ref, wk_ref = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"], near=(0, 0), work=True,
                                  field=0)
    got, st, wk = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"], near=near, work=True, field=0)
    assert got.tobytes() == ref.tobytes()
    assert np.array_equal(st, st_ref)
    assert wk[0] < wk_ref[0] and wk[1] <= wk_ref[1]          # likelihood: fewer windows opened
    if not use_dda:
        assert wk[4] < wk_ref[4] and wk[3] == wk_ref[3]      # KD caster: fewer points tested, same collisions


@pytest.mark.parametrize("seed,w,spread,use_dda,r", [(21, (1, 1, 1), False, False, 0.2), (22, (1, 1, 5), True, False, 0.2),
                                                      (23, (2, 1, 3), False, True, 0.35), (24, (1, 1, 5), False, True, 0.2),
                                                      (25, (0.5, 2, 1), True, False, 0.1)])
def test_nn_field_changes_no_result(hostsim, seed, w, spread, use_dda, r):
    """The NN field (per-voxel candidate lists, device_funcs.cuh: nnf_select / nnf_dist2 / nnf_search_arg) against the
    CSR window searches: records — likelihood scores bit for bit — and per-ray status are identical, and far fewer map
    points are distance-tested."""
    s = synth.scene(30_000, 24, 64, 24, spread=spread, seed=seed)
    lik = engine.LikParams(dist_weight=w, match_dist_min=r)
    beam = engine.beam_params_from_reference(num_points_default=24, use_raycast_using_dda=use_dda)
    ref, st_ref, wk_ref = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"], near=(0, 0), work=True,
                                  field=0)
    got, st, wk = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"], near=(2, 1), work=True, field=1)
    assert got.tobytes() == ref.tobytes()
    assert np.array_equal(st, st_ref)
    assert wk[5] > 0 and wk[6] > 0 and wk[7] == 0             # candidates stored, no overflow cell on a voxel-filtered map
    assert wk[1] < wk_ref[1]                                  # fewer map points tested by the likelihood evals
    assert wk[5] / wk[6] < 8.0                                # a handful of candidates per voxel
    if not use_dda:
        assert wk[4] < wk_ref[4] and wk[3] == wk_ref[3]      # KD caster: fewer points tested, same collisions


def test_nn_field_overflow_cells_fall_back(hostsim, port):
    """A raw cloud with thousands of points per voxel: more than 14 candidates survive in most voxels (wide cells, byte
    counts in the side table) and more than 40 in some (overflow cells: the queries there run the CSR window search) —
    same records as the oracle."""
    rng = np.random.default_rng(91)
    pts = rng.uniform(0.0, 1.0, (20_000, 3)).astype(np.float32)
    mp = synth.make_points(pts)
    P, n_lik = 5, 40
    poses = synth.make_poses(rng.uniform(0.3, 0.7, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.3, (P, 3))))
    scan = synth.make_points(rng.uniform(-0.7, 0.7, (n_lik, 3)))
    lik = engine.LikParams(dist_weight=(1, 1, 1))
    cpu = port.create(mp, cc.lik_params(dist_weight=(1, 1, 1)), None, 20.0, 0.4)
    want = cpu.measure(poses, scan, None, np.zeros((1, 3), np.float32))
    got, _, wk = hostsim(mp, lik, None, poses, scan, None, np.zeros((1, 3), np.float32), work=True, field=1)
    assert np.array_equal(got["match_cnt"], want["match_cnt"]) and np.array_equal(got["score_like"], want["score_like"])
    assert wk[7] > 0 and wk[8] > 0 and want["match_cnt"].sum() > 0


def _sparse_volume_scene(n_map=600, P=64, n_lik=64, seed=92):
    """A uniform random cloud sparse enough that no voxel keeps more than 40 candidates but some keep more than 14."""
    rng = np.random.default_rng(seed)
    mp = synth.make_points(rng.uniform(0.0, 1.0, (n_map, 3)).astype(np.float32))
    poses = synth.make_poses(rng.uniform(0.3, 0.7, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.3, (P, 3))))
    scan = synth.make_points(rng.uniform(-0.7, 0.7, (n_lik, 3)))
    return mp, poses, scan


def test_nn_field_wide_cells_change_no_result(hostsim):
    """Voxels with 15..40 candidates live in wide cells (byte counts in a side table, device_funcs.cuh: nnf_slot): the
    records equal the CSR window search's bit for bit and no cell overflows."""
    mp, poses, scan = _sparse_volume_scene()
    lik = engine.LikParams(dist_weight=(1, 1, 1))
    org = np.zeros((1, 3), np.float32)
    ref, _ = hostsim(mp, lik, None, poses, scan, None, org, near=(0, 0), field=0)
    got, _, wk = hostsim(mp, lik, None, poses, scan, None, org, work=True, field=1)
    assert got.tobytes() == ref.tobytes()
    assert wk[8] > 0 and wk[7] == 0 and ref["match_cnt"].sum() > 0


def test_nn_field_directory_decoding(hostsim):
    """nnf_slot: nibble counts of a regular cell, byte counts of a wide cell (side table), the overflow marker - against
    plain prefix sums, for every voxel position and random counts up to the caps (14 / 40, and up to 255 per byte)."""
    L = C.CDLL(LIB)
    L.hostsim_nnf_slot.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(C.c_uint32), C.c_int, C.POINTER(C.c_uint32)]
    rng = np.random.default_rng(5)
    none = (C.c_uint32 * 4)(0, 0, 0, 0)
    for trial in range(300):
        first = int(rng.integers(0, 2 ** 31 - 400))
        # regular cell
        cnt = rng.integers(0, 15, 8)
        nib = 0
        for k in range(8):
            nib |= int(cnt[k]) << (4 * k)
        for sub in range(8):
            st = C.c_uint32(0)
            assert L.hostsim_nnf_slot(first, nib, none, sub, C.byref(st)) == cnt[sub]
            assert st.value == first + int(cnt[:sub].sum())
        # wide cell: entry `idx` of the side table holds {first, counts 0..3, counts 4..7}
        cnt = rng.integers(0, 256 if trial % 3 == 0 else 41, 8)
        lo = sum(int(cnt[k]) << (8 * k) for k in range(4))
        hi = sum(int(cnt[4 + k]) << (8 * k) for k in range(4))
        idx = int(rng.integers(0, 1000))
        w = (C.c_uint32 * 4)(first, lo, hi, 0)
        for sub in range(8):
            st = C.c_uint32(0)
            assert L.hostsim_nnf_slot(0x80000000 | idx, 0xfffffffe, w, sub, C.byref(st)) == cnt[sub]
            assert st.value == first + int(cnt[:sub].sum())
    st = C.c_uint32(0)
    assert L.hostsim_nnf_slot(0xffffffff, 0xffffffff, none, 3, C.byref(st)) == -1


def test_device_functions_survive_garbage_inputs_under_sanitizers(tmp_path):
    """NaN / inf / 1e30 poses and scan points, one-point maps, zero-length rays: no out-of-bounds access, no signed
    overflow and bounded work in the per-thread device functions (ASan + UBSan build of tests/hostsim/fuzz_main.cpp)."""
    exe = str(tmp_path / "hostsim_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined",
                        "-fno-sanitize-recover=undefined", "-o", exe, os.path.join(HS, "fuzz_main.cpp"),
                        os.path.join(HS, "hostsim.cpp")], capture_output=True, text=True)
    if r.returncode != 0 and "sanitize" in r.stderr:
        pytest.skip("sanitizer runtimes not available: " + r.stderr.splitlines()[0])
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "fuzz ok" in r.stdout


def _near_query(map_xyz, w, r, k, queries, max_bytes=64 << 20):
    hs_lib = C.CDLL(LIB)
    vp, sz = C.c_void_p, C.c_size_t
    hs_lib.hostsim_near_query.argtypes = [vp, sz, vp, C.c_float, C.c_int, sz, vp, sz, vp, vp, vp]
    pts = synth.make_points(np.asarray(map_xyz, dtype=np.float32))
    wv = np.asarray(w, dtype=np.float32)
    q = np.ascontiguousarray(queries, dtype=np.float32)
    out = np.zeros(len(q), dtype=np.uint8)
    lay = np.zeros(4, dtype=np.int32)
    cell = C.c_float(0)
    p = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    assert hs_lib.hostsim_near_query(p(pts), len(pts), p(wv), r, k, max_bytes, p(q), len(q), p(out), p(lay), C.byref(cell)) == 0
    return out.astype(bool), lay, cell.value


@pytest.mark.parametrize("offset", [0.0, 37.5, 4000.0, -65000.0])
@pytest.mark.parametrize("r,k", [(0.2, 1), (0.2, 2), (0.0707, 1), (0.45, 3), (1.5, 4), (0.01, 2)])
def test_near_field_never_hides_a_neighbour(hostsim, r, k, offset):
    """THE invariant of the screens: whenever a map point lies within r of a query (rescaled metric), the query's bit is
    set — for clustered and scattered maps, anisotropic weights, maps far from the origin (float cell arithmetic),
    radii from 1 cm to 1.5 m, and fields that had to be coarsened to fit the byte cap.  A screen that answered "clear"
    here would silently drop a match on the device."""
    rng = np.random.default_rng(int(1000 * r) + 7 * k + int(abs(offset)))
    w = np.array([1.0, 1.0, 5.0] if k % 2 else [2.0, 1.0, 3.0], dtype=np.float32)
    span = 400.0 * r                      # ~400 search radii across: several hundred fine cells per axis
    pts = rng.uniform(0, span, (1500, 3)).astype(np.float32)
    pts[:300] = pts[0] + rng.normal(0, r, (300, 3)).astype(np.float32)   # a dense cluster
    pts += np.float32(offset)
    sc = (pts * w).astype(np.float32)
    # queries: near map points (just inside / just outside the radius), inside the box, far outside it
    d = rng.normal(0, 1, (4000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    near_q = sc[rng.integers(0, len(sc), 4000)] + (d * rng.uniform(0.0, 1.3 * r, (4000, 1))).astype(np.float32)
    box_q = rng.uniform(sc.min(0) - 3 * r, sc.max(0) + 3 * r, (3000, 3)).astype(np.float32)
    far_q = (sc.mean(0) + rng.normal(0, 50 * span, (300, 3))).astype(np.float32)
    q = np.vstack([near_q, box_q, far_q, sc[:200]]).astype(np.float32)
    for cap in (64 << 20, 1 << 16):       # the second cap forces the layout to coarsen the cells
        maybe, lay, cell = _near_query(pts, w, r, k, q, max_bytes=cap)
        assert cell >= 1.0099 * r / k
        assert int(lay[3]) * int(lay[1]) * int(lay[2]) * 4 <= cap
        from scipy.spatial import cKDTree
        dist, _ = cKDTree(sc.astype(np.float64)).query(q.astype(np.float64))
        hidden = (~maybe) & (dist < r * (1 + 1e-6))
        assert not hidden.any(), (int(hidden.sum()), float(dist[hidden].min()))
        # and the screen is not vacuous: far queries are reported clear
        assert not maybe[len(near_q) + len(box_q):len(near_q) + len(box_q) + len(far_q)].all()


def test_near_field_degenerate_maps(hostsim):
    """One point, a flat map, and a bounding box too large for any field (the engine then searches unscreened)."""
    one = np.array([[1.0, 2.0, 3.0]], np.float32)
    maybe, lay, cell = _near_query(one, (1, 1, 1), 0.2, 2, [[1.0, 2.0, 3.1], [5.0, 2.0, 3.0], [np.nan, 0, 0], [np.inf, 0, 0]])
    assert maybe[0] and not maybe[1] and not maybe[3] and cell > 0
    flat = np.array([[x, y, 0.0] for x in range(5) for y in range(5)], np.float32)
    maybe, _, _ = _near_query(flat, (1, 1, 5), 0.3, 1, [[2.0, 2.0, 0.25], [2.0, 2.0, 5.0]])
    assert maybe[0] and not maybe[1]
    huge = np.array([[0, 0, 0], [3e38, 0, 0]], np.float32)
    maybe, lay, cell = _near_query(huge, (1, 1, 1), 0.2, 2, [[0, 0, 0], [1e30, 5, 5]])
    assert cell == 0.0 and maybe.all()


# ------------------------------------------------------------------ scope row f3 groundwork (csrc/pf_funcs.cuh)
def _pf_lib():
    L = C.CDLL(LIB)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_pf_predict.argtypes = [vp, vp, C.c_float, C.c_float, C.c_float, vp, sz]
    L.hostsim_pf_resample_ref_rng.argtypes = [vp, vp, sz, C.c_uint, vp, vp, vp, vp, vp, vp]
    L.hostsim_pf_resample_philox.argtypes = [vp, vp, sz, C.c_float, C.c_uint64, C.c_uint32, vp, vp, vp, vp, vp, vp, vp]
    L.hostsim_philox.argtypes = [vp, C.c_uint32, C.c_uint32]
    L.hostsim_philox.restype = None
    L.hostsim_noise6.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, vp, vp]
    L.hostsim_noise6.restype = None
    return L


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _motion_states(n, seed):
    rng = np.random.default_rng(seed)
    st = np.zeros(n, dtype=cc.MOTION_STATE)
    st["pos"] = rng.uniform(-20, 20, (n, 3))
    q = rng.normal(0, 1, (n, 4))
    st["rot"] = q / np.linalg.norm(q, axis=1, keepdims=True) * rng.uniform(0.98, 1.02, (n, 1))   # nearly unit, as in the node
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        st[f] = rng.normal(0, 0.05, n)
    st["odom_err_integ_lin"] = rng.normal(0, 0.1, (n, 3))
    st["odom_err_integ_ang"] = rng.normal(0, 0.1, (n, 3))
    return st


@pytest.mark.parametrize("seed,turn", [(1, 0.3), (2, -2.9), (3, 0.0), (4, 3.1)])
def test_pf_predict_on_host_equals_oracle(hostsim, port, seed, turn):
    """pf_predict + pf_set_odoms (MotionPredictionModelDifferentialDrive::setOdoms / predict) bit for bit against the
    port, which is pinned to the reference build (test_oracle_golden.py)."""
    L = _pf_lib()
    rng = np.random.default_rng(100 + seed)
    q0 = synth.quat_from_rpy(np.array([[0.02, -0.01, 0.4]]))[0]
    q1 = synth.quat_from_rpy(np.array([[0.01, 0.03, 0.4 + turn]]))[0]
    prev = synth.make_poses(np.array([[1.0, 2.0, 0.1]]), q0[None])
    cur = synth.make_poses(np.array([[1.0, 2.0, 0.1]]) + rng.normal(0, 0.2 if turn else 0.0, (1, 3)), q1[None])
    st = _motion_states(500, seed)
    want = port.motion_predict(prev, cur, 0.1, 10.0, 10.0, st.copy())
    got = st.copy()
    assert L.hostsim_pf_predict(_ptr(prev), _ptr(cur), 0.1, 10.0, 10.0, _ptr(got), len(got)) == 0
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("n,seed,sigma", [(64, 12345, 0.0), (64, 7, 0.05), (1000, 99, 0.02), (4096, 5, 0.1), (3, 1, 0.3)])
def test_pf_resample_on_host_equals_oracle(hostsim, port, n, seed, sigma):
    """pf_pick + pf_add_noise with the reference's random stream: the resampled State6DOF set of
    pf::ParticleFilter::resample (pf.h:182-225) bit for bit, including which outputs count as duplicates."""
    L = _pf_lib()
    rng = np.random.default_rng(seed)
    probs = rng.uniform(0.05, 1.0, n).astype(np.float32) ** 3        # skewed weights: many duplicates
    probs /= probs.sum(dtype=np.float32)
    assert (np.diff(np.cumsum(probs, dtype=np.float32)) > 0).all()   # no accumulated-probability ties (see the test below)
    st = _motion_states(n, seed + 1)
    sp = np.array([sigma, sigma, sigma / 2], np.float32)
    sr = np.array([0.0, sigma / 4, sigma], np.float32)               # one zero sigma: that draw is skipped
    want_s, want_p = port.pf_resample_6dof(probs, st, seed, sp, sr)
    got = np.zeros(n, dtype=cc.MOTION_STATE)
    got_p = np.zeros(n, np.float32)
    src = np.zeros(n, np.uint32)
    dup = np.zeros(n, np.uint8)
    assert L.hostsim_pf_resample_ref_rng(_ptr(probs), _ptr(st), n, seed, _ptr(sp), _ptr(sr), _ptr(got), _ptr(got_p), _ptr(src),
                                         _ptr(dup)) == 0
    assert got.tobytes() == want_s.tobytes() and np.array_equal(got_p, want_p)
    assert (np.diff(src.astype(np.int64)) >= 0).all() and dup.sum() > 0 or n <= 3


def test_pf_resample_ties_go_to_the_lowest_index(hostsim, port):
    """Documented departure: a particle whose weight is below half an ulp of the running sum leaves accum unchanged, so
    two particles tie in the reference's std::sort key; which of them std::lower_bound then meets first is up to the
    (unstable) sort.  The device takes the lowest index, i.e. the particle that actually carries the weight.  Outside
    such tie groups the picks are the reference's."""
    L = _pf_lib()
    n, seed = 4096, 5
    rng = np.random.default_rng(seed)
    probs = rng.uniform(0.01, 1.0, n).astype(np.float32) ** 4
    probs /= probs.sum(dtype=np.float32)
    accum = np.zeros(n, np.float32)
    a = np.float32(0)
    for i in range(n):
        a = np.float32(a + probs[i])
        accum[i] = a
    tie_with_prev = np.concatenate([[False], np.diff(accum) == 0])
    assert tie_with_prev.sum() > 50
    st = _motion_states(n, seed + 1)
    zero = np.zeros(3, np.float32)
    want_s, _ = port.pf_resample_6dof(probs, st, seed, zero, zero)     # sigma 0: picks only
    got = np.zeros(n, dtype=cc.MOTION_STATE)
    got_p = np.zeros(n, np.float32)
    src = np.zeros(n, np.uint32)
    dup = np.zeros(n, np.uint8)
    assert L.hostsim_pf_resample_ref_rng(_ptr(probs), _ptr(st), n, seed, _ptr(zero), _ptr(zero), _ptr(got), _ptr(got_p), _ptr(src),
                                         _ptr(dup)) == 0
    assert not tie_with_prev[src].any()                                 # never a weightless member of a tie group
    differs = np.array([got[i].tobytes() != want_s[i].tobytes() for i in range(n)])
    in_tie_group = tie_with_prev[np.minimum(src + 1, n - 1)]            # the pick heads a tie group
    dup_b = dup.astype(bool)
    # a disagreement needs a tie group at the pick; duplicates differ only through normalize() of the copied state
    assert (~differs | in_tie_group | dup_b).all()
    assert differs.sum() < tie_with_prev.sum() + dup_b.sum()


def test_philox_known_answers(hostsim):
    """Philox-4x32-10 against the Random123 known-answer vectors."""
    L = _pf_lib()
    for ctr, key, want in [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
                           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
                           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
                            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]:
        c = np.array(ctr, dtype=np.uint32)
        L.hostsim_philox(_ptr(c), key[0], key[1])
        assert tuple(int(v) for v in c) == want


def test_device_noise_is_normal_and_independent(hostsim):
    """pf_noise6 (Philox + Box-Muller): zero mean, the requested sigmas, uncorrelated components, different streams per
    output index and per call, and bit-reproducible."""
    L = _pf_lib()
    sigma = np.array([0.1, 0.2, 0.05, 0.0, 0.02, 0.3], np.float32)
    n = 60_000
    out = np.zeros((n, 6), np.float32)
    o = np.zeros(6, np.float32)
    for i in range(n):
        L.hostsim_noise6(1234567890123, i, 7, _ptr(sigma), _ptr(o))
        out[i] = o
    assert (out[:, 3] == 0).all()                                       # sigma == 0: no noise
    live = [0, 1, 2, 4, 5]
    assert np.allclose(out[:, live].mean(0), 0, atol=5 * sigma[live].max() / np.sqrt(n))
    assert np.allclose(out[:, live].std(0), sigma[live], rtol=0.02)
    corr = np.corrcoef(out[:, live].T)
    assert np.abs(corr - np.eye(5)).max() < 0.02
    from scipy import stats
    for k in live:
        assert stats.kstest(out[:, k] / sigma[k], "norm").pvalue > 1e-3
    L.hostsim_noise6(1234567890123, 5, 7, _ptr(sigma), _ptr(o))
    assert np.array_equal(o, out[5])                                    # reproducible
    L.hostsim_noise6(1234567890123, 5, 8, _ptr(sigma), _ptr(o))
    assert not np.array_equal(o, out[5])                                # next resampling call: new numbers


def test_pf_resample_device_semantics(hostsim, port):
    """The device's own resampling (host-drawn initial offset, Philox noise): the picks equal the reference's systematic
    picks for the same offset, duplicates get noise of the right size, plain copies are untouched."""
    L = _pf_lib()
    n = 2000
    rng = np.random.default_rng(3)
    probs = rng.uniform(0.01, 1.0, n).astype(np.float32) ** 3
    probs /= probs.sum(dtype=np.float32)
    st = _motion_states(n, 8)
    sp = np.array([0.05, 0.05, 0.01], np.float32)
    sr = np.array([0.0, 0.0, 0.02], np.float32)
    out = np.zeros(n, dtype=cc.MOTION_STATE)
    out_p = np.zeros(n, np.float32)
    src = np.zeros(n, np.uint32)
    dup = np.zeros(n, np.uint8)
    noise = np.zeros((n, 6), np.float32)
    assert L.hostsim_pf_resample_philox(_ptr(probs), _ptr(st), n, 0.37, 42, 1, _ptr(sp), _ptr(sr), _ptr(out), _ptr(out_p),
                                        _ptr(src), _ptr(dup), _ptr(noise)) == 0
    # systematic picks, restated with numpy on the sequential float prefix sum
    accum = np.zeros(n, np.float32)
    a = np.float32(0)
    for i in range(n):
        a = np.float32(a + probs[i])
        accum[i] = a
    pstep = np.float32(a / np.float32(n))
    pscan = (pstep * np.arange(n, dtype=np.float32) + np.float32(np.float32(0.37) * pstep)).astype(np.float32)
    want_src = np.searchsorted(accum, pscan, side="left")
    assert (want_src < n).all() and np.array_equal(src, want_src)
    want_dup = np.concatenate([[want_src[0] == 0], want_src[1:] == want_src[:-1]])
    assert np.array_equal(dup.astype(bool), want_dup)
    plain = ~want_dup
    assert out[plain].tobytes() == st[want_src[plain]].tobytes()        # copies are bit-identical
    d = out["pos"][want_dup] - st["pos"][want_src[want_dup]]
    assert np.allclose(d, noise[want_dup][:, :3], atol=1e-5)
    assert 0.8 * sp[0] < d[:, 0].std() < 1.2 * sp[0] and abs(d[:, 0].mean()) < 0.01
    assert (out["noise_ll"][want_dup] == 0).all()                       # duplicates are fresh states
    assert np.allclose(np.linalg.norm(out["rot"][want_dup], axis=1), 1.0, atol=1e-5)
    assert np.all(out_p == np.float32(1.0 / n))


def test_pf_funcs_compile_for_sm_90a(tmp_path):
    """The f3 groundwork is device code: nvcc must accept it for sm_90a with the product's flags (no GPU needed)."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-fmad=false", "-std=c++17", "-c",
                        "-o", str(tmp_path / "pf.o"), os.path.join(HS, "pf_compile_check.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_pf_pick_past_the_end_takes_the_last_particle_found(hostsim):
    """pstep * i + initial_p can round above the last accumulated probability: the reference then copies the particle of
    it_prev, without noise (pf.h:208-212).  Forced here with initial_frac one ulp below 1."""
    L = _pf_lib()
    frac = np.float32(0.99999994)
    hits = 0
    for seed in range(400):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(2, 300))
        prob = rng.uniform(0.05, 1.0, n).astype(np.float32)
        acc = np.zeros(n, np.float32)
        a = np.float32(0)
        for i in range(n):
            a = np.float32(a + prob[i])
            acc[i] = a
        pstep = np.float32(a / np.float32(n))
        pscan = (pstep * np.arange(n, dtype=np.float32) + np.float32(frac * pstep)).astype(np.float32)
        ss = np.searchsorted(acc, pscan, side="left")
        found = ss < n
        if found.all():
            continue
        hits += 1
        want = np.where(found, ss, ss[found][-1] if found.any() else 0)
        want_dup = np.concatenate([[ss[0] == 0], ss[1:] == ss[:-1]]) & found
        st = np.zeros(n, dtype=cc.MOTION_STATE)
        st["rot"][:, 3] = 1
        out = np.zeros(n, dtype=cc.MOTION_STATE)
        out_p = np.zeros(n, np.float32)
        src = np.zeros(n, np.uint32)
        dup = np.zeros(n, np.uint8)
        z = np.zeros(3, np.float32)
        assert L.hostsim_pf_resample_philox(_ptr(prob), _ptr(st), n, float(frac), 1, 1, _ptr(z), _ptr(z), _ptr(out), _ptr(out_p),
                                            _ptr(src), _ptr(dup), None) == 0
        assert np.array_equal(src, want) and np.array_equal(dup.astype(bool), want_dup)
    assert hits > 20


def test_pf_resample_equals_oracle_on_many_small_sets(hostsim, port):
    """Several hundred random particle sets of 2..40 particles (unnormalised weights included): bit-identical to the oracle,
    including the quirk that output 0 counts as a duplicate whenever it picks particle 0."""
    L = _pf_lib()
    dup0 = 0
    for seed in range(600):
        rng = np.random.default_rng(seed)
        n = int(rng.integers(2, 40))
        prob = (rng.uniform(0.05, 1.0, n) ** int(rng.integers(1, 4))).astype(np.float32)
        if seed % 3 == 0:
            prob = (prob / prob.sum(dtype=np.float32)).astype(np.float32)
        if not (np.diff(np.cumsum(prob, dtype=np.float32)) > 0).all():
            continue
        st = _motion_states(n, seed)
        sg = np.full(3, 0.01 if seed % 2 else 0.0, np.float32)
        want, _ = port.pf_resample_6dof(prob, st, seed, sg, sg)
        got = np.zeros(n, dtype=cc.MOTION_STATE)
        got_p = np.zeros(n, np.float32)
        src = np.zeros(n, np.uint32)
        dup = np.zeros(n, np.uint8)
        assert L.hostsim_pf_resample_ref_rng(_ptr(prob), _ptr(st), n, seed, _ptr(sg), _ptr(sg), _ptr(got), _ptr(got_p), _ptr(src),
                                             _ptr(dup)) == 0
        assert got.tobytes() == want.tobytes(), seed
        dup0 += int(dup[0])
    assert dup0 > 100


def test_screens_and_nn_field_randomized_differential(hostsim):
    """Forty random configurations (map size, metric weights, match radius, map grid, caster, tracking / spread poses):
    every near-field setting, with and without the NN field, returns the records and per-ray status of the unscreened
    CSR window searches."""
    for seed in range(40):
        rng = np.random.default_rng(seed)
        n_map = int(rng.choice([500, 5000, 30000]))
        w = [(1, 1, 1), (1, 1, 5), (2, 1, 3), (0.5, 2, 1)][seed % 4]
        s = synth.scene(n_map, int(rng.integers(1, 10)), int(rng.integers(1, 60)), int(rng.integers(1, 24)),
                        spread=(seed % 3 == 0), seed=seed)
        lik = engine.LikParams(dist_weight=w, match_dist_min=float(rng.choice([0.1, 0.2, 0.35, 0.6])))
        g = float(rng.choice([0.05, 0.1, 0.2]))
        beam = engine.beam_params_from_reference(map_grid=(g, g, g * float(rng.choice([1, 2]))), num_points_default=8,
                                                 use_raycast_using_dda=bool(seed % 2), dda_grid_size=max(0.2, 2 * g))
        ref, st_ref = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"], near=(0, 0), field=0)
        for near, field in (((2, 1), 1), ((1, 2), 0), ((3, 1), 1)):
            got, st = hostsim(s["map"], lik, beam, s["particles"], s["lik"], s["beam"], s["origins"], near=near, field=field)
            assert got.tobytes() == ref.tobytes() and np.array_equal(st, st_ref), (seed, near, field)


def test_nn_field_volume_clouds_randomized_differential(hostsim):
    """Uniform VOLUME clouds of random density (the maps above are surfaces): regular, wide and overflow cells all occur,
    for both casters (the KD caster's searches go through the same lists at its own radius) — records and per-ray
    status equal the unscreened CSR window searches'."""
    seen_wide = seen_ovf = 0
    for seed in range(16):
        rng = np.random.default_rng(700 + seed)
        n_map = int(rng.choice([150, 400, 900, 2500, 8000]))
        ext = float(rng.choice([1.0, 2.0]))
        mp = synth.make_points(rng.uniform(0.0, ext, (n_map, 3)).astype(np.float32), rng.integers(0, 2, n_map))
        P, n_lik, n_beam = int(rng.integers(2, 12)), int(rng.integers(8, 48)), int(rng.integers(1, 10))
        poses = synth.make_poses(rng.uniform(0.2 * ext, 0.8 * ext, (P, 3)), synth.quat_from_rpy(rng.normal(0, 0.4, (P, 3))))
        lik_pts = synth.make_points(rng.uniform(-0.7 * ext, 0.7 * ext, (n_lik, 3)))
        beam_pts = synth.make_points(rng.uniform(-0.6 * ext, 0.6 * ext, (n_beam, 3)))
        org = np.array([[0.0, 0.0, 0.05]], np.float32)
        w = [(1, 1, 1), (1, 1, 5), (2, 1, 3)][seed % 3]
        lik = engine.LikParams(dist_weight=w, match_dist_min=float(rng.choice([0.1, 0.2, 0.3])))
        g = float(rng.choice([0.05, 0.1]))
        beam = engine.beam_params_from_reference(map_grid=(g, g, g), num_points_default=n_beam,
                                                 use_raycast_using_dda=bool(seed % 2), dda_grid_size=0.2)
        ref, st_ref = hostsim(mp, lik, beam, poses, lik_pts, beam_pts, org, near=(0, 0), field=0)
        got, st, wk = hostsim(mp, lik, beam, poses, lik_pts, beam_pts, org, near=(2, 1), field=1, work=True)
        assert got.tobytes() == ref.tobytes() and np.array_equal(st, st_ref), seed
        seen_wide += int(wk[8] > 0)
        seen_ovf += int(wk[7] > 0)
    assert seen_wide >= 3 and seen_ovf >= 2   # the draw does exercise both special cell kinds


def test_field_mode_trilinear_lookup_on_host(hostsim):
    """field_dist (the opt-in field mode's lookup, device_funcs.cuh) against a numpy trilinear interpolation of the same
    node volume: inside the lattice to float rounding, `clamp` outside, exact at the nodes."""
    L = C.CDLL(LIB)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_field_dist.argtypes = [vp, vp, vp, C.c_float, C.c_float, vp, sz, vp]
    rng = np.random.default_rng(3)
    dims = np.array([9, 7, 6], np.int32)            # nodes per axis (x, y, z)
    nodes = rng.uniform(0.0, 0.2, (dims[2], dims[1], dims[0])).astype(np.float32)
    org, e, clamp = np.array([-1.0, 2.0, 0.5], np.float32), np.float32(0.101), np.float32(0.2)
    q = np.concatenate([rng.uniform(org, org + (dims - 1) * e, (500, 3)),
                        rng.uniform(org - 1.0, org - 0.01, (20, 3)),           # outside
                        org + np.array([[3, 2, 1], [0, 0, 0], [7, 5, 4]]) * e]).astype(np.float32)   # on nodes
    out = np.zeros(len(q), np.float32)
    p = lambda a: a.ctypes.data_as(vp)  # noqa: E731
    assert L.hostsim_field_dist(p(nodes), p(dims), p(org), e, clamp, p(q), len(q), p(out)) == 0
    t = (q.astype(np.float64) - org) / np.float64(e)
    i = np.floor(t).astype(int)
    inside = ((i >= 0) & (i < dims - 1)).all(axis=1)
    f = t - i
    want = np.full(len(q), clamp, np.float64)
    for n in np.nonzero(inside)[0]:
        x, y, z = i[n]
        c = nodes[z:z + 2, y:y + 2, x:x + 2].astype(np.float64)
        cz = c[0] * (1 - f[n, 2]) + c[1] * f[n, 2]
        cy = cz[0] * (1 - f[n, 1]) + cz[1] * f[n, 1]
        want[n] = cy[0] * (1 - f[n, 0]) + cy[1] * f[n, 0]
    assert inside[:500].all() and not inside[500:520].any()
    assert np.allclose(out, want, rtol=0, atol=2e-5)
    assert np.allclose(out[-3:], [nodes[1, 2, 3], nodes[0, 0, 0], nodes[4, 5, 7]], atol=2e-5)
