"""Global localisation and the resident set's resize without a GPU: the device functions of
mcl_3dl_b200/csrc/gl_funcs.cuh, compiled for the host by tests/hostsim/gl_hostsim.cpp, equal both CPU checkers bit for
bit — the port (oracle/gl_oracle.cpp) and the reference tier (oracle/gl_ref_driver.cpp: the reference's own
ParticleFilter::resizeParticle, Quat, Vec3 and State6DOF and the shim KdTreeFLANN).

The checkers take the downsampled cloud from hostsim_scan_voxel_grid (PCL is absent; that VoxelGrid is the one
tests/test_gpu_scan_exact.py holds the device to), so the seeds are compared from the free-space filter on."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from oracle import gl_checker as gc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "gl_hostsim.cpp")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("glhs") / "libglhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    L.hostsim_scan_voxel_grid.restype = C.c_long
    L.hostsim_scan_voxel_grid.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.hostsim_gl_seed.restype = C.c_long
    L.hostsim_gl_seed.argtypes = [C.c_void_p, C.c_size_t, C.c_double, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.POINTER(C.c_uint64)]
    L.hostsim_gl_probability.restype = C.c_float
    L.hostsim_gl_probability.argtypes = [C.c_uint64]
    L.hostsim_gl_resize.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_void_p]
    return L


@pytest.fixture(scope="module")
def port():
    gc.build("port")
    return gc.GlChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not gc.build("reference"):
        pytest.skip("reference checker not built (no reference checkout)")
    return gc.GlChecker("reference")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def voxel_grid(L, pts, grid):
    """The downsampled cloud of the service's VoxelGrid (leaf float(grid)), as the device computes it."""
    pts = np.ascontiguousarray(pts, dtype=synth.POINT)
    out = np.zeros(len(pts), dtype=synth.POINT)
    leaf = np.full(3, np.float32(grid), np.float32)
    m = L.hostsim_scan_voxel_grid(_p(pts), len(pts), _p(leaf), _p(out))
    return pts.copy() if m < 0 else out[:m]


def hs_seed(L, ds, grid, div_yaw, imu=(0, 0, 0, 1), w=(1, 1, 1)):
    ds = np.ascontiguousarray(ds, dtype=synth.POINT)
    q = np.ascontiguousarray(imu, np.float32)
    wv = np.ascontiguousarray(w, np.float32)
    states = np.zeros(len(ds) * div_yaw, synth.STATE)
    probs = np.zeros(len(ds) * div_yaw, np.float32)
    ns = C.c_uint64(0)
    n = L.hostsim_gl_seed(_p(ds), len(ds), grid, div_yaw, _p(q), _p(wv), _p(states), _p(probs), C.byref(ns))
    assert n >= 0
    return states[:n], probs[:n], ns.value


def hs_resize(L, states, probs, num):
    states = np.ascontiguousarray(states, synth.STATE)
    probs = np.ascontiguousarray(probs, np.float32)
    out_s = np.zeros(num, synth.STATE)
    out_p = np.zeros(num, np.float32)
    L.hostsim_gl_resize(_p(probs), _p(states), len(states), num, _p(out_s), _p(out_p))
    return out_s, out_p


def same(a, b):
    """byte equality of two (states, probs) pairs"""
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def random_cloud(seed, n=6000):
    """Points in a 6 x 6 x 3 m box, denser in a few slabs, so that many voxels have a neighbour just above them."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform([0, 0, 0], [6, 6, 3], (n, 3))
    xyz[: n // 2, 2] = rng.choice([0.05, 0.4, 1.2], n // 2) + rng.normal(0, 0.03, n // 2)
    return synth.make_points(xyz.astype(np.float32), rng.integers(0, 3, n))


IMU = (0.02, -0.03, 0.01, 0.9993)  # a slightly tilted, not exactly unit imu_quat
SEED_CASES = [("warehouse", 0, 0.3, (1, 1, 1), 12), ("warehouse", 1, 0.2, (1, 1, 5), 13), ("warehouse", 2, 0.5, (1, 1, 1), 1),
              ("random", 3, 0.3, (1, 1, 5), 12), ("random", 4, 0.2, (1, 1, 1), 13), ("random", 5, 0.5, (1, 1, 5), 1)]


@pytest.mark.parametrize("kind,seed,grid,w,div_yaw", SEED_CASES)
def test_seed_equals_both_checkers(hs, port, ref, kind, seed, grid, w, div_yaw):
    cloud = synth.warehouse_map(20_000, seed=seed + 1)[0] if kind == "warehouse" else random_cloud(seed)
    ds = voxel_grid(hs, cloud, grid)
    got_s, got_p, n_seeds = hs_seed(hs, ds, grid, div_yaw, IMU, w)
    assert 0 < n_seeds < len(ds)  # the filter dropped some voxels and kept some
    assert len(got_s) == n_seeds * div_yaw
    for chk in (port, ref):
        assert same((got_s, got_p), chk.gl_seed(ds, grid, div_yaw, IMU, w)), chk.kind
    # the seeds are every div_yaw-th particle's position, in the downsampled cloud's order
    pos = got_s["pos"][::div_yaw]
    idx = [int(np.flatnonzero((ds["x"] == p[0]) & (ds["y"] == p[1]) & (ds["z"] == p[2]))[0]) for p in pos[:50]]
    assert idx == sorted(idx)
    assert np.all(got_p == np.float32(1.0 / np.float32(n_seeds)))


@pytest.mark.parametrize("div_yaw", [1, 12, 13, 360])
def test_yaw_table_identity_imu(hs, ref, div_yaw):
    """The headings with imu_quat = identity (the node's value before any IMU message), every bit of them."""
    ds = synth.make_points(np.array([[0.0, 0.0, 0.0]], np.float32))
    got_s, _, _ = hs_seed(hs, ds, 0.3, div_yaw)
    want_s, _ = ref.gl_seed(ds, 0.3, div_yaw)
    assert got_s.tobytes() == want_s.tobytes()


def test_radius_boundary(hs, port, ref):
    """Grid 0.5 (r2 = 0.25 exactly): a point B at dx = 0.5 beside A's raised query has d2 == r2 and does not drop A;
    one float closer, it does."""
    z = np.float32(0.51)  # float(0.0 + (0.01 + 0.5))
    edge = np.float32(0.5)
    inside = np.nextafter(edge, np.float32(0))
    for bx, want in ((edge, 2), (inside, 1)):
        ds = synth.make_points(np.array([[0.0, 0.0, 0.0], [bx, 0.0, z]], np.float32))
        got_s, got_p, n_seeds = hs_seed(hs, ds, 0.5, 1)
        assert n_seeds == want
        if want == 1:
            assert got_s["pos"][0][0] == bx  # A dropped, B kept
        for chk in (port, ref):
            assert same((got_s, got_p), chk.gl_seed(ds, 0.5, 1)), chk.kind


def test_no_survivors(hs, port, ref):
    """With dist_weight z = 0.5 every point's own raised query lies within grid of itself: nothing survives."""
    ds = voxel_grid(hs, random_cloud(7, 2000), 0.3)
    got_s, got_p, n_seeds = hs_seed(hs, ds, 0.3, 12, IMU, (1, 1, 0.5))
    assert n_seeds == 0 and len(got_s) == 0
    for chk in (port, ref):
        s, p = chk.gl_seed(ds, 0.3, 12, IMU, (1, 1, 0.5))
        assert len(s) == 0 and len(p) == 0


def test_probability_rule_above_2_24(hs):
    """float(1.0 / float(n_seeds)): above 2^24 the count is rounded to float first, which changes the result."""
    differs = 0
    for n in (1, 3, 80_000, 2 ** 24 - 1, 2 ** 24 + 1, 2 ** 24 + 3, 100_000_007, 2 ** 31 - 1):
        want = np.float32(1.0 / np.float64(np.float32(n)))
        got = np.float32(hs.hostsim_gl_probability(n))
        assert got.tobytes() == want.tobytes(), n
        differs += got != np.float32(1.0 / n)
    assert differs > 0


# ---- resize
def random_states(n, seed):
    rng = np.random.default_rng(seed)
    s = np.zeros(n, synth.STATE)
    for f in synth.STATE.names:
        s[f] = rng.normal(0, 1, s[f].shape).astype(np.float32)
    return s


def resize_three(hs, port, ref, states, probs, num, with_ref=True):
    got = hs_resize(hs, states, probs, num)
    assert same(got, port.resize(states, probs, num))
    if with_ref:
        assert same(got, ref.resize(states, probs, num))
    return got


def chain(probs, num):
    """numpy restatement of accum / pstep / the pscan chain in float32"""
    a = np.float32(0)
    for p in probs.astype(np.float32):
        a = np.float32(a + p)
    pstep = np.float32(a / np.float32(num))
    c = np.zeros(num, np.float32)
    s = np.float32(0)
    for i in range(num):
        s = np.float32(s + pstep)
        c[i] = s
    return a, c


@pytest.mark.parametrize("n,num", [(5000, 3750), (1000, 2500), (4000, 1), (1, 7), (3000, 3000)])
def test_resize_tie_free(hs, port, ref, n, num):
    rng = np.random.default_rng(n + num)
    probs = rng.uniform(0.1, 1.0, n).astype(np.float32)
    probs /= probs.sum()
    states = random_states(n, n)
    s, p = resize_three(hs, port, ref, states, probs, num)
    assert np.all(p == np.float32(1.0 / num))


def test_resize_end_suffix(hs, port, ref):
    """A pscan chain that overshoots the total: the last outputs copy the last pick that found a particle."""
    rng = np.random.default_rng(11)
    for trial in range(200):
        n = int(rng.integers(50, 400))
        num = int(rng.integers(50, 2000))
        probs = rng.uniform(0.0, 1.0, n).astype(np.float32)
        total, c = chain(probs, num)
        if c[-1] > total:
            break
    else:
        pytest.fail("no overshooting chain found")
    states = random_states(n, 12)
    s, _ = resize_three(hs, port, ref, states, probs, num)
    n_end = int(np.count_nonzero(c > total))
    assert n_end > 0
    last = s[num - n_end - 1] if num > n_end else states[0]
    assert all(s[i].tobytes() == last.tobytes() for i in range(num - n_end, num))


def test_resize_all_zero_total(hs, port, ref):
    """All probabilities 0: pstep = 0, every pscan is 0 and every output copies particle 0.  (n <= 16: std::sort in the
    reference then runs an insertion sort, which keeps the order of the all-equal prefix sums.)"""
    states = random_states(10, 13)
    probs = np.zeros(10, np.float32)
    s, p = resize_three(hs, port, ref, states, probs, 25)
    assert all(x.tobytes() == states[0].tobytes() for x in s)


def test_resize_ties_lowest_index(hs, port, ref):
    """Zero-probability particles tie in accum with the one before them: the pick takes the lowest index.  Against the
    port at any size; against the reference where its std::sort keeps ties in order (n <= 16)."""
    rng = np.random.default_rng(14)
    probs = rng.uniform(0.1, 1.0, 3000).astype(np.float32)
    probs[rng.random(3000) < 0.3] = 0.0
    states = random_states(3000, 15)
    resize_three(hs, port, ref, states, probs, 2000, with_ref=False)
    small = np.array([0.2, 0, 0, 0.1, 0, 0.3, 0, 0, 0, 0.4, 0, 0.1], np.float32)
    s, _ = resize_three(hs, port, ref, random_states(12, 16), small, 9)
