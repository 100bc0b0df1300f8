"""Scan preparation (mcl3dl_scan_prepare) bit for bit against plain restatements, at the edges where it goes wrong.

* VoxelGrid: a numpy restatement of pcl::VoxelGrid::applyFilter in float32 (voxel_grid_ref): non-finite points skipped
  in the bounding box and in the voxel pass, PCL's overflow rule with PCL's own per-axis count
  dx = int64((max - min) * inv) + 1 (more than INT32_MAX voxels: the cloud passes unfiltered), leaf index
  floor(coord * inv) - min_b with x fastest, output in ascending voxel index, centroid = float sums in input order over
  float(cnt), majority label with the lowest label winning ties.  The device's downsampled cloud must equal it byte for
  byte.
* Clip: the keep mask of both models' windows is the oracle's filter_clip (the reference's code), order kept.
* Sampler: a numpy Philox-4x32-10 (checked against the Random123 known answers) drawing from counter
  (t, stream, 0x5ca11ab1, 0), key = the 64-bit seed's low and high words, index (c0 * n) >> 32.

The CPU tests run the same restatements against the device's own per-point functions (scan_funcs.cuh, built for the
host by tests/hostsim/scan_hostsim.cpp), so a GPU failure can only come from the kernels or their plumbing.
"""
import ctypes as C
import os
import subprocess
import time

import numpy as np
import pytest

from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "scan_hostsim.cpp")
POINT = synth.POINT
INT32_MAX = 2 ** 31 - 1
NODE_LEAF = (0.1, 0.1, 0.05)  # the node's downsample_x/y/z defaults
WIDE = (0.0, 1e6, -1e6, 1e6)  # a clip window that keeps every finite point


# ---------------------------------------------------------------- restatements
def philox4x32_10(ctr, key):
    """Philox-4x32-10 (Salmon et al., SC'11) on arrays: ctr = four uint32 arrays, key = (k0, k1)."""
    mask = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = (np.asarray(x, np.uint64) & mask for x in ctr)
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & mask
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & mask, (k1 + np.uint64(0xBB67AE85)) & mask
    return [x.astype(np.uint32) for x in (c0, c1, c2, c3)]


def sample_ref(seed, stream, num, n):
    """Indices of draws 0..num-1 over n clipped points."""
    t = np.arange(num, dtype=np.uint64)
    c0 = philox4x32_10((t, np.full_like(t, stream), np.full_like(t, 0x5CA11AB1), np.zeros_like(t)),
                       (seed & 0xFFFFFFFF, seed >> 32))[0]
    return ((c0.astype(np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64)


def _sequential_sums(v, starts, cnt):
    """Float32 sums of v[starts[g] : starts[g] + cnt[g]], each added from 0 in order."""
    out = np.zeros((len(starts), 3), np.float32)
    big = cnt > 4096
    for g in np.flatnonzero(big):  # add.accumulate is a sequential loop
        seg = np.concatenate([np.zeros((1, 3), np.float32), v[starts[g]:starts[g] + cnt[g]]])
        out[g] = np.add.accumulate(seg, axis=0, dtype=np.float32)[-1]
    small = np.flatnonzero(~big)
    small = small[np.argsort(-cnt[small], kind="stable")]  # the groups still open at rank r are a prefix
    c, st = cnt[small], starts[small]
    acc = np.zeros((len(small), 3), np.float32)
    for r in range(int(c.max()) if len(c) else 0):
        m = np.searchsorted(-c, -r, side="left")
        acc[:m] += v[st[:m] + r]
    out[small] = acc
    return out


def _majority(keys, lab):
    """Per key (keys ascending): the most frequent label, the lowest one on ties."""
    o = np.lexsort((lab, keys))
    k, l = keys[o], lab[o]
    hs = np.flatnonzero(np.concatenate([[True], (k[1:] != k[:-1]) | (l[1:] != l[:-1])]))
    rc = np.diff(np.concatenate([hs, [len(k)]]))
    rk, rl = k[hs], l[hs]
    o2 = np.lexsort((rl, -rc, rk))
    rk2 = rk[o2]
    return rl[o2][np.concatenate([[True], rk2[1:] != rk2[:-1]])]


def lattice_ref(leaf, mn, mx):
    """PCL's overflow rule and lattice: None (unfiltered) or (inv, min_b, div_b).  Beyond PCL's rule, the cloud also
    passes unfiltered where PCL's own int arithmetic would overflow (min_b / max_b past int, div_b's product past 32
    bits): the device's keys are exact only below that."""
    with np.errstate(all="ignore"):
        inv = (np.float32(1) / np.asarray(leaf, np.float32)).astype(np.float32)
        mn, mx = np.asarray(mn, np.float32), np.asarray(mx, np.float32)
        ext = (mx - mn) * inv
        if not (ext < np.float32(2.0 ** 31)).all():
            return None
        d = [int(v) + 1 for v in ext]
        if d[0] * d[1] * d[2] > INT32_MAX:
            return None
        lo, hi = np.floor(mn * inv), np.floor(mx * inv)
    if not ((lo >= -2.0 ** 31).all() and (hi < 2.0 ** 31).all()):
        return None
    min_b = lo.astype(np.int64)
    div = hi.astype(np.int64) - min_b + 1
    if int(div[0]) * int(div[1]) * int(div[2]) > 0xFFFFFFFF:
        return None
    return inv, min_b, div


def voxel_grid_ref(pts, leaf):
    """pcl::VoxelGrid::applyFilter on a cloud that is not dense, float32 throughout.  None: the cloud passes unfiltered."""
    xyz = np.stack([pts["x"], pts["y"], pts["z"]], axis=1).astype(np.float32)
    fin = np.isfinite(xyz).all(axis=1)
    if not fin.any():
        return pts[:0].copy()
    xyz, lab = xyz[fin], pts["label"][fin]
    lat = lattice_ref(leaf, xyz.min(axis=0), xyz.max(axis=0))
    if lat is None:
        return None
    inv, min_b, div = lat
    ijk = np.floor(xyz * inv).astype(np.int64) - min_b
    key = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * (div[0] * div[1])
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.concatenate([[True], ks[1:] != ks[:-1]]))
    cnt = np.diff(np.concatenate([starts, [len(ks)]]))
    cen = _sequential_sums(xyz[order], starts, cnt) / cnt.astype(np.float32)[:, None]
    out = np.zeros(len(starts), POINT)
    out["x"], out["y"], out["z"] = cen[:, 0], cen[:, 1], cen[:, 2]
    out["label"] = _majority(ks, lab[order])
    return out


# ---------------------------------------------------------------- clouds
def _pts(xyz, label=None):
    return synth.make_points(np.asarray(xyz, np.float32), label)


def _on_planes(leaf, seed, n=6000):
    """Coordinates float(k) / inv (on a lattice plane, or as close as floats get) and their nextafter neighbours."""
    rng = np.random.default_rng(seed)
    inv = (np.float32(1) / np.float32(leaf)).astype(np.float32)
    base = (np.arange(-12, 13).astype(np.float32) / inv).astype(np.float32)
    vals = np.concatenate([base, np.nextafter(base, np.float32(-np.inf)), np.nextafter(base, np.float32(np.inf))])
    return _pts(rng.choice(vals, (n, 3)), rng.integers(0, 3, n)), (leaf, leaf, leaf)


def _accumulated(n, seed, centre=(0.0, 0.0, 0.0)):
    """An accumulated cloud: floor, walls and clutter around the sensor, labels 0..3."""
    rng = np.random.default_rng(seed)
    m = n // 8
    floor = rng.uniform([-25, -25, -0.02], [25, 25, 0.02], (m * 3, 3))
    walls = np.concatenate([rng.uniform([-25, 20, 0], [25, 20.05, 3], (m, 3)), rng.uniform([-25, -20.05, 0], [25, -20, 3], (m, 3)),
                            rng.uniform([18, -20, 0], [18.05, 20, 3], (m, 3))])
    clutter = rng.uniform([-20, -18, 0], [16, 18, 2], (n - 6 * m, 3))
    xyz = np.concatenate([floor, walls, clutter]) + np.asarray(centre)
    xyz = xyz[rng.permutation(len(xyz))]
    return _pts(xyz, rng.integers(0, 4, len(xyz)))


def _limit_cloud(dy):
    """Leaf 1: dx = 65536, dz = 1 and dy as given, so PCL's count is 65536 * dy."""
    xyz = [(0.0, 0.0, 0.0), (65535.5, dy - 0.5, 0.5), (100.25, 7.5, 0.25), (100.75, 7.25, 0.75), (3.5, 2.5, 0.5)]
    return _pts(xyz, [1, 2, 3, 3, 4]), (1.0, 1.0, 1.0)


def _with_nonfinite(pts, seed, frac=0.05):
    rng = np.random.default_rng(seed)
    pts = pts.copy()
    bad = rng.random(len(pts)) < frac
    f = np.array(["x", "y", "z"])[rng.integers(0, 3, len(pts))]
    vals = rng.choice(np.array([np.nan, np.inf, -np.inf], np.float32), len(pts))
    for i in np.flatnonzero(bad):
        pts[f[i]][i] = vals[i]
    pts[0]["x"], pts[1]["y"], pts[2]["z"] = np.nan, np.inf, -np.inf  # each kind at least once
    return pts


def case(name):
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "straddle_zero":
        return _pts(rng.uniform(-3, 3, (20000, 3)), rng.integers(0, 4, 20000)), (0.1, 0.1, 0.1)
    if name == "planes_0.1":
        return _on_planes(0.1, 1)
    if name == "planes_0.125":
        return _on_planes(0.125, 2)
    if name == "node_leaf":
        return _pts(rng.uniform([-8, -8, -1], [8, 8, 2], (30000, 3)), rng.integers(0, 5, 30000)), NODE_LEAF
    if name == "skewed_leaf":
        return _pts(rng.uniform([-5, -7, -2], [6, 4, 3], (20000, 3)), rng.integers(0, 5, 20000)), (0.2, 0.1, 0.3)
    if name == "single_point":
        return _pts([(1.25, -3.5, 0.75)], [7]), (0.1, 0.1, 0.1)
    if name == "one_voxel":
        return _pts(rng.uniform(0.01, 0.09, (5000, 3)), rng.integers(0, 3, 5000)), (0.1, 0.1, 0.1)
    if name == "duplicates":
        base = rng.uniform(-1, 1, (300, 3)).astype(np.float32)
        return _pts(np.tile(base, (7, 1)), rng.integers(0, 3, 2100)), (0.1, 0.1, 0.1)
    if name == "own_voxels":
        g = np.stack(np.meshgrid(np.arange(-10, 10), np.arange(-8, 8), np.arange(-3, 3), indexing="ij"), -1).reshape(-1, 3)
        xyz = ((g + 0.5) * 0.25).astype(np.float32)
        return _pts(xyz[rng.permutation(len(xyz))], rng.integers(0, 2 ** 32, len(xyz), dtype=np.uint64)), (0.25, 0.25, 0.25)
    if name == "label_ties":
        # voxels of 2, 4 and 6 points split evenly between two or three labels, the extremes of uint32 included
        labs = np.array([0, 1, 5, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF], np.uint64)
        xyz, lab = [], []
        for v in range(400):
            k = int(rng.integers(1, 4))
            ls = rng.choice(labs, k, replace=False)
            per = int(rng.integers(1, 4))
            cen = np.array([v % 20, (v // 20) % 20, 0], np.float32) * 0.1 + 0.05
            for l in ls:
                xyz += [cen + rng.uniform(-0.04, 0.04, 3) for _ in range(per)]
                lab += [l] * per
        o = rng.permutation(len(xyz))
        return _pts(np.array(xyz)[o], np.array(lab, np.uint64)[o]), (0.1, 0.1, 0.1)
    if name == "key_bits_31":  # 2^30 < cells < 2^31
        xyz = [(0.0, 0.0, 0.0), (0.5, 0.5, 1.5e9), (0.25, 0.25, 300.5), (0.5, 0.0, 5.0e8), (0.0, 0.5, 7.0e8), (0.1, 0.1, 7.0e8)]
        return _pts(xyz, [1, 2, 3, 4, 5, 6]), (1.0, 1.0, 1.0)
    if name == "key_bits_32":  # PCL's count 2^29 + 1, div_b's product 2^31 + 4
        xyz = [(0.9, 0.9, 0.0), (1.1, 1.1, 2.0 ** 29), (1.05, 0.95, 2.0 ** 29), (0.95, 1.05, 3.0), (1.0, 1.0, 2.0 ** 28)]
        return _pts(xyz, [1, 2, 3, 4, 5]), (1.0, 1.0, 1.0)
    if name == "below_limit":
        return _limit_cloud(32767)
    if name == "above_limit":
        return _limit_cloud(32769)
    if name == "issue_200m":  # 200 m x 200 m x 27 m at the node's leaves: 2.17e9 voxels by PCL's count
        xyz = np.concatenate([[(-100, -100, -2), (100, 100, 25)], rng.uniform([-100, -100, -2], [100, 100, 25], (5000, 3))])
        return _pts(xyz, rng.integers(0, 3, len(xyz))), NODE_LEAF
    if name == "far_1km":
        return _accumulated(60000, 3, centre=(1000.0, -700.0, 20.0)), NODE_LEAF
    if name == "accumulated_1.3M":
        return _accumulated(1_300_000, 4), NODE_LEAF
    if name == "nonfinite":
        return _with_nonfinite(_accumulated(40000, 5), 6), NODE_LEAF
    if name == "nonfinite_small":
        return _with_nonfinite(_pts(rng.uniform(-2, 2, (2000, 3)), rng.integers(0, 3, 2000)), 10), (0.1, 0.1, 0.1)
    if name == "all_nonfinite":
        return _pts(np.full((20, 3), np.nan), np.arange(20)), NODE_LEAF
    if name == "dense_voxel":  # a sensor's (0, 0, 0) "no return" points: one voxel of 131 072 points, mixed-label tail
        n = 1 << 17
        xyz = np.zeros((n, 3), np.float32)
        tail = rng.random(n) < 0.3
        xyz[tail] = rng.uniform(0.0, 0.05, (int(tail.sum()), 3))
        lab = np.where(tail, rng.integers(0, 6, n), 3)
        cloud = np.concatenate([_pts(xyz, lab), _accumulated(20000, 7)])
        return cloud, NODE_LEAF
    raise KeyError(name)


VOXEL_CASES = ["straddle_zero", "planes_0.1", "planes_0.125", "node_leaf", "skewed_leaf", "single_point", "one_voxel",
               "duplicates", "own_voxels", "label_ties", "key_bits_31", "key_bits_32", "below_limit", "above_limit",
               "issue_200m", "far_1km", "accumulated_1.3M", "nonfinite", "nonfinite_small", "all_nonfinite", "dense_voxel"]
UNFILTERED = {"above_limit", "issue_200m"}
_CACHE = {}


def case_ref(name):
    """(raw, leaf, restated downsampled cloud or None), computed once per session."""
    if name not in _CACHE:
        raw, leaf = case(name)
        _CACHE[name] = (raw, leaf, voxel_grid_ref(raw, leaf))
    return _CACHE[name]


def test_cases_reach_their_edges():
    """The clouds are what their names say (checked on the restatement itself)."""
    for name in ("below_limit", "key_bits_31", "key_bits_32"):
        raw, leaf = case(name)
        xyz = np.stack([raw["x"], raw["y"], raw["z"]], 1)
        inv, _, div = lattice_ref(leaf, xyz.min(0), xyz.max(0))
        cells = int(np.prod(div))
        bits = {"below_limit": None, "key_bits_31": 31, "key_bits_32": 32}[name]
        if bits:
            assert 2 ** (bits - 1) <= cells < 2 ** bits  # the non-finite key == cells needs exactly `bits` bits
        else:
            assert cells > 2 ** 31 - 2 ** 17
    for name in UNFILTERED:
        assert case_ref(name)[2] is None
    raw, leaf, ds = case_ref("planes_0.1")
    x = raw["x"] * np.float32(1 / np.float32(0.1))
    assert (x == np.floor(x)).mean() > 0.3  # a good share of the coordinates land exactly on a plane
    raw, leaf, ds = case_ref("label_ties")
    assert len(ds) == 400
    raw, leaf, ds = case_ref("dense_voxel")
    assert ds is not None and len(ds) > 1


# ---------------------------------------------------------------- host build of the device functions
@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("scanhs") / "libscanhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_scan_lattice.argtypes = [vp] * 8
    L.hostsim_scan_lattice.restype = C.c_int
    L.hostsim_scan_voxel_grid.argtypes = [vp, sz, vp, vp]
    L.hostsim_scan_voxel_grid.restype = C.c_long
    L.hostsim_scan_voxel_point.argtypes = [vp, vp, vp, C.c_uint32, vp]
    L.hostsim_scan_clip.argtypes = [vp, sz, C.c_float, C.c_float, C.c_float, C.c_float, vp]
    L.hostsim_scan_sample.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_voxel_grid(L, raw, leaf):
    out = np.zeros(max(len(raw), 1), POINT)
    m = L.hostsim_scan_voxel_grid(_p(raw), len(raw), _p(np.asarray(leaf, np.float32)), _p(out))
    return None if m < 0 else out[:m]


def test_philox_known_answers():
    """The numpy Philox-4x32-10 against the Random123 known-answer vectors."""
    for ctr, key, want in [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
                           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
                           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
                            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]:
        got = philox4x32_10([np.array([v], np.uint32) for v in ctr], key)
        assert tuple(int(v[0]) for v in got) == want


@pytest.mark.parametrize("seed,stream,num,n", [(1, 0, 1000, 997), (1, 1, 1000, 997), (0xDEADBEEF12345678, 0, 5000, 3),
                                               (7, 1, 257, 1 << 20), (2 ** 64 - 1, 0, 300, 0xFFFFFFFF), (5, 0, 10, 1)])
def test_sample_index_host(hs, seed, stream, num, n):
    got = np.zeros(num, np.uint32)
    hs.hostsim_scan_sample(seed, stream, num, n, _p(got))
    assert np.array_equal(got, sample_ref(seed, stream, num, n))


LATTICES = [  # (leaf, min, max)
    ((1, 1, 1), (0, 0, 0), (65535.5, 32766.5, 0.5)),       # PCL count just below INT32_MAX
    ((1, 1, 1), (0, 0, 0), (65535.5, 32768.5, 0.5)),       # just above it, div_b's product below 2^32
    ((0.1, 0.1, 0.05), (-100, -100, -2), (100, 100, 25)),  # 2.17e9 by PCL's count
    ((0.1, 0.1, 0.05), (-100, -100, -2), (100, 100, 20)),  # 1.77e9: downsampled
    ((1, 1, 1), (0.9, 0.9, 0), (1.1, 1.1, 2.0 ** 29)),     # 32-bit keys
    ((1, 1, 1), (0.9, 0.9, 0), (1.1, 1.1, 2.0 ** 31 - 256)),  # PCL passes, div_b's product past 32 bits
    ((1, 1, 1), (0, 0, 0), (0, 0, 0)),                     # one voxel: a one-bit key space
    ((1e-3, 1e-3, 1e-3), (3e6, 0, 0), (3e6, 0, 0)),        # min_b past int
    ((1e-40, 1, 1), (0, 0, 0), (1, 1, 1)),                 # inv_leaf = inf
    ((0.25, 0.5, 2), (-1e3, 7, -3), (1e3, 8, 3)),
]


@pytest.mark.parametrize("leaf,mn,mx", LATTICES)
def test_lattice_host(hs, leaf, mn, mx):
    """scan_voxel_lattice: PCL's overflow rule, the lattice, and radix bits that hold every key and the non-finite one."""
    leaf, mn, mx = (np.asarray(v, np.float32) for v in (leaf, mn, mx))
    inv, min_b, div = np.zeros(3, np.float32), np.zeros(3, np.int32), np.zeros(3, np.uint32)
    cells, end_bit = np.zeros(1, np.uint32), np.zeros(1, np.int32)
    ok = hs.hostsim_scan_lattice(_p(leaf), _p(mn), _p(mx), _p(inv), _p(min_b), _p(div), _p(cells), _p(end_bit))
    want = lattice_ref(leaf, mn, mx)
    assert ok == (want is not None)
    if want is not None:
        assert inv.tobytes() == want[0].tobytes()
        assert list(min_b) == list(want[1]) and list(div) == list(want[2])
        assert int(cells[0]) == int(np.prod(want[2].astype(object)))
        assert 2 ** (int(end_bit[0]) - 1) <= int(cells[0]) < 2 ** int(end_bit[0])


@pytest.mark.parametrize("name", VOXEL_CASES)
def test_voxel_grid_host(hs, name):
    """The device's voxel key / centroid / vote functions, sorted serially on the host, against the restatement."""
    raw, leaf, want = case_ref(name)
    got = host_voxel_grid(hs, raw, leaf)
    if want is None:
        assert got is None
    else:
        assert got is not None and got.tobytes() == want.tobytes()


def test_dense_voxel_vote_is_linear_host(hs):
    """One voxel of 2^18 points with a mixed-label tail: the vote walks the voxel's (key, label)-sorted run once.  A vote
    that recounts each point's label over the voxel makes 2^36 loads here (about a minute on one CPU core)."""
    n = 1 << 18
    rng = np.random.default_rng(11)
    lab = np.where(rng.random(n) < 0.4, rng.integers(0, 9, n), 4).astype(np.uint32)
    pts = _pts(rng.uniform(0.001, 0.049, (n, 3)), lab)
    order = np.arange(n, dtype=np.uint32)
    key_label = np.sort(lab.astype(np.uint64))  # voxel key 0
    out = np.zeros(1, POINT)
    t0 = time.perf_counter()
    hs.hostsim_scan_voxel_point(_p(pts), _p(order), _p(key_label), n, _p(out))
    dt = time.perf_counter() - t0
    want = voxel_grid_ref(pts, (0.05, 0.05, 0.05))
    assert len(want) == 1 and out.tobytes() == want.tobytes()
    assert dt < 1.0, dt


def test_vote_ties_host(hs):
    """Equal counts go to the lowest label, whatever the order the points came in."""
    pts = _pts(np.zeros((6, 3)), [9, 0xFFFFFFFF, 2, 9, 2, 0xFFFFFFFF])
    order = np.arange(6, dtype=np.uint32)
    out = np.zeros(1, POINT)
    hs.hostsim_scan_voxel_point(_p(pts), _p(order), _p(np.sort(pts["label"].astype(np.uint64))), 6, _p(out))
    assert out["label"][0] == 2
    pts["label"] = [0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFE, 0xFFFFFFFE, 0xFFFFFFFF, 0xFFFFFFFE]
    hs.hostsim_scan_voxel_point(_p(pts), _p(order), _p(np.sort(pts["label"].astype(np.uint64))), 6, _p(out))
    assert out["label"][0] == 0xFFFFFFFE


def clip_cloud(seed=21):
    """Points on and next to r^2 = near^2, r^2 = far^2, z_min and z_max of CLIP_A / CLIP_B, plus a random cloud."""
    rng = np.random.default_rng(seed)
    xyz = []
    for r in (0.5, 10.0, 4.0, 1.5):
        th = rng.uniform(0, 2 * np.pi, 3000)
        x = (np.float32(r) * np.cos(th)).astype(np.float32)
        y = (np.float32(r) * np.sin(th)).astype(np.float32)
        for dx in (x, np.nextafter(x, np.float32(np.inf)), np.nextafter(x, np.float32(-np.inf))):
            xyz.append(np.stack([dx, y, rng.uniform(-1, 1, 3000).astype(np.float32)], 1))
        axis = np.array([[r, 0, 0], [0, -r, 0], [-r, 0, 0]], np.float32)
        xyz.append(axis)
    for z in (-2.0, 2.0, -1.0, 1.5):
        zz = np.float32(z)
        zs = np.array([zz, np.nextafter(zz, np.float32(np.inf)), np.nextafter(zz, np.float32(-np.inf))], np.float32)
        p = rng.uniform(-3, 3, (900, 3)).astype(np.float32)
        p[:, 2] = np.repeat(zs, 300)
        xyz.append(p)
    xyz.append(rng.uniform(-12, 12, (20000, 3)).astype(np.float32))
    xyz = np.concatenate(xyz).astype(np.float32)
    return _pts(xyz[rng.permutation(len(xyz))], rng.integers(0, 3, len(xyz)))


CLIP_A = (0.5, 10.0, -2.0, 2.0)
CLIP_B = (1.5, 4.0, -1.0, 1.5)


def test_clip_cloud_hits_the_boundaries():
    raw = clip_cloud()
    r2 = raw["x"] * raw["x"] + raw["y"] * raw["y"]
    for b in (0.25, 100.0, 16.0, 2.25):
        assert (r2 == np.float32(b)).sum() > 100 and (r2 > np.float32(b)).any() and (r2 < np.float32(b)).any()
    for z in (-2.0, 2.0, -1.0, 1.5):
        assert (raw["z"] == np.float32(z)).sum() >= 300


@pytest.mark.parametrize("window", [CLIP_A, CLIP_B, (0.0, 3.0, -1.0, 1.0), (5.0, 1.0, -2.0, 2.0), (0.0, 10.0, 1.0, -1.0)])
def test_clip_host(hs, port, window):
    raw = np.concatenate([clip_cloud(), _with_nonfinite(clip_cloud(5)[:100], 8, 0.5)])
    keep = np.zeros(len(raw), np.uint8)
    hs.hostsim_scan_clip(_p(raw), len(raw), *window, _p(keep))
    assert np.array_equal(keep.astype(bool), port.filter_clip(raw, *window))


# ---------------------------------------------------------------- on the device
@pytest.fixture(scope="module")
def eng():
    from mcl_3dl_b200 import engine
    engine.load_library()
    e = engine.Engine((0,))
    yield e
    e.close()


def scan_params(leaf=(0.0, 0.0, 0.0), lik_clip=WIDE, beam_clip=WIDE, lik_num=96, beam_num=3, seed=1):
    from mcl_3dl_b200 import engine
    return engine.ScanParams(downsample=leaf, lik_clip=lik_clip, beam_clip=beam_clip, lik_num_points=lik_num,
                             beam_num_points=beam_num, seed=seed)


def check_prepared(e, port, raw, sp, want_ds=None):
    """Every stage of one mcl3dl_scan_prepare against the restatements: downsampled cloud (want_ds, or the raw cloud
    where it passes unfiltered), both clips (the oracle's filter_clip), both samples; and the counts."""
    info = e.scan_prepare(raw, sp)
    ds = raw if want_ds is None else want_ds
    got_ds = e.scan_get(0)
    assert info["n_raw"] == len(raw) and info["n_downsampled"] == len(ds) == len(got_ds)
    assert got_ds.tobytes() == ds.tobytes()
    windows = ((sp.lik_clip_near, sp.lik_clip_far, sp.lik_clip_z_min, sp.lik_clip_z_max),
               (sp.beam_clip_near, sp.beam_clip_far, sp.beam_clip_z_min, sp.beam_clip_z_max))
    for k, (win, num) in enumerate(zip(windows, (sp.lik_num_points, sp.beam_num_points))):
        clipped = ds[port.filter_clip(ds, *win)]
        got = e.scan_get(1 + k)
        assert info[("n_lik_clipped", "n_beam_clipped")[k]] == len(clipped) == len(got)
        assert got.tobytes() == clipped.tobytes()
        want = clipped[sample_ref(sp.seed, k, num, len(clipped))] if len(clipped) else clipped[:0]
        got = e.scan_get(3 + k)
        assert info[("n_lik", "n_beam")[k]] == len(want) == len(got)
        assert got.tobytes() == want.tobytes()
    return info


@pytest.mark.gpu
@pytest.mark.parametrize("name", VOXEL_CASES)
def test_voxel_grid_device(eng, port, name):
    raw, leaf, want = case_ref(name)
    sp = scan_params(leaf, lik_clip=(0.5, 10.0, -2.0, 2.0), beam_clip=(0.5, 4.0, -2.0, 2.0), lik_num=200, beam_num=17, seed=3)
    info = check_prepared(eng, port, raw, sp, want)
    if want is None:
        assert info["n_downsampled"] == info["n_raw"]


@pytest.mark.gpu
def test_nonfinite_without_downsampling(eng, port):
    """No VoxelGrid: NaN / Inf points reach the clip unchanged and the oracle's filter() decides (NaN passes it)."""
    raw = _with_nonfinite(clip_cloud(), 9, 0.02)
    info = check_prepared(eng, port, raw, scan_params(lik_clip=CLIP_A, beam_clip=CLIP_B, lik_num=500, beam_num=50))
    assert np.isnan(eng.scan_get(1)["x"]).any()
    assert info["n_lik_clipped"] < len(raw)


@pytest.mark.gpu
@pytest.mark.parametrize("lik,beam", [(CLIP_A, CLIP_B), ((0.0, 3.0, -1.0, 1.0), CLIP_A), ((5.0, 1.0, -2.0, 2.0), CLIP_B),
                                      (CLIP_B, (0.0, 10.0, 1.0, -1.0))])
def test_clip_device(eng, port, lik, beam):
    """Both windows at once, points on every boundary; near = 0; windows that remove everything."""
    raw = clip_cloud()
    info = check_prepared(eng, port, raw, scan_params(lik_clip=lik, beam_clip=beam, lik_num=300, beam_num=30))
    empty = lik[0] > lik[1] or lik[2] > lik[3], beam[0] > beam[1] or beam[2] > beam[3]
    assert (info["n_lik_clipped"] == 0) == empty[0] and (info["n_beam_clipped"] == 0) == empty[1]
    assert (info["n_lik"] == 0) == empty[0] and (info["n_beam"] == 0) == empty[1]


@pytest.mark.gpu
@pytest.mark.parametrize("n_clip", [1, 2, 3, 997, 1 << 20])
def test_sample_device(eng, port, n_clip):
    """Bit-exact draws for several sample sizes; a seed with its high word set; the two streams differ."""
    rng = np.random.default_rng(n_clip)
    raw = _pts(rng.uniform(-5, 5, (n_clip, 3)), rng.integers(0, 2 ** 32, n_clip, dtype=np.uint64))
    for num in (1, 255, 256, 257, 70000):
        for seed in (12345, 0xDEADBEEF00C0FFEE):
            info = check_prepared(eng, port, raw, scan_params(lik_num=num, beam_num=num, seed=seed))
            assert info["n_lik_clipped"] == n_clip
            if n_clip > 1 and num > 1:
                assert eng.scan_get(3).tobytes() != eng.scan_get(4).tobytes()


@pytest.mark.gpu
def test_sample_is_uniform(eng):
    """One fixed chi-square test: 10^6 draws over 997 points."""
    from scipy import stats
    n, num = 997, 1_000_000
    raw = _pts(np.zeros((n, 3)) + 1.0, np.arange(n))
    info = eng.scan_prepare(raw, scan_params(lik_num=num, beam_num=0, seed=77))
    assert info["n_lik"] == num
    got = eng.scan_get(3)["label"]
    assert np.array_equal(got, sample_ref(77, 0, num, n))
    counts = np.bincount(got, minlength=n)
    chi2 = float(((counts - num / n) ** 2 / (num / n)).sum())
    assert stats.chi2.sf(chi2, n - 1) > 1e-3, chi2


@pytest.mark.gpu
def test_reprepare(eng, port):
    """Large, small, empty, large again: every stage right each time, nothing stale from the call before."""
    big1 = _with_nonfinite(_accumulated(300_000, 31), 32, 0.01)
    small = _accumulated(500, 33)
    big2 = _accumulated(250_000, 34, centre=(3.0, -2.0, 0.0))
    clips = dict(lik_clip=(0.5, 10.0, -2.0, 2.0), beam_clip=(0.5, 4.0, -2.0, 2.0))
    for raw, leaf, seed in ((big1, NODE_LEAF, 1), (small, NODE_LEAF, 2), (small[:0], NODE_LEAF, 3), (big2, NODE_LEAF, 4),
                            (small, (0, 0, 0), 5), (big1, (0.2, 0.1, 0.3), 6)):
        sp = scan_params(leaf, lik_num=400, beam_num=20, seed=seed, **clips)
        want = voxel_grid_ref(raw, leaf) if all(v > 0 for v in leaf) else None
        info = check_prepared(eng, port, raw, sp, want)
        if len(raw) == 0:
            assert info == {"n_raw": 0, "n_downsampled": 0, "n_lik_clipped": 0, "n_beam_clipped": 0, "n_lik": 0, "n_beam": 0}


@pytest.mark.gpu
def test_prepared_update_after_nonfinite_and_dense_voxel(eng):
    """mcl3dl_particles_measure_update_prepared == mcl3dl_particles_measure_update fed with the scans read back, after a
    raw cloud with NaN / Inf points and one voxel of 100 000 points."""
    from mcl_3dl_b200 import engine
    s = synth.scene(60_000, 500, 64, 8, seed=172)
    e = engine.Engine((0,))
    e.set_map(s["map"], engine.LikParams(dist_weight=(1, 1, 5)), engine.beam_params_from_reference(num_points_default=8))
    rng = np.random.default_rng(6)
    base = np.concatenate([s["lik"], s["beam"]])
    raw = np.tile(base, 40)
    for f in ("x", "y", "z"):
        raw[f] += rng.normal(0, 0.03, len(raw)).astype(np.float32)
    dense = _pts(np.tile(np.float32([[1.01, 0.51, 0.02]]), (100_000, 1)) + rng.uniform(0, 0.02, (100_000, 3)).astype(np.float32),
                 rng.integers(0, 3, 100_000))
    raw = _with_nonfinite(np.concatenate([raw, dense])[rng.permutation(len(raw) + 100_000)], 7, 0.01)
    st = np.zeros(500, dtype=synth.STATE)
    st["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], axis=1)
    st["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], axis=1)
    prior = np.full(500, 1.0 / 500, np.float32)
    sp = engine.ScanParams(lik_num_points=96, beam_num_points=6, seed=9)
    info = e.scan_prepare(raw, sp)
    ds = e.scan_get(0)
    assert ds.tobytes() == voxel_grid_ref(raw, tuple(sp.downsample)).tobytes()
    assert info["n_lik"] == 96 and info["n_beam"] == 6
    for k in (3, 4):
        g = e.scan_get(k)
        assert np.isfinite(np.stack([g["x"], g["y"], g["z"]])).all()
    e.particles_set(st, prior)
    a = e.particles_measure_update_prepared(s["origins"], 0.0)
    _, post_a = e.particles_get()
    e.particles_set(st, prior)
    b = e.particles_measure_update(e.scan_get(3), e.scan_get(4), s["origins"], 0.0)
    _, post_b = e.particles_get()
    assert a == b and np.array_equal(post_a, post_b)
    e.close()
