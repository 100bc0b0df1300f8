"""The node's matched / unmatched output (src/mcl_3dl.cpp:761-805) without a GPU: the port's restatement of the loop
equals the reference's own loop point for point, hand-built cases pin the two comparisons (the match test squared in
double, d2 == r2 excluded), and the device functions of mcl_3dl_b200/csrc/match_funcs.cuh, compiled for the host by
tests/hostsim/match_hostsim.cpp, equal the port.  The scenes use 1-2 m chunks, so that many queries sit in chunk halos,
where the search radius (0.5) above max_search_radius (0.2) makes chunk visibility decide the class."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import cpu_checker as cc
from oracle import match_checker as mc
from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "match_hostsim.cpp")
MATCHED, UNMATCHED, NEITHER = 1, 2, 0


def match_scene(seed=0, n_map=20_000, n_scan=3000, n_off=200, n_nan=6):
    """A warehouse map, a scan around a pose in it with wide noise (so distances spread across match_dist and
    unmatch_dist), points far off the map and non-finite points; the pose's quaternion is not exactly unit."""
    mp, info = synth.warehouse_map(n_map, seed=seed + 1)
    rng = np.random.default_rng(seed + 10)
    pos = synth.free_space_position(info, rng)
    yaw = rng.uniform(-np.pi, np.pi)
    q = synth.quat_from_rpy(np.array([[0.01, -0.02, yaw]]))[0] * np.float32(1.0007)
    scan = synth.make_scan(mp, pos, q, n_scan, 0.5, 10.0, sigma=0.15, seed=seed + 2)
    # the generator puts every surface next to a multiple of 1 m, i.e. in a chunk halo: move the world off that lattice
    shift = np.array([0.37, 0.61, 0.45])
    for k, a in enumerate("xyz"):
        mp[a] += np.float32(shift[k])
    pos = pos + shift
    off = rng.uniform(-8.0, 8.0, (n_off, 3)).astype(np.float32)
    off[:, 2] = rng.uniform(4.0, 9.0, n_off)  # above the ceiling
    bad = np.zeros((n_nan, 3), np.float32)
    bad[0::3, 0] = np.nan
    bad[1::3, 1] = np.inf
    bad[2::3, 2] = -np.inf
    extra = synth.make_points(np.concatenate([off, bad]), np.arange(n_off + n_nan) % 3)
    pts = np.concatenate([scan, extra])
    pts = pts[rng.permutation(len(pts))]
    pose = cc.poses(pos, q)
    return mp, pose, pts


def transformed(port, pose, pts):
    return np.array([port.transform_point(pose, (p["x"], p["y"], p["z"])) for p in pts], np.float32).reshape(-1, 3)


def global_classes(mp, tf, w, match_dist, unmatch_dist):
    """The same tests against EVERY map point (no chunk rule): float L2_Simple in the rescaled space."""
    m = np.stack([mp["x"] * np.float32(w[0]), mp["y"] * np.float32(w[1]), mp["z"] * np.float32(w[2])], 1).astype(np.float32)
    r = np.float32(unmatch_dist)
    r2 = np.float32(np.float64(r) * np.float64(r))
    out = np.full(len(tf), UNMATCHED, np.uint8)
    for i, t in enumerate(tf):
        if not np.all(np.isfinite(t)):
            continue
        q = (t * np.asarray(w, np.float32)).astype(np.float32)
        d = m - q
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        best = d2[d2 < r2]
        if len(best):
            out[i] = MATCHED if np.float64(best.min()) < match_dist * match_dist else NEITHER
    return out


@pytest.fixture(scope="module")
def mport():
    mc.build("port")
    return mc.MatchChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not mc.build("reference"):
        pytest.skip("reference checker not built (no reference checkout)")
    return mc.MatchChecker("reference")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("matchhs") / "libmatchhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    L.hostsim_match_output.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_double,
                                       C.c_double, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    return L


def hostsim_match(L, mp, weights, pose, pts, match_dist, unmatch_dist, chunk_length, max_r):
    lik = cc.lik_params(dist_weight=weights)
    mp = np.ascontiguousarray(mp, dtype=cc.POINT)
    pose = np.ascontiguousarray(pose, dtype=cc.POSE).reshape(1)
    pts = np.ascontiguousarray(pts, dtype=cc.POINT)
    cls = np.zeros(len(pts), np.uint8)
    tf = np.zeros(len(pts), cc.POINT)
    L.hostsim_match_output(cc._ptr(mp), len(mp), C.byref(lik), cc._ptr(pose), cc._ptr(pts), len(pts), match_dist,
                           unmatch_dist, chunk_length, max_r, cc._ptr(cls), cc._ptr(tf))
    return cls, tf


SCENES = [(1.0, (1, 1, 1), 0), (1.5, (1, 1, 1), 1), (2.0, (1, 1, 5), 2), (1.0, (1, 1, 5), 3)]


@pytest.mark.parametrize("chunk_length,weights,seed", SCENES)
def test_port_equals_reference_per_point(mport, ref, chunk_length, weights, seed):
    mp, pose, pts = match_scene(seed)
    lik = cc.lik_params(dist_weight=weights)
    a = mport.create(mp, lik, chunk_length, 0.2).match_output(pose, pts, 0.1, 0.5)
    b = ref.create(mp, lik, chunk_length, 0.2).match_output(pose, pts, 0.1, 0.5)
    assert np.array_equal(a, b), np.flatnonzero(a != b)[:20]
    counts = np.bincount(a, minlength=3)
    assert counts.min() > 0, counts


@pytest.mark.parametrize("chunk_length,weights,seed", SCENES)
def test_hostsim_equals_port_and_chunks_matter(port, mport, hs, chunk_length, weights, seed):
    mp, pose, pts = match_scene(seed)
    want = mport.create(mp, cc.lik_params(dist_weight=weights), chunk_length, 0.2).match_output(pose, pts, 0.1, 0.5)
    got, tf = hostsim_match(hs, mp, weights, pose, pts, 0.1, 0.5, chunk_length, 0.2)
    assert np.array_equal(got, want), np.flatnonzero(got != want)[:20]
    xyz = transformed(port, pose, pts)
    assert np.array_equal(np.stack([tf["x"], tf["y"], tf["z"]], 1).view(np.uint32), xyz.view(np.uint32))
    assert np.array_equal(tf["label"], pts["label"])
    non_finite = ~np.all(np.isfinite(xyz), axis=1)
    assert non_finite.sum() == 6 and np.all(got[non_finite] == UNMATCHED)
    # chunk visibility must decide some classes here, or the chunk rule would be untested
    glob = global_classes(mp, xyz, weights, 0.1, 0.5)
    assert np.count_nonzero(glob != want) > 0


def _query_with_d2(pred):
    """(qx, qy) near (0.6, 0.5) whose float L2_Simple distance^2 d2 to (0.5, 0.5, 0.5) satisfies pred(d2)."""
    m0 = np.float32(0.5)
    qx = np.float32(0.6) + np.arange(-300, 300, dtype=np.float32) * np.float32(2 ** -24)
    qy = m0 + np.linspace(0.0, 1e-4, 400, dtype=np.float32)
    dx = (qx - m0).astype(np.float32)[:, None]
    dy = (qy - m0).astype(np.float32)[None, :]
    d2 = ((dx * dx).astype(np.float32) + (dy * dy).astype(np.float32)).astype(np.float32)
    i, j = np.argwhere(pred(d2))[0]
    return qx[i], qy[j], d2[i, j]


def test_hand_built_comparisons(mport, ref, hs):
    """One map point at (0.5, 0.5, 0.5), chunk 20 (no halo involved), identity pose (the transform is exact): queries
    whose float d2 is the last float below the double 0.1^2 and the first one above it, and queries on r2 = 0.25 itself
    and one float inside it."""
    mp = cc.points([[0.5, 0.5, 0.5]])
    match_sq = 0.1 * 0.1  # 0.010000000000000002 in double
    lo = np.float32(match_sq)
    lo = lo if np.float64(lo) < match_sq else np.nextafter(lo, np.float32(0))
    hi = np.nextafter(lo, np.float32(1))
    bx, by, b = _query_with_d2(lambda d: d == lo)
    ax, ay, a = _query_with_d2(lambda d: d == hi)
    assert np.float64(b) < match_sq <= np.float64(a)
    # compared with float(0.1^2) (== b) the first query would be rejected: the double rule is what is pinned here
    assert not (b < np.float32(match_sq))
    edge = np.float32(1.0)  # dx = 0.5: d2 == r2 == 0.25, excluded
    inside = np.nextafter(edge, np.float32(0))
    pts = cc.points([[bx, by, 0.5], [ax, ay, 0.5], [edge, 0.5, 0.5], [inside, 0.5, 0.5]])
    pose = cc.poses([0, 0, 0], [0, 0, 0, 1])
    want = np.array([MATCHED, NEITHER, UNMATCHED, NEITHER], np.uint8)
    for chk in (mport, ref):
        assert np.array_equal(chk.create(mp, cc.lik_params(), 20.0, 0.2).match_output(pose, pts, 0.1, 0.5), want)
    got, _ = hostsim_match(hs, mp, (1, 1, 1), pose, pts, 0.1, 0.5, 20.0, 0.2)
    assert np.array_equal(got, want)


def test_radius_above_chunk_length_is_rejected(mport, ref):
    mp = cc.points([[0.5, 0.5, 0.5]])
    pts = cc.points([[0.5, 0.5, 0.5]])
    pose = cc.poses([0, 0, 0], [0, 0, 0, 1])
    for chk in (mport, ref):
        m = chk.create(mp, cc.lik_params(), 1.0, 0.2)
        assert np.array_equal(m.match_output(pose, pts, 0.1, 1.0), [MATCHED])  # radius == chunk length is allowed
        with pytest.raises(RuntimeError):
            m.match_output(pose, pts, 0.1, 1.5)
