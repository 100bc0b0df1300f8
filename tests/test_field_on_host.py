"""Field mode's per-eval device functions without a GPU: field_dist, lik_term and near_layout of
mcl_3dl_b200/csrc/device_funcs.cuh, compiled verbatim for the host by tests/hostsim/field_hostsim.cpp, equal the numpy
restatement of tests/field_restate.py bit for bit, on random node volumes and at the lookup's edges (nodes, one ulp
either side of them, the last cell, the upper faces, outside the lattice and past int range).  NaN queries are left to
the GPU suite (test_gpu_field_exact.py).  The restatement's lattice rule (ef = 1.01 r / 2, doubled until the field fits;
inv_e = 1 / ef) is held to near_layout itself."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import field_restate as FR
from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "field_hostsim.cpp")
F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fieldhs") / "libfieldhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return load(so)


def load(so):
    L = C.CDLL(so)
    vp, sz, f = C.c_void_p, C.c_size_t, C.c_float
    L.hostsim_field_dist.argtypes = [vp, vp, vp, f, f, vp, sz, vp]
    L.hostsim_field_dist.restype = None
    L.hostsim_field_term.argtypes = [vp, sz, f, f, f, vp, vp]
    L.hostsim_field_term.restype = None
    L.hostsim_field_terms.argtypes = [vp, sz, vp, sz, vp, vp, vp, f, f, vp, f, f, f, vp, vp]
    L.hostsim_field_terms.restype = None
    L.hostsim_near_layout.argtypes = [f, C.c_int, vp, vp, sz, vp, vp, vp]
    L.hostsim_near_layout.restype = C.c_int
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_field_dist(hs, V, org, inv_e, clamp, q):
    cells = FR.expand(V)
    dims = np.array([V.shape[2] - 1, V.shape[1] - 1, V.shape[0] - 1], np.int32)
    q = np.ascontiguousarray(q, F)
    out = np.zeros(len(q), F)
    hs.hostsim_field_dist(_p(cells), _p(dims), _p(np.asarray(org, F)), F(inv_e), F(clamp), _p(q), len(q), _p(out))
    return out


def random_volume(rng, dims, clamp, flat):
    """Distinct random node values in (flat, clamp), with a few exact 0 and clamp values."""
    n = (dims[2] + 1) * (dims[1] + 1) * (dims[0] + 1)
    v = rng.uniform(float(flat), float(clamp), n).astype(F)
    v[rng.choice(n, n // 20, replace=False)] = F(0)
    v[rng.choice(n, n // 20, replace=False)] = F(clamp)
    return v.reshape(dims[2] + 1, dims[1] + 1, dims[0] + 1)


# ------------------------------------------------------------------ the lattice rule
@pytest.mark.parametrize("seed", range(6))
def test_near_layout_restated(hs, seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        lo = rng.uniform(-3000, 3000, 3).astype(F)
        hi = (lo + rng.uniform(0, 40, 3) * rng.choice([1, 1e-3, 10], 3)).astype(F)
        r = F(rng.choice([FR.lik_rpad(0.2), FR.kd_pads()[0], FR.kd_pads()[1], rng.uniform(1e-3, 2)]))
        k = int(rng.choice([1, 2, 3, 15]))
        cap = int(rng.choice([1 << 40, 1 << 20, 1 << 14]))   # small caps force the doubling retries
        dims, org, inv = np.zeros(3, np.int32), np.zeros(3, F), np.zeros(1, F)
        ok = hs.hostsim_near_layout(r, k, _p(lo), _p(hi), cap, _p(dims), _p(org), _p(inv))
        want = FR.near_layout(r, k, lo, hi, cap)
        assert bool(ok) == (want is not None)
        if ok:
            assert tuple(dims) == want[0] and org.tobytes() == want[1].tobytes() and inv[0] == want[2]
            assert F(F(1) / inv[0]) == F(F(1) / want[2])


def test_field_radius_restated():
    """The radii build_map_on_device picks for the default 0.1 m map grid: the KD second search's pad lies above
    match_dist_min, the marching search's below it."""
    r1, r2 = FR.kd_pads()
    assert FR.field_radius(0.2, FR.LIK) == FR.field_radius(0.2, FR.DDA) == FR.lik_rpad(0.2)
    assert FR.field_radius(0.2, FR.KD_R2) == r2 and abs(float(r2) - 0.2707) < 1e-3
    assert FR.field_radius(0.2, FR.KD_R1) == FR.lik_rpad(0.2) and r1 < FR.lik_rpad(0.2)


# ------------------------------------------------------------------ field_dist and lik_term
@pytest.mark.parametrize("seed", range(8))
def test_field_dist_restated(hs, seed):
    rng = np.random.default_rng(100 + seed)
    dims = tuple(int(v) for v in rng.integers(1, 12, 3))
    if seed == 0:
        dims = (1, 1, 1)
    radius = F(rng.choice([FR.lik_rpad(0.2), FR.kd_pads()[1]]))
    lo = rng.uniform(-50, 50, 3).astype(F)
    _, _, inv_e, ef = FR.near_layout(radius, 2, lo, lo + F(1))
    org = (lo - rng.uniform(0, 1, 3)).astype(F)
    edge = F(F(1) / inv_e)
    V = random_volume(rng, dims, radius, 0.05)
    q = FR.edge_queries((dims[0] + 1, dims[1] + 1, dims[2] + 1), org, edge, inv_e, rng, n=30000)
    got = host_field_dist(hs, V, org, inv_e, radius, q)
    want = FR.field_dist(V, org, inv_e, radius, q)
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert len(bad) == 0, (len(bad), q[bad[:3]], got[bad[:3]], want[bad[:3]])
    # the edges are reached on every axis: tx on node 0, both sides of the upper face and of 0, past int range
    t = ((q - org).astype(F) * inv_e).astype(F)
    n = np.array(dims)
    assert (t == 0).any(axis=0).all() and (t > 2.0 ** 31).any(axis=0).all() and (t < -2.0 ** 31).any(axis=0).all()
    assert ((t < n) & (t > n - 1e-3)).any(axis=0).all() and ((t >= n) & (t < n + 1e-3)).any(axis=0).all()
    assert ((t < 0) & (t > -1e-3)).any(axis=0).all()
    inside = ((t >= 0) & (t < n)).all(axis=1)
    assert inside.sum() > 1000 and (~inside).sum() > 1000
    assert (got[~inside] == radius).all()


def test_lik_term_restated(hs):
    R, flat = F(0.2), F(0.05)
    d = [F(0), F(flat), F(R), F(0.27), F(1e30)]
    for v in (flat, R):
        for s in (-1, 1):
            x = v
            for _ in range(4):
                x = np.nextafter(x, F(s * np.inf), dtype=F)
                d.append(x)
    d = np.concatenate([np.array(d, F), np.random.default_rng(7).uniform(0, 0.3, 2000).astype(F)])
    for w in (5.0, -3.0, 0.7, 0.0):
        term, cnt = np.zeros(len(d), F), np.zeros(len(d), np.uint8)
        hs.hostsim_field_term(_p(d), len(d), R, flat, F(w), _p(term), _p(cnt))
        want_t, want_m = FR.field_term(d, R, flat, w)
        assert term.tobytes() == want_t.tobytes() and np.array_equal(cnt.astype(bool), want_m)
        assert want_m.any() and not want_m.all()


@pytest.mark.parametrize("dw", [(1, 1, 1), (1, 1, 5), (0.7, 1.3, 2.9)])
def test_one_eval_per_record(hs, dw):
    """A particle at q with the identity rotation and the one-point scan (0, 0, 0): the transform returns q exactly, so
    its record is the lookup at float(q * dist_weight) - the premise of test_gpu_field_exact.py's lookup test."""
    rng = np.random.default_rng(11)
    dims = (7, 5, 9)
    radius = FR.lik_rpad(0.2)
    org = np.array([-0.3, 0.1, -0.2], F)
    _, _, inv_e, _ = FR.near_layout(radius, 2, org, org + F(1))
    edge = F(F(1) / inv_e)
    V = random_volume(rng, dims, radius, 0.05)
    qs = FR.edge_queries((8, 6, 10), org, edge, inv_e, rng, n=5000)
    pos = (qs / np.asarray(dw, F)).astype(F)
    poses = synth.make_poses(pos, np.tile(np.array([0, 0, 0, 1], F), (len(pos), 1)))
    scan = synth.make_points(np.zeros((1, 3), F))
    cells = FR.expand(V)
    T, M = np.zeros(len(pos), F), np.zeros(len(pos), np.uint8)
    hs.hostsim_field_terms(_p(poses), len(poses), _p(scan), 1, _p(cells), _p(np.array(dims, np.int32)), _p(org),
                           inv_e, radius, _p(np.asarray(dw, F)), F(0.2), F(0.05), F(5.0), _p(T), _p(M))
    q = (pos * np.asarray(dw, F)).astype(F)
    score, cnt = FR.one_eval_records(V, org, inv_e, radius, q, 0.2, 0.05, 5.0)
    assert T.tobytes() == score.tobytes() and np.array_equal(M.astype(np.uint32), cnt)
    assert cnt.any() and not cnt.all()
