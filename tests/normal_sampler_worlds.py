"""Shared pieces of the normal-weighted sampler's tests (tests/test_normal_sampler_on_host.py, on the host, and
tests/test_gpu_normal_sampler.py, on the device): the test worlds, the host build of the ns_* functions of
mcl_3dl_b200/csrc/scan_funcs.cuh (tests/hostsim/normal_sampler_hostsim.cpp), a numpy restatement of the draw rule
(include/mcl3dl_b200.h: mcl3dl_scan_sample_with_normal, step 5) and the eigengap of each point's covariance."""
import ctypes as C
import os
import subprocess

import numpy as np
from scipy.spatial import cKDTree

from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "normal_sampler_hostsim.cpp")
F = np.float32
ROUND0, ROUND_MAX = 2048, 1 << 22  # the engine's round schedule (engine.cu: ns_sample_model)


def load_hostsim(out_dir):
    so = os.path.join(str(out_dir), "libnshs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_ns_consts.argtypes = [vp, vp, vp, vp]
    L.hostsim_ns_consts.restype = None
    L.hostsim_ns_lattice.argtypes = [C.c_double, vp, vp, vp, vp, vp, vp, vp]
    L.hostsim_ns_normals.argtypes = [vp, sz, C.c_double, vp, C.c_double, C.c_double, vp, vp, vp]
    L.hostsim_ns_weights.argtypes = [vp, sz, vp, C.c_double, vp]
    L.hostsim_ns_weights.restype = None
    L.hostsim_ns_acos.argtypes = [vp, sz, vp]
    L.hostsim_ns_acos.restype = None
    L.hostsim_ns_draws.argtypes = [vp, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint32, vp]
    L.hostsim_ns_draws.restype = None
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_normals(hs, pts, r, fpc, max_weight, shift):
    """-> (rc, normals float32[n, 3], counts uint32[n], q uint64[n]) of the host build."""
    pts = np.ascontiguousarray(pts, synth.POINT)
    n = len(pts)
    nrm, cnt, q = np.zeros((max(n, 1), 3), F), np.zeros(max(n, 1), np.uint32), np.zeros(max(n, 1), np.uint64)
    src = pts if n else np.zeros(1, synth.POINT)
    rc = hs.hostsim_ns_normals(_p(src), n, r, _p(np.ascontiguousarray(fpc, F)), max_weight, float(np.ldexp(1.0, shift)),
                               _p(nrm), _p(cnt), _p(q))
    return rc, nrm[:n], cnt[:n], q[:n]


def host_draws(hs, cum, seed, stream, t0, cnt):
    idx = np.zeros(cnt, np.uint32)
    hs.hostsim_ns_draws(_p(cum), len(cum), seed, stream, t0, cnt, _p(idx))
    return idx


def restate_sample(hs, q, num, seed, stream):
    """Step 5 over the fixed-point weights q: -> (indices in output order, rounds, draws)."""
    n = len(q)
    if n == 0 or num == 0:
        return np.zeros(0, np.int64), 0, 0
    if n <= num:
        return np.arange(n), 0, 0
    cum = np.ascontiguousarray(np.cumsum(q.astype(np.uint64), dtype=np.uint64))
    seen = np.zeros(n, bool)
    out, d0, rounds = [], 0, 0
    r0 = max(ROUND0, 2 * num)
    while len(out) < num:
        cnt = min(r0 << min(rounds, 16), ROUND_MAX)
        idx = host_draws(hs, cum, seed, stream, d0, cnt)
        # first occurrences, in draw order
        _, first = np.unique(idx, return_index=True)
        for k in np.sort(first):
            i = idx[k]
            if not seen[i]:
                seen[i] = True
                out.append(int(i))
        d0 += cnt
        rounds += 1
    return np.array(out[:num]), rounds, d0


def consts(hs, prm):
    """ns_host_consts of an engine.NormalSamplerParams -> (max_weight, fpc_local float32[3], F)."""
    mw, fpc, sh = C.c_double(0), np.zeros(3, F), C.c_int(0)
    hs.hostsim_ns_consts(C.byref(prm), C.byref(mw), _p(fpc), C.byref(sh))
    return mw.value, fpc, sh.value


def eigengap(pts, r):
    """(lambda1 - lambda0) / lambda2 of each finite point's neighbour covariance (float L2_Simple d2 < float(r * r)),
    in float64; NaN where there are fewer than 3 neighbours or the point is not finite."""
    xyz = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(F)
    fin = np.isfinite(xyz).all(1)
    gap = np.full(len(pts), np.nan)
    if not fin.any():
        return gap
    idx_f = np.nonzero(fin)[0]
    tree = cKDTree(xyz[fin].astype(np.float64))
    r2 = F(r * r)
    for i in idx_f:
        cand = idx_f[tree.query_ball_point(xyz[i].astype(np.float64), r * 1.001)]
        d = xyz[i] - xyz[cand]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        nb = xyz[cand[d2 < r2]].astype(np.float64) - xyz[i].astype(np.float64)
        if len(nb) < 3:
            continue
        m = nb.mean(0)
        w = np.linalg.eigvalsh(nb.T @ nb / len(nb) - np.outer(m, m))
        gap[i] = (w[1] - w[0]) / w[2] if w[2] > 0 else 0.0
    return gap


def _pts(xyz, label=0):
    p = np.zeros(len(xyz), synth.POINT)
    p["x"], p["y"], p["z"] = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    p["label"] = label
    return p


def world(name, seed=0):
    """Raw clouds (before scan_prepare): floor_walls, cylinder, edge (two planes meeting in a line), outliers (isolated
    points with fewer than 3 neighbours beside a patch), nan (a patch with NaN points; run it with downsampling off)."""
    rng = np.random.default_rng(seed)
    if name == "floor_walls":
        g = rng.uniform(-6, 6, (6000, 2))
        floor = np.c_[g, np.full(len(g), -0.6)]
        w1 = np.c_[rng.uniform(-6, 6, 2500), np.full(2500, 3.0), rng.uniform(-0.6, 1.5, 2500)]
        w2 = np.c_[np.full(2500, -2.5), rng.uniform(-6, 6, 2500), rng.uniform(-0.6, 1.5, 2500)]
        xyz = np.r_[floor, w1, w2]
    elif name == "cylinder":
        a = rng.uniform(0, 2 * np.pi, 8000)
        xyz = np.c_[2.0 * np.cos(a), 2.0 * np.sin(a), rng.uniform(-1, 1, 8000)]
    elif name == "edge":
        u = rng.uniform(0, 1.5, (3000, 2))
        xyz = np.r_[np.c_[1.0 + u[:, 0], u[:, 1] - 0.75, np.zeros(3000)], np.c_[np.full(3000, 1.0), u[:, 1] - 0.75, u[:, 0]]]
    elif name == "outliers":
        g = rng.uniform(-1.5, 1.5, (1500, 2))
        patch = np.c_[g[:, 0] + 3.0, g[:, 1], 0.2 * g[:, 0]]
        iso = np.c_[np.linspace(-5, 5, 12), np.full(12, 4.0), np.zeros(12)]
        pair = np.array([[-4.0, -4.0, 0.0], [-4.0, -3.9, 0.0]])
        xyz = np.r_[patch, iso, pair]
    elif name == "nan":
        g = rng.uniform(-2, 2, (2000, 2))
        xyz = np.c_[g[:, 0] + 2.5, g[:, 1], 0.1 * g[:, 1]]
        xyz[::97] = np.nan
        xyz[5::131, 2] = np.nan
    else:
        raise ValueError(name)
    return _pts(xyz.astype(F), label=0)


WORLDS = ("floor_walls", "cylinder", "edge", "outliers", "nan")
