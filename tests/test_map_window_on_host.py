"""The map window's arithmetic without a GPU: mcl_3dl_b200/csrc/window_funcs.cuh, compiled for the host by
tests/hostsim/window_hostsim.cpp, against a Python restatement of the required box, the growth, the clamp, the lattice
and the containment test; and a randomized property check that every query of a call, transformed with the kernels' own
float transform, lies inside the required box with each search radius around it."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "window_hostsim.cpp")
F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("winhs") / "libwinhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hostsim_win_need.argtypes = [vp, C.c_size_t, vp, C.c_size_t, vp, C.c_size_t, vp]
    L.hostsim_win_required.argtypes = [vp, C.c_float, C.c_float, C.c_float, vp, vp]
    L.hostsim_win_reach.argtypes = [vp]
    L.hostsim_win_reach.restype = C.c_double
    L.hostsim_win_choose.argtypes = [vp, C.c_double, vp, C.c_float, C.c_uint64, vp]
    L.hostsim_win_lattice.argtypes = [vp, vp, C.c_float, vp, vp]
    L.hostsim_win_lattice.restype = C.c_uint64
    L.hostsim_win_contains.argtypes = [vp, vp]
    L.hostsim_win_transform.argtypes = [vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---- Python restatement
def ordf(u):
    u = int(u)
    b = (u & 0x7fffffff) if (u & 0x80000000) else (~u & 0xffffffff)
    return float(np.array([b], np.uint32).view(F)[0])


def bitsf(u):
    return float(np.array([u], np.uint32).view(F)[0])


def r_reach(need):
    return bitsf(need[6]) * bitsf(need[7]) * (1.0 + 2.0 ** -20)


def r_required(need, r_scaled, grid_min, hit_tol, w):
    pmin = [ordf(~int(need[k]) & 0xffffffff) for k in range(3)]
    pmax = [ordf(need[3 + k]) for k in range(3)]
    reach = r_reach(need)
    extra = steps = 0.0
    if grid_min > 0:
        extra = max(float(F(hit_tol)), float(F(grid_min))) * (1.0 + 2.0 ** -10)
        steps = math.ceil((2.0 * reach + float(F(hit_tol))) / float(F(grid_min))) + 2.0
    lo, hi = [], []
    for k in range(3):
        r = float(F(r_scaled)) / float(F(w[k])) * (1.0 + 2.0 ** -20)
        mag = max(abs(pmin[k]), abs(pmax[k])) + reach + extra + r
        half = reach + extra + r + mag * (2.0 ** -16 + steps * 2.0 ** -21)
        a, b = pmin[k] - half, pmax[k] + half
        if not (math.isfinite(a) and math.isfinite(b)) or abs(a) > 1e30 or abs(b) > 1e30:
            return None
        fa, fb = F(a), F(b)
        if float(fa) > a:
            fa = np.nextafter(fa, F(-np.inf))
        if float(fb) < b:
            fb = np.nextafter(fb, F(np.inf))
        lo.append(fa)
        hi.append(fb)
    return np.array(lo + hi, F)


def r_lattice(box, w, cell):
    total = 1
    dims = []
    for k in range(3):
        smin, smax = F(box[k]) * F(w[k]), F(box[3 + k]) * F(w[k])
        if not (np.isfinite(smin) and np.isfinite(smax)) or not smax >= smin:
            return 0, None
        org = F(smin - F(0.5) * F(cell))
        d = math.floor((float(smax) - float(org)) / float(F(cell))) + 2
        if d >= 2 ** 31:
            return 0, None
        dims.append(d)
        total *= d
        if total >= 2 ** 31:
            return 0, None
    return total, dims


def r_grown(req, g):
    lo = [min(F(float(req[k]) - g), req[k]) for k in range(3)]
    hi = [max(F(float(req[3 + k]) + g), req[3 + k]) for k in range(3)]
    return np.array(lo + hi, F)


def r_choose(req, reach, w, cell, cap):
    g = reach
    for _ in range(8):
        b = r_grown(req, g)
        cells, _d = r_lattice(b, w, cell)
        if cells and cells <= cap:
            return b
        g *= 0.5
    cells, _d = r_lattice(req, w, cell)
    return req if cells and cells <= cap else None


def r_need(poses, pts, org):
    """window_need_kernel's reduction, restated with numpy (float64 products, rounded up to float)."""
    w = [0] * 8

    def ordu(f):
        b = int(np.array([f], F).view(np.uint32)[0])
        return (~b & 0xffffffff) if b & 0x80000000 else (b | 0x80000000)

    for p in poses:
        c = [p["px"], p["py"], p["pz"], p["qx"], p["qy"], p["qz"], p["qw"]]
        if not all(np.isfinite(c)):
            continue
        for k in range(3):
            w[k] = max(w[k], ~ordu(c[k]) & 0xffffffff)
            w[3 + k] = max(w[3 + k], ordu(c[k]))
        q2 = max(sum(float(v) * float(v) for v in c[3:]), 1.0)
        s = F(q2)
        if float(s) < q2:
            s = np.nextafter(s, F(np.inf))
        w[7] = max(w[7], int(np.array([s], F).view(np.uint32)[0]))
    for x, y, z in list(zip(pts["x"], pts["y"], pts["z"])) + [tuple(o) for o in org]:
        if not (np.isfinite(x) and np.isfinite(y) and np.isfinite(z)):
            continue
        n2 = float(x) * float(x) + float(y) * float(y) + float(z) * float(z)
        r = math.sqrt(n2)
        if r * r < n2:
            r = math.nextafter(r, math.inf)
        r *= 1.0 + 2.0 ** -40
        f = F(r)
        if float(f) < r:
            f = np.nextafter(f, F(np.inf))
        w[6] = max(w[6], int(np.array([f], F).view(np.uint32)[0]))
    return np.array(w, np.uint32)


def hs_need(L, poses, pts, org):
    out = np.zeros(8, np.uint32)
    org = np.ascontiguousarray(org, F).reshape(-1, 3)
    L.hostsim_win_need(_p(poses), len(poses), _p(pts), len(pts), _p(org), len(org), _p(out))
    return out


def random_call(rng, n_p=64, n_pts=200, spread=50.0, reach=10.0, nonfinite=False):
    pos = rng.uniform(-spread, spread, (n_p, 3)) + rng.uniform(-2000, 2000, 3)
    q = synth.quat_from_rpy(rng.uniform(-math.pi, math.pi, (n_p, 3)))
    q = (q * (1.0 + rng.normal(0, 1e-3, (n_p, 1)))).astype(F)  # raw, not quite unit quaternions
    poses = synth.make_poses(pos, q)
    d = rng.normal(0, 1, (n_pts, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    pts = synth.make_points((d * rng.uniform(0.0, reach, (n_pts, 1))).astype(F))
    org = rng.uniform(-0.3, 0.3, (2, 3)).astype(F)
    if nonfinite:
        poses["px"][0] = np.nan
        poses["qw"][1] = np.inf
        pts["x"][0] = np.nan
        pts["z"][1] = -np.inf
    return poses, pts, org


CASES = [(0.20002, 0.0, 0.0, (1.0, 1.0, 5.0)), (0.35, 0.1, 0.3, (1.0, 1.0, 5.0)), (0.5, 0.0, 0.0, (2.0, 0.5, 1.0)),
         (0.22, 0.05, 0.5, (1.0, 1.0, 1.0))]


@pytest.mark.parametrize("nonfinite", [False, True])
def test_need_and_required_box_equal_the_restatement(hs, nonfinite):
    rng = np.random.default_rng(11 + nonfinite)
    for _ in range(20):
        poses, pts, org = random_call(rng, nonfinite=nonfinite)
        need = hs_need(hs, poses, pts, org)
        assert need.tolist() == r_need(poses, pts, org).tolist()
        assert hs.hostsim_win_reach(_p(need)) == r_reach(need)
        for r_sc, gmin, htol, w in CASES:
            wv = np.array(w, F)
            box = np.zeros(6, F)
            ok = hs.hostsim_win_required(_p(need), r_sc, gmin, htol, _p(wv), _p(box))
            want = r_required(need, r_sc, gmin, htol, w)
            assert bool(ok) == (want is not None)
            assert box.tobytes() == want.tobytes()


def test_choose_lattice_and_containment_equal_the_restatement(hs):
    rng = np.random.default_rng(5)
    for _ in range(200):
        c = rng.uniform(-3000, 3000, 3)
        ext = rng.uniform(0.5, 40.0, 3)
        req = np.concatenate([c - ext, c + ext]).astype(F)
        w = np.array(rng.choice([(1.0, 1.0, 5.0), (1.0, 1.0, 1.0), (0.5, 2.0, 3.0)]), F)
        cell = F(rng.uniform(0.15, 0.6))
        cap = int(rng.choice([10 ** 5, 10 ** 6, 10 ** 7, 2 ** 31 - 1]))
        reach = float(rng.uniform(0.0, 20.0))
        dims = np.zeros(3, np.int32)
        org = np.zeros(3, F)
        cells = hs.hostsim_win_lattice(_p(req), _p(w), cell, _p(dims), _p(org))
        want_cells, want_dims = r_lattice(req, w, cell)
        assert cells == want_cells
        if cells:
            assert dims.tolist() == want_dims
        out = np.zeros(6, F)
        ok = hs.hostsim_win_choose(_p(req), reach, _p(w), cell, cap, _p(out))
        want = r_choose(req, reach, w, cell, cap)
        assert bool(ok) == (want is not None)
        if ok:
            assert out.tobytes() == want.tobytes()
            assert hs.hostsim_win_contains(_p(out), _p(req)) == 1
            got, _d = r_lattice(out, w, cell)
            assert 0 < got <= cap
        # containment: the restated rule on shifted boxes
        inner = req + F(rng.uniform(-1.0, 1.0))
        want_in = all(req[k] <= inner[k] and inner[3 + k] <= req[3 + k] for k in range(3))
        assert hs.hostsim_win_contains(_p(req), _p(inner)) == int(want_in)


def test_every_query_lies_inside_the_required_box(hs):
    """Property: with the kernels' float transform, each transformed scan point and each beam origin +/- every search
    radius (per axis, raw space) lies inside the required box; the KD march's overshoot of hit_tolerance past the end and
    one step before the begin as well."""
    rng = np.random.default_rng(23)
    for trial in range(40):
        poses, pts, org = random_call(rng, n_p=32, n_pts=64, spread=float(rng.uniform(0.1, 300.0)),
                                      reach=float(rng.uniform(0.5, 40.0)))
        need = hs_need(hs, poses, pts, org)
        for r_sc, gmin, htol, w in CASES:
            wv = np.array(w, F)
            box = np.zeros(6, F)
            assert hs.hostsim_win_required(_p(need), r_sc, gmin, htol, _p(wv), _p(box))
            rad = np.array([float(F(r_sc)) / float(wv[k]) for k in range(3)])
            ext = max(htol, gmin) if gmin > 0 else 0.0
            out = np.zeros(6, F)
            for pose in poses:
                for src in list(zip(pts["x"], pts["y"], pts["z"])) + [tuple(o) for o in org]:
                    p3 = np.array(src, F)
                    L = hs.hostsim_win_transform
                    L(_p(pose.reshape(1)), _p(p3), _p(out))
                    for q in (out[:3], out[3:]):
                        qd = q.astype(np.float64)
                        t = np.array([pose["px"], pose["py"], pose["pz"]], np.float64)
                        d = qd - t
                        nd = np.linalg.norm(d)
                        tip = qd + (d / nd * ext if nd > 0 else 0.0)  # the march's overshoot along the ray
                        # a point, anything within one march step of it (the second search behind the begin), and
                        # the overshoot past the end, each with the search radius around it
                        for c, e in ((qd, ext), (tip, 0.0)):
                            assert np.all(c - rad - e >= box[:3]) and np.all(c + rad + e <= box[3:]), (trial, c, box)
