"""The NN field after an append (engine.cu: update_nn_field), on the host (tests/hostsim/nnf_append_hostsim.cpp): the
field of map A, with only the directory cells marked by the device's marking function (device_funcs.cuh:
nnf_mark_append) re-selected over the grid of A + P, equals a fresh build of A + P in every directory cell (kind,
per-voxel counts, candidate bytes in order).  Every cell whose lists the patch changes is marked, and a small patch marks
a small share of the cells, so marking everything would fail."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "nnf_append_hostsim.cpp")


class Lik(C.Structure):
    _fields_ = [("match_weight", C.c_float), ("match_dist_min", C.c_float), ("match_dist_flat", C.c_float),
                ("dist_weight", C.c_float * 3)]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nnfappend") / "libnnfappend.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    L.hostsim_nnf_append.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.hostsim_nnf_append.restype = C.c_int
    return L


@pytest.fixture(scope="module")
def base():
    mp, info = synth.warehouse_map(12_000, seed=7)
    return mp, info


def run(lib, a, p, w=(1.0, 1.0, 5.0)):
    a = np.ascontiguousarray(a, synth.POINT)
    p = np.ascontiguousarray(p, synth.POINT)
    lik = Lik(5.0, 0.2, 0.05, (C.c_float * 3)(*w))
    out = np.zeros(8, np.uint64)
    assert lib.hostsim_nnf_append(a.ctypes.data, len(a), p.ctypes.data, len(p), C.byref(lik), out.ctypes.data) == 0
    keys = ("cells", "marked", "differ", "changed", "changed_unmarked", "same_box", "wide", "overflow")
    return dict(zip(keys, (int(v) for v in out)))


def pts(xyz):
    return synth.make_points(np.asarray(xyz, np.float32))


def box_faces(x0, y0, z0, size, h, rng):
    u = np.arange(0.0, size + 1e-6, h)
    a, b = [g.ravel() for g in np.meshgrid(u, u, indexing="ij")]
    z = np.zeros_like(a)
    one = np.concatenate([np.stack([a, z, b], 1), np.stack([a, z + size, b], 1), np.stack([z, a, b], 1),
                          np.stack([z + size, a, b], 1), np.stack([a, b, z + size], 1)])
    return one + (x0, y0, z0) + rng.normal(0.0, 0.01, one.shape)


def patch(kind, mp, info, seed):
    rng = np.random.default_rng(seed)
    L, H = info["L"], info["H"]
    xyz = np.stack([mp["x"], mp["y"], mp["z"]], 1).astype(np.float64)
    if kind == "dense":  # on and next to existing surface points
        near = xyz[rng.choice(len(xyz), 40, replace=False)]
        return pts(near + rng.normal(0.0, 0.05, near.shape))
    if kind == "empty":  # a new obstacle in free space inside the box
        return pts(box_faces(rng.uniform(1.0, L - 2.0), rng.uniform(1.0, L - 2.0), rng.uniform(0.3, H - 1.3), 0.9, 0.3, rng))
    c = np.array([rng.uniform(1.0, L - 1.0), rng.uniform(1.0, L - 1.0), rng.uniform(0.5, H - 0.5)])
    if kind == "wide":  # a tight cluster: 15..40 points none of which provably dominates the others
        return pts(c + rng.normal(0.0, 2e-4, (24, 3)))
    if kind == "overflow":  # a duplicate cluster: more survivors than a wide cell holds
        return pts(np.tile(c, (64, 1)))
    if kind == "boundary":  # points on the box's faces: the boxes do not move
        lo, hi = xyz.min(0), xyz.max(0)
        q = rng.uniform(lo, hi, (30, 3))
        q[:10, 0] = hi[0]
        q[10:20, 1] = lo[1]
        q[20:, 2] = hi[2]
        return synth.make_points(q.astype(np.float32))
    raise ValueError(kind)


@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("kind", ["dense", "empty", "wide", "overflow", "boundary"])
def test_append_reselects_exactly_what_changes(lib, base, kind, seed):
    mp, info = base
    p = patch(kind, mp, info, seed)
    for k in ("x", "y", "z"):  # inside the map's box (the lattice-change decision has its own test)
        p[k] = np.clip(p[k], mp[k].min(), mp[k].max())
    r = run(lib, mp, p)
    assert r["same_box"] == 1
    assert r["differ"] == 0, r
    assert r["changed_unmarked"] == 0, r
    assert r["changed"] > 0, r
    assert 0 < r["marked"] < 0.05 * r["cells"], r
    if kind == "wide":
        assert r["wide"] > 0, r
    if kind == "overflow":
        assert r["overflow"] > 0, r


def test_patch_outside_the_box_changes_the_lattice(lib, base):
    mp, info = base
    p = pts([[info["L"] + 0.5, info["L"] / 2, 1.0]])
    assert run(lib, mp, p)["same_box"] == 0
