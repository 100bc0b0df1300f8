"""The NN-field lookup of the likelihood kernels' phase A, split into an address step, the directory load and the decode
(device_funcs.cuh: nnf_address, nnf_entry, nnf_slot; kernels.cuh: nf_phase_a), must give every query the count and
first candidate nnf_lookup gives it: inside the lattice, on its last voxel of each axis, just outside it on every face,
and in regular, wide and overflow cells.  Run on the host (tests/hostsim/nnf_split_hostsim.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "nnf_split_hostsim.cpp")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nnfsplit") / "libnnfsplit.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hostsim_nnf_split.argtypes = [vp, vp, C.c_float, vp, vp, vp, C.c_size_t, vp, vp, vp, vp, vp]
    L.hostsim_nnf_split.restype = C.c_int
    return L


def directory(dims, rng):
    """Directory entries of every coarse cell: regular (nibble counts), wide (byte counts in a side table) or overflow."""
    n_cells = int(np.prod([(d + 1) // 2 for d in dims]))
    dir_ = np.zeros((n_cells, 2), np.uint32)
    wide = []
    kinds = rng.choice(3, n_cells, p=[0.6, 0.2, 0.2])
    for c in range(n_cells):
        if kinds[c] == 0:
            nib = rng.integers(0, 15, 8)
            dir_[c] = (rng.integers(0, 1 << 24), sum(int(v) << (4 * k) for k, v in enumerate(nib)))
        elif kinds[c] == 1:
            cnt = rng.integers(0, 41, 8)
            lo = sum(int(v) << (8 * k) for k, v in enumerate(cnt[:4]))
            hi = sum(int(v) << (8 * k) for k, v in enumerate(cnt[4:]))
            dir_[c] = (0x80000000 | len(wide), 0xfffffffe)
            wide.append((rng.integers(0, 1 << 24), lo, hi, 0))
        else:
            dir_[c] = (0xffffffff, 0xffffffff)
    wide = np.array(wide or [(0, 0, 0, 0)], np.uint32)
    return dir_, wide, kinds


def queries(dims, origin, e, rng):
    """Voxel centres of the whole lattice, the faces just outside it, its exact bounds and a few far points."""
    o = np.asarray(origin, np.float64)
    n = np.asarray(dims)
    grid = np.stack(np.meshgrid(*[np.arange(d) for d in dims], indexing="ij"), -1).reshape(-1, 3)
    inside = o + (grid + 0.5) * e
    out = []
    for a in range(3):
        for v in (-0.5, n[a] + 0.5, -3.5, n[a] + 3.5):
            p = o + (rng.integers(0, n, (16, 3)) + 0.5) * e
            p[:, a] = o[a] + v * e
            out.append(p)
    outside = np.concatenate(out)
    bounds = []
    for a in range(3):
        p = o + (rng.integers(0, n, (2, 3)) + 0.5) * e
        lo, hi = p.copy(), p.copy()
        lo[:, a] = o[a]                 # the lattice's lower face: voxel 0
        hi[:, a] = o[a] + n[a] * e      # its upper face: one past the last voxel
        bounds += [lo, hi]
    far = np.array([[1e30, 0.0, 0.0], [0.0, -1e30, 0.0], [0.0, 0.0, 3e9]])
    return inside.astype(np.float32), outside.astype(np.float32), np.concatenate(bounds + [far]).astype(np.float32)


def run(lib, dims, origin, e, dir_, wide, q):
    q = np.ascontiguousarray(q, np.float32)
    nq = len(q)
    lc, sc = np.zeros(nq, np.int32), np.zeros(nq, np.int32)
    ls, ss = np.zeros(nq, np.uint32), np.zeros(nq, np.uint32)
    inside = np.zeros(nq, np.uint8)
    d = np.asarray(dims, np.int32)
    o = np.asarray(origin, np.float32)
    assert lib.hostsim_nnf_split(d.ctypes.data, o.ctypes.data, 1.0 / e, dir_.ctypes.data, wide.ctypes.data,
                                 q.ctypes.data, nq, lc.ctypes.data, ls.ctypes.data, sc.ctypes.data, ss.ctypes.data,
                                 inside.ctypes.data) == 0
    return lc, ls, sc, ss, inside.astype(bool)


@pytest.mark.parametrize("dims", [(7, 6, 5), (8, 3, 9), (1, 1, 1)])
def test_nnf_split_equals_lookup(lib, dims):
    rng = np.random.default_rng(sum(dims))
    origin, e = (-1.25, 0.75, 2.125), 0.25
    dir_, wide, kinds = directory(dims, rng)
    inside, outside, bounds = queries(dims, origin, e, rng)
    for name, q in (("inside", inside), ("outside", outside), ("bounds", bounds)):
        lc, ls, sc, ss, in_ = run(lib, dims, origin, e, dir_, wide, q)
        bad = np.flatnonzero((lc != sc) | (ls != ss))
        assert bad.size == 0, (name, q[bad[:4]], lc[bad[:4]], sc[bad[:4]], ls[bad[:4]], ss[bad[:4]])
        if name == "inside":
            assert in_.all()
            assert (lc == -1).any() == (kinds == 2).any()
        elif name == "outside":
            assert not in_.any() and (lc == 0).all()
        else:
            # per axis: the lower face is voxel 0 (inside), the upper face is one past the last voxel (outside)
            assert in_[:-3].reshape(3, 2, 2)[:, 0].all() and not in_[:-3].reshape(3, 2, 2)[:, 1].any()
            assert not in_[-3:].any()


def test_nnf_split_sees_wide_and_overflow_cells(lib):
    """The directory draw of the cases above does exercise wide cells with more than 14 candidates in a voxel."""
    dims = (7, 6, 5)
    rng = np.random.default_rng(sum(dims))
    origin, e = (-1.25, 0.75, 2.125), 0.25
    dir_, wide, kinds = directory(dims, rng)
    inside, _, _ = queries(dims, origin, e, rng)
    lc, ls, sc, ss, _ = run(lib, dims, origin, e, dir_, wide, inside)
    assert (kinds == 1).any() and (kinds == 2).any()
    assert (lc > 14).any() and (lc == -1).any()
    assert np.array_equal(lc, sc) and np.array_equal(ls, ss)
