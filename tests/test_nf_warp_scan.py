"""lik_kernel_nf's warp-cooperative candidate scan, modelled lane by lane on the host (tests/hostsim/nf_scan_hostsim.cpp,
built from the device helpers nnf_fill_owner / nnf_cand_d2 of device_funcs.cuh): the flattened (eval, candidate) list,
its owner table and the unsigned min over distance bits must give every eval exactly the serial fminf of its list, for
any processing order and pass size, with regular (0-14), wide (15-40) and overflow (-1) cells."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HS = os.path.join(ROOT, "tests", "hostsim")
SRC = os.path.join(HS, "nf_scan_hostsim.cpp")
DEPS = [SRC, os.path.join(HS, "cuda_shim.h"), os.path.join(ROOT, "mcl_3dl_b200", "csrc", "device_funcs.cuh"),
        os.path.join(ROOT, "mcl_3dl_b200", "csrc", "device_math.cuh")]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nfscan") / "libnfscan.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hostsim_nf_warp_scan.argtypes = [C.c_int, vp, vp, vp, vp, C.c_float, C.c_int, vp, vp]
    L.hostsim_nf_warp_scan.restype = C.c_int
    return L


def serial(count, first, q, cand, r2):
    """The kernel before: per eval, fminf over its list in order (float32 throughout, L2_Simple's order)."""
    out = np.full(len(count), r2, np.float32)
    for e, (c, s) in enumerate(zip(count, first)):
        for i in range(max(c, 0)):
            m = cand[s + i]
            dx, dy, dz = (np.float32(q[e, k]) - m[k] for k in range(3))
            out[e] = min(out[e], np.float32(np.float32(dx * dx + dy * dy) + dz * dz))
    return out


@pytest.mark.parametrize("U", [1, 4])
@pytest.mark.parametrize("seed", range(6))
def test_warp_scan_matches_serial_min(lib, U, seed):
    rng = np.random.default_rng(seed)
    E = 32 * U
    kind = rng.random(E)
    count = np.where(kind < 0.15, 0, rng.integers(1, 15, E))
    count = np.where(kind > 0.9, rng.integers(15, 41, E), count)  # wide cells
    count = np.where((kind > 0.85) & (kind <= 0.9), -1, count).astype(np.int32)  # overflow cells
    cand = (rng.random((4096, 4)) * 4.0 - 2.0).astype(np.float32)
    cand[rng.random(4096) < 0.05, :3] = 0.0  # ties: equal distances from several candidates
    first = rng.integers(0, 4096 - 41, E).astype(np.uint32)
    q = (rng.random((E, 3)) * 4.0 - 2.0).astype(np.float32)
    q[rng.random(E) < 0.1] = 0.0
    r2 = np.float32(rng.choice([0.04, 1.0, 9.0]))
    want = serial(count, first, q, cand, r2)
    for pass_slots in (1024, 64, 32):
        for order in range(3):
            perm = (np.arange(pass_slots) if order == 0 else rng.permutation(pass_slots)).astype(np.int32)
            best = np.zeros(E, np.float32)
            W = lib.hostsim_nf_warp_scan(U, count.ctypes.data, first.ctypes.data, q.ctypes.data, cand.ctypes.data, r2,
                                         pass_slots, perm.ctypes.data, best.ctypes.data)
            assert W == int(np.maximum(count, 0).sum())
            assert np.array_equal(best.view(np.uint32), want.view(np.uint32)), (pass_slots, order)
