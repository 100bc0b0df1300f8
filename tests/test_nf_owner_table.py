"""The owner table of lik_kernel_nf's candidate scan (kernels.cuh: nf_warp_scan), built from marks and a warp max-scan
(device_funcs.cuh: nnf_owner_mark, nnf_owner_run_max, nnf_owner_scan_word, nnf_owner_evals), modelled lane by lane on
the host (tests/hostsim/nf_owner_hostsim.cpp): every pass's table must equal, byte for byte, the table of the serial
per-list fill it replaces (nnf_fill_owner), and the candidate scan run on it must give every eval the serial fminf of
its list."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "nf_owner_hostsim.cpp")
PASSES = (1024, 64, 32, 16)


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nfowner") / "libnfowner.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hostsim_nf_owner_tables.argtypes = [C.c_int, vp, C.c_int, C.c_int, vp, vp]
    L.hostsim_nf_owner_tables.restype = C.c_int
    L.hostsim_nf_owner_scan_words.argtypes = [vp, C.c_int, C.c_uint32, vp]
    L.hostsim_nf_owner_scan_words.restype = None
    L.hostsim_nf_owner_warp_scan.argtypes = [C.c_int, vp, vp, vp, vp, C.c_float, C.c_int, vp, vp]
    L.hostsim_nf_owner_warp_scan.restype = C.c_int
    return L


def tables(lib, U, count, pass_slots):
    count = np.ascontiguousarray(count, np.int32)
    assert count.shape == (32 * U,)
    max_passes = int(np.maximum(count, 0).sum()) // pass_slots + 1
    table = np.full(max_passes * pass_slots, 0xAB, np.uint8)
    serial = np.full(max_passes * pass_slots, 0xCD, np.uint8)
    W = lib.hostsim_nf_owner_tables(U, count.ctypes.data, pass_slots, max_passes, table.ctypes.data,
                                    serial.ctypes.data)
    assert W == int(np.maximum(count, 0).sum())
    return W, table[:W], serial[:W]


def check(lib, U, count):
    for pass_slots in PASSES:
        W, table, serial = tables(lib, U, count, pass_slots)
        bad = np.flatnonzero(table != serial)
        assert bad.size == 0, (pass_slots, W, bad[:8], table[bad[:8]], serial[bad[:8]])


def owners(U, count):
    """Slot -> eval by the definition: eval e = u * 32 + lane, lists laid out lane after lane."""
    return np.concatenate([np.full(max(count[u * 32 + lane], 0), u * 32 + lane, np.uint8)
                           for lane in range(32) for u in range(U)] + [np.zeros(0, np.uint8)])


@pytest.mark.parametrize("U", [1, 2, 4, 8])
@pytest.mark.parametrize("seed", range(8))
def test_table_equals_serial_fill(lib, U, seed):
    """Regular (0-14), wide (15-40) and overflow (-1) cells, as in the candidate-scan test."""
    rng = np.random.default_rng(100 + seed)
    E = 32 * U
    kind = rng.random(E)
    count = np.where(kind < 0.15 + 0.1 * (seed % 3), 0, rng.integers(1, 15, E))
    count = np.where(kind > 0.9, rng.integers(15, 41, E), count)
    count = np.where((kind > 0.85) & (kind <= 0.9), -1, count).astype(np.int32)
    check(lib, U, count)
    W, table, _ = tables(lib, U, count, 1024)
    assert np.array_equal(table, owners(U, count))


def test_no_candidates(lib):
    """W = 0: no pass, nothing written."""
    for count in (np.zeros(128, np.int32), np.full(128, -1, np.int32)):
        W, table, _ = tables(lib, 4, count, 1024)
        assert W == 0 and table.size == 0


def test_empty_lists_at_pass_boundaries(lib):
    """Every pass boundary of 16 and 32 slots falls between lists, with empty and overflow lists sitting on it."""
    count = np.zeros(128, np.int32)
    order = [(lane, u) for lane in range(32) for u in range(4)]  # slot order of the lists
    for i, (lane, u) in enumerate(order):
        count[u * 32 + lane] = [8, 0, 8, -1][i % 4]
    check(lib, 4, count)


def test_list_spanning_three_passes(lib):
    """One 40-candidate list over passes of 16 slots: it starts mid-pass, fills the next and ends in the third."""
    count = np.zeros(128, np.int32)
    count[0 * 32 + 0] = 5   # lane 0, u 0: slots 0-4
    count[1 * 32 + 0] = 40  # lane 0, u 1: slots 5-44 (passes 0, 1 and 2 of 16)
    count[0 * 32 + 1] = 3
    count[3 * 32 + 31] = 1  # the last ordinal
    check(lib, 4, count)
    W, table, _ = tables(lib, 4, count, 16)
    assert W == 49 and (table[5:45] == 32).all() and table[48] == 3 * 32 + 31


def test_single_and_last_lists(lib):
    """Only ordinal 0, only the last ordinal (255 with U = 8), one slot each and many."""
    for U in (4, 8):
        for e, c in ((0, 1), (0, 40), (32 * U - 1, 1), (32 * U - 1, 40)):
            count = np.zeros(32 * U, np.int32)
            count[e] = c
            check(lib, U, count)


def test_every_slot_its_own_list(lib):
    """128 lists of one slot: a mark in every byte, across round and pass boundaries."""
    check(lib, 4, np.ones(128, np.int32))
    check(lib, 8, np.ones(256, np.int32))


@pytest.mark.parametrize("seed", range(4))
def test_scan_word_is_the_prefix_maximum(lib, seed):
    """nnf_owner_scan_word on arbitrary bytes (not only growing marks): the running maximum in slot order."""
    rng = np.random.default_rng(seed)
    n = 256
    b = rng.integers(0, 256, 4 * n).astype(np.uint8)
    b[rng.random(4 * n) < 0.5] = 0
    run0 = int(rng.integers(0, 256))
    out = np.zeros(n, np.uint32)
    words = np.ascontiguousarray(b.view("<u4"))
    lib.hostsim_nf_owner_scan_words(words.ctypes.data, n, run0, out.ctypes.data)
    want = np.maximum.accumulate(np.concatenate([[run0], b]).astype(np.uint8))[1:]
    assert np.array_equal(out.view(np.uint8), want)


@pytest.mark.parametrize("U", [1, 4])
@pytest.mark.parametrize("seed", range(4))
def test_scan_on_the_table_matches_serial_min(lib, U, seed):
    """The candidate scan reading the new table: each eval's best is the serial fminf over its list, any slot order."""
    rng = np.random.default_rng(200 + seed)
    E = 32 * U
    kind = rng.random(E)
    count = np.where(kind < 0.15, 0, rng.integers(1, 15, E))
    count = np.where(kind > 0.9, rng.integers(15, 41, E), count)
    count = np.where((kind > 0.85) & (kind <= 0.9), -1, count).astype(np.int32)
    cand = (rng.random((4096, 4)) * 4.0 - 2.0).astype(np.float32)
    first = rng.integers(0, 4096 - 41, E).astype(np.uint32)
    q = (rng.random((E, 3)) * 4.0 - 2.0).astype(np.float32)
    r2 = np.float32(1.0)
    want = np.full(E, r2, np.float32)
    for e in range(E):
        for i in range(max(count[e], 0)):
            d = q[e] - cand[first[e] + i, :3]
            want[e] = min(want[e], np.float32(np.float32(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
    for pass_slots in (1024, 64, 32):
        perm = rng.permutation(pass_slots).astype(np.int32)
        best = np.zeros(E, np.float32)
        W = lib.hostsim_nf_owner_warp_scan(U, count.ctypes.data, first.ctypes.data, q.ctypes.data, cand.ctypes.data,
                                           r2, pass_slots, perm.ctypes.data, best.ctypes.data)
        assert W == int(np.maximum(count, 0).sum())
        assert np.array_equal(best.view(np.uint32), want.view(np.uint32)), pass_slots
