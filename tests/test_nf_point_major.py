"""lik_kernel_nf_pm's point-major mapping and cross-CTA fold, modelled warp by warp on the host
(tests/hostsim/nf_pm_hostsim.cpp, built from nf_pm_shape / nf_fx_term / nf_pm_word / nf_pm_done of device_funcs.cuh): the slices
cover every scan point once, every live particle's record is stored exactly once whatever order the CTAs finish in, the
counts equal the serial counts, the score is the exact sum of the float contributions rounded once (so it is within the
rounding of the reference's serial float sum), the packed fields of the accumulator never overflow, and the
accumulators are left at zero."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "nf_pm_hostsim.cpp")
UNIT = 4  # kNfU: the points of one warp trip


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("nfpm") / "libnfpm.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hostsim_nf_pm_shape.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, vp]
    L.hostsim_nf_pm_run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, vp, vp, vp, vp, vp]
    L.hostsim_nf_pm_run.restype = C.c_int
    return L


def shape(lib, N, P, slots, r=0.2, w=5.0):
    s = np.zeros(6, np.int32)
    lib.hostsim_nf_pm_shape(N, (P + 255) // 256, slots, UNIT, r, w, s.ctypes.data)
    return [int(v) for v in s]  # slice, n_slices, fx_shift, arr_bits, cnt_bits, ok


@pytest.mark.parametrize("P,N", [(1024, 512), (65536, 64), (256, 96), (300, 97), (1000, 5), (4096, 1), (256, 0),
                                 (1 << 20, 512)])
def test_slices_cover_the_scan_once(lib, P, N):
    slots = 132 * 4
    slice_, n_slices, _, arr_bits, cnt_bits, ok = shape(lib, N, P, slots)
    assert ok
    assert n_slices < 2 ** arr_bits and N < 2 ** cnt_bits  # the arrival and count fields never carry
    assert slice_ % UNIT == 0 and slice_ >= UNIT
    assert n_slices >= 1 and (n_slices - 1) * slice_ < max(N, 1) <= n_slices * slice_ or N == 0
    blocks = (P + 255) // 256
    assert blocks * n_slices <= max(slots, blocks)  # one wave whenever the particle blocks alone fit


@pytest.mark.parametrize("w", [5.0, 1e-6, 3e4, -2.0])
@pytest.mark.parametrize("N,P", [(512, 1024), (64, 65536), (1, 256), (1024, 4096)])
def test_fixed_point_headroom(lib, N, P, w):
    r = 0.2
    _, _, k, a, c, ok = shape(lib, N, P, 528, r, w)
    assert ok
    sum_bits = 64 - a - c
    worst = Fraction(N) * Fraction(float(np.float32(r))) * Fraction(abs(float(np.float32(w)))) * (1 + Fraction(1, 1 << 20))
    assert worst * (Fraction(2) ** k) < 2 ** (sum_bits - 2)  # N maximal contributions fit the signed sum field
    assert Fraction(N, 2) / (worst * Fraction(2) ** k) <= Fraction(1, 1 << 30)  # N roundings: < 2^-30 of the bound


def test_long_scans_keep_the_particle_major_kernel(lib):
    assert not shape(lib, 1 << 16, 1024, 528)[5]


@pytest.mark.parametrize("N,P,slots", [(512, 1024, 528), (1, 256, 528), (2047, 1024, 528), (96, 4097, 132)])
def test_clamped_scales_keep_the_particle_major_kernel(lib, N, P, slots):
    """fx_shift is clamped to +-120 (2^fx_shift stays a normal float).  Where the clamp binds, the N roundings to
    2^-fx_shift are no longer below 2^-30 of the bound (match_weight = 1e-36: every term rounds to zero or one step),
    so the shape must not report ok.  Every shape that does report ok, over |match_weight| from 1e-40 to 1e38, keeps
    the headroom and rounding bounds of test_fixed_point_headroom."""
    r = 0.2
    assert not shape(lib, N, P, slots, r, 1e-36)[5] and not shape(lib, N, P, slots, r, -1e-36)[5]
    for w in [s * 10.0 ** d for d in range(-40, 39) for s in (1.0, -1.0)]:
        _, _, k, a, c, ok = shape(lib, N, P, slots, r, w)
        assert ok or abs(w) < 1e-6, w  # the clamp binds only for tiny weights
        if not ok:
            continue
        sum_bits = 64 - a - c
        worst = Fraction(N) * Fraction(float(np.float32(r))) * Fraction(abs(float(np.float32(w)))) * (1 + Fraction(1, 1 << 20))
        assert worst * (Fraction(2) ** k) < 2 ** (sum_bits - 2), w
        assert Fraction(N, 2) / (worst * Fraction(2) ** k) <= Fraction(1, 1 << 30), w


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("P,N,slots", [(1024, 512, 528), (300, 97, 528), (65, 40, 3), (513, 33, 528), (256, 0, 528)])
def test_fold_matches_serial(lib, seed, P, N, slots):
    rng = np.random.default_rng(seed)
    r, w = np.float32(0.2), np.float32(rng.choice([5.0, 0.01, -3.0]))
    slice_, n_slices, k, _, _, ok = shape(lib, N, P, slots, float(r), float(w))
    assert ok
    dist = (rng.random((P, N)) * r).astype(np.float32)
    dist[rng.random((P, N)) < 0.02] = 0.0  # a match at exactly match_dist_min still counts
    contrib = (dist * w).astype(np.float32)
    contrib[rng.random((P, N)) < 0.6] = np.nan  # no match
    contrib[P - 7:] = np.nan  # particles with no match at all
    contrib = np.ascontiguousarray(contrib)
    blocks = ((P + 31) // 32 + 7) // 8
    scores = []
    for order in range(3):
        cta = np.arange(blocks * n_slices, dtype=np.int32)
        if order:
            cta = rng.permutation(cta).astype(np.int32)
        score = np.full(P, np.nan, np.float32)
        cnt = np.zeros(P, np.uint32)
        written = np.zeros(P, np.int32)
        dirty = lib.hostsim_nf_pm_run(P, N, slots, UNIT, float(r), float(w), contrib.ctypes.data, cta.ctypes.data,
                                      score.ctypes.data, cnt.ctypes.data, written.ctypes.data)
        assert dirty == 0
        assert np.all(written == 1)
        m = ~np.isnan(contrib)
        assert np.array_equal(cnt, m.sum(axis=1).astype(np.uint32))
        scores.append(score)
    for s in scores[1:]:
        assert np.array_equal(s.view(np.uint32), scores[0].view(np.uint32))  # independent of the CTAs' order
    score = scores[0]
    if N == 0:
        assert np.all(score == 1.0)
        return
    for p in range(P):
        terms = contrib[p][~np.isnan(contrib[p])]
        exact = sum((Fraction(float(t)) for t in terms), Fraction(0))
        serial = np.float32(0.0)
        for t in terms:  # likelihood.cpp:128-133, one float addition per matched point in scan order
            serial = np.float32(serial + t)
        assert abs(Fraction(float(score[p])) - exact) <= abs(exact) * Fraction(1, 1 << 24) + Fraction(2) ** -k * len(terms)
        assert abs(float(score[p]) - float(serial)) <= 1e-5 * abs(float(serial)) + 1e-12
