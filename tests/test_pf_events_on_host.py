"""The odometry-noise redraw, expansion resetting's noise and the IMU gravity update without a GPU: the device functions
of mcl_3dl_b200/csrc/pf_funcs.cuh, compiled for the host by tests/hostsim/pf_events_hostsim.cpp, equal both CPU checkers
bit for bit given the same draws — the port (oracle/pf_events_oracle.cpp) and the reference tier
(oracle/pf_events_ref_driver.cpp: the node's redraw lambda through pf::ParticleFilter::predict,
addNoiseUsingNoiseGenerator and ImuMeasurementModelGravity inside pf::ParticleFilter::measure, all the reference's own
code).  The draws themselves are recomputed here from the counter layout include/mcl3dl_b200.h documents, with glibc's
logf / cosf / sinf, which the host build calls too."""
import ctypes as C
import ctypes.util
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from oracle import pf_events_checker as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "pf_events_hostsim.cpp")
SIGMA_CASES = [(0.0, 0.0, 0.0, 0.0), (0.1, 0.05, 0.02, 0.07), (1e3, 1e-3, 3.0, 1e30)]


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pfehs") / "libpfehs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, sz, u32, u64, d = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.c_double
    L.hostsim_pf_redraw.argtypes = [vp, sz, u64, u32, d, d, d, d]
    L.hostsim_pf_redraw.restype = None
    L.hostsim_pf_noise.argtypes = [vp, sz, u64, u32, vp, vp, vp]
    L.hostsim_pf_noise.restype = None
    L.hostsim_pf_noise6_event.argtypes = [u64, u32, u32, u32, vp, vp]
    L.hostsim_pf_noise6_event.restype = None
    L.hostsim_pf_imu.argtypes = [vp, sz, vp, d, vp, vp]
    L.hostsim_pf_imu.restype = None
    return L


@pytest.fixture(scope="module")
def port():
    pc.build("port")
    return pc.PfEventsChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not pc.build("reference"):
        pytest.skip("reference checker not built (no reference checkout)")
    return pc.PfEventsChecker("reference")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def states(n, seed, scale=(0.9, 1.1)):
    """Non-unit rotations (half of them with w < 0), nonzero noise and odometry-error fields, signed zeros."""
    rng = np.random.default_rng(seed)
    st = np.zeros(n, synth.STATE)
    st["pos"] = rng.uniform(-30, 30, (n, 3))
    q = rng.normal(0, 1, (n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[::2, 3] = -np.abs(q[::2, 3])
    st["rot"] = q * rng.uniform(*scale, (n, 1))
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        st[f] = rng.normal(0, 0.1, n)
    st["odom_err_integ_lin"] = rng.normal(0, 0.2, (n, 3))
    st["odom_err_integ_ang"] = rng.normal(0, 0.2, (n, 3))
    st["pos"][::5, 2] = -0.0
    return st


# ------------------------------------------------------------------ the draws, recomputed from the documented layout
_M = C.CDLL(ctypes.util.find_library("m"))
for _f in ("logf", "cosf", "sinf"):
    getattr(_M, _f).argtypes = [C.c_float]
    getattr(_M, _f).restype = C.c_float
F = np.float32


def philox(ctr, seed):
    c = [int(x) & 0xFFFFFFFF for x in ctr]
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c[3] ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF]
        k0, k1 = (k0 + 0x9E3779B9) & 0xFFFFFFFF, (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c


def box_muller(u_word, v_word):
    u = F(F((u_word >> 8) + 1) * F(2.0 ** -24))
    v = F(F((v_word >> 8) + 1) * F(2.0 ** -24))
    rad = F(np.sqrt(F(F(-2.0) * F(_M.logf(u)))))
    phi = F(F(6.283185307179586) * v)
    return F(rad * F(_M.cosf(phi))), F(rad * F(_M.sinf(phi)))


def redraw_z(seed, index, call):
    w = philox((index, call, 0, 1), seed)
    return box_muller(w[0], w[1]) + box_muller(w[2], w[3])


def noise6(seed, index, call, event, sigma):
    a, b = philox((index, call, 0, event), seed), philox((index, call, 1, event), seed)
    z = box_muller(a[0], a[1]) + box_muller(a[2], a[3]) + box_muller(b[0], b[1])
    return np.array([F(0) if s == 0 else F(zk * F(s)) for zk, s in zip(z, sigma)], F)


def test_draws_follow_the_documented_counter_layout(hs):
    sigma = np.array([0.3, 0.0, 2.0, 0.1, 0.2, 1e-3], F)
    for seed, call, index in [(0, 1, 0), (12345, 1, 7), (2 ** 63 + 99, 4, 65535), (77, 3, 1 << 20)]:
        for event in (0, 2):   # 0: resampling's stream, 2: the expansion noise
            got = np.zeros(6, F)
            hs.hostsim_pf_noise6_event(seed, index, call, event, _p(sigma), _p(got))
            assert got.tobytes() == noise6(seed, index, call, event, sigma).tobytes(), (seed, call, index, event)
        st = np.zeros(index + 1, synth.STATE)
        hs.hostsim_pf_redraw(_p(st), len(st), seed, call, 1.0, 1.0, 1.0, 1.0)
        z = np.array(redraw_z(seed, index, call), F)
        got = np.array([st["noise_ll"][index], st["noise_la"][index], st["noise_aa"][index], st["noise_al"][index]], F)
        assert got.tobytes() == z.tobytes()
    # the three events of one (seed, index, call) draw from different blocks
    a = noise6(5, 3, 1, 0, np.ones(6, F))
    b = noise6(5, 3, 1, 2, np.ones(6, F))
    assert not np.array_equal(a, b) and not np.array_equal(a[:4], np.array(redraw_z(5, 3, 1), F))


# ------------------------------------------------------------------ the redraw
def host_z(hs, n, seed, call):
    st = np.zeros(n, synth.STATE)
    hs.hostsim_pf_redraw(_p(st), n, seed, call, 1.0, 1.0, 1.0, 1.0)   # float(double(z) * 1.0) == z
    return np.stack([st["noise_ll"], st["noise_la"], st["noise_aa"], st["noise_al"]], 1)


@pytest.mark.parametrize("sg", SIGMA_CASES)
@pytest.mark.parametrize("n", [1, 1000])
def test_redraw_equals_both_checkers(hs, port, ref, sg, n):
    st = states(n, 3)
    z = host_z(hs, n, 99, 2)
    got = st.copy()
    hs.hostsim_pf_redraw(_p(got), n, 99, 2, *sg)
    want = port.redraw(st, z, *sg)
    assert got.tobytes() == want.tobytes()
    assert ref.redraw(st, z, *sg).tobytes() == want.tobytes()
    for f in ("pos", "rot", "odom_err_integ_lin", "odom_err_integ_ang"):   # nothing else changes
        assert got[f].tobytes() == st[f].tobytes()
    if sg == SIGMA_CASES[0]:
        assert (got["noise_ll"] == 0).all() and (np.signbit(got["noise_ll"]) == (z[:, 0] < 0)).all()   # -0.0 kept


# ------------------------------------------------------------------ expansion noise
@pytest.mark.parametrize("sp,sr", [((0, 0, 0), (0, 0, 0)), ((0.2, 0.2, 0.05), (0.02, 0.02, 0.1)),
                                   ((100.0, 0.0, 5.0), (3.0, 1.5, 6.0))])
@pytest.mark.parametrize("n", [1, 1000])
def test_noise_equals_both_checkers_unnormalised(hs, port, ref, sp, sr, n):
    st = states(n, 4)
    got = st.copy()
    org = np.zeros((n, 6), F)
    hs.hostsim_pf_noise(_p(got), n, 2024, 3, _p(np.array(sp, F)), _p(np.array(sr, F)), _p(org))
    want = port.noise(st, org)
    assert got.tobytes() == want.tobytes()
    assert ref.noise(st, org).tobytes() == want.tobytes()
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        assert (got[f] == 0).all()
    norm = np.linalg.norm(got["rot"].astype(np.float64), axis=1)
    assert np.abs(norm - 1).max() > 0.05          # the input's non-unit norms survive: no normalize()
    if max(sp + sr) == 0:   # zero sigma: pos + 0 (-0.0 becomes +0.0, as in the reference)
        assert (got["pos"] == st["pos"]).all() and not np.signbit(got["pos"][st["pos"] == 0]).any()


# ------------------------------------------------------------------ IMU gravity update
def same(a, b):
    """Bit for bit, except that a NaN only has to be a NaN (its sign and payload depend on the compiler's negation)."""
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def host_imu(hs, st, acc, var):
    lik = np.zeros(len(st), F)
    consts = np.zeros(3, F)
    hs.hostsim_pf_imu(_p(np.ascontiguousarray(st)), len(st), _p(np.array(acc, F)), var, _p(lik), _p(consts))
    return lik, consts


def check_imu(hs, port, ref, st, probs, acc, var):
    lik, consts = host_imu(hs, st, acc, var)
    p_port, l_port, k_port, s_port, e_port = port.imu(st, probs, acc, var)
    p_ref, l_ref, k_ref, s_ref, e_ref = ref.imu(st, probs, acc, var)
    assert same(lik, l_port) and same(lik, l_ref)
    assert p_port.tobytes() == p_ref.tobytes() and k_port == k_ref
    assert same(np.array([s_port, e_port]), np.array([s_ref, e_ref]))
    s = F(np.float64(var))
    assert consts[1] == F(1.0 / np.sqrt(2.0 * np.pi * np.float64(s) * np.float64(s)))
    assert consts[2] == F(np.float64(F(s * s)) * 2.0)
    if not k_ref:
        assert p_ref.tobytes() == np.asarray(probs, F).tobytes()   # the prior, untouched
    return lik, k_ref


@pytest.mark.parametrize("var", [0.01, 0.3, 1e3])
@pytest.mark.parametrize("n", [1, 1000])
def test_imu_equals_both_checkers(hs, port, ref, var, n):
    st = states(n, 5)
    probs = np.random.default_rng(6).uniform(0.1, 1.0, n).astype(F)
    for acc in [(0.0, 0.0, 1.0), (0.1, -0.05, 0.98), (0.0, 0.0, 9.81), (-0.3, 0.2, -0.9)]:
        check_imu(hs, port, ref, st, probs, acc, var)


def test_imu_identity_rotations(hs, port, ref):
    st = np.zeros(4, synth.STATE)
    st["rot"] = [[0, 0, 0, 1], [0, 0, 0, -1], [0, 0, 0, 1], [0, 0, 0, -1]]
    lik, kept = check_imu(hs, port, ref, st, np.full(4, 0.25, F), (0.0, 0.0, 1.0), 0.1)
    a = F(1.0 / np.sqrt(2.0 * np.pi * np.float64(F(0.1)) ** 2))
    assert kept and (lik == a).all()      # diff = acosf(1) = 0


def nan_states(hs, n_want=3):
    """Particles whose acosf argument rounds above 1 for acc = their own float estimate of gravity."""
    rng = np.random.default_rng(11)
    found = []
    for _ in range(200):
        q = rng.normal(0, 1, 4)
        q /= np.linalg.norm(q)
        st = np.zeros(1, synth.STATE)
        st["rot"] = q
        x, y, z, w = q
        g = np.array([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)])   # R^T e_z
        lik, _ = host_imu(hs, st, g.astype(F), 0.1)
        if np.isnan(lik[0]):
            found.append((st[0], g.astype(F)))
            if len(found) == n_want:
                break
    assert found, "no NaN-producing rotation found"
    return found


def test_imu_nan_discards_the_update(hs, port, ref):
    for s0, acc in nan_states(hs):
        st = states(64, 8)
        st[17] = s0
        probs = np.random.default_rng(9).uniform(0.1, 1.0, 64).astype(F)
        lik, kept = check_imu(hs, port, ref, st, probs, acc, 0.1)
        assert np.isnan(lik[17]) and np.isfinite(np.delete(lik, 17)).all() and not kept


def test_imu_all_zero_likelihoods_keep_the_prior(hs, port, ref):
    st = np.zeros(16, synth.STATE)
    st["rot"] = [1.0, 0.0, 0.0, 0.0]          # upside down: diff = pi
    probs = np.full(16, 1 / 16, F)
    lik, kept = check_imu(hs, port, ref, st, probs, (0.0, 0.0, 1.0), 0.01)
    assert (lik == 0).all() and not kept
