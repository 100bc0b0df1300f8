"""The odometry-noise redraw, expansion resetting and the IMU gravity update on the resident set (H100) against the host
build of their device functions (tests/hostsim/pf_events_hostsim.cpp), which tests/test_pf_events_on_host.py holds bit
for bit to the port and reference checkers given the same draws.

Bars, derived as in tests/test_gpu_pf_exact.py (LIBM, R, ORG_REL there).  Everything in the new device functions is
explicit round-to-nearest arithmetic except logf / cosf / sinf (the draws), acosf and expf (the IMU likelihood):
  - redraw: noise_x = float(double(z) sigma) with z = rad cos(phi) (or sin): |Δ| <= ORG_REL |noise| + ulp(noise), every
    other field and the probabilities bit for bit.  The Philox words and the uniforms are integer and exact arithmetic;
    one different word would move its draws by O(1), far outside the bar, so agreement on every particle pins them;
  - expansion noise: pos, lin and ang within ulp(value) + ORG_REL |org| (org from the host's draws), noise_* exactly 0,
    rot within NOISE_ROT_BAR |rot|: RESAMPLE_ROT_BAR without the final normalisation's rounding (10 2^-23 for both
    sides), kept as the larger bar for simplicity;
  - IMU: diff = acosf(c) with c computed identically; acosf differs by <= LIBM["acosf"] ulp(diff); x = diff^2 / sq2 then
    carries 2 LIBM["acosf"] + 2 relative ulps, expf adds |x| times that plus LIBM["expf"], the two products one each:
    eps_i = ((2 LIBM["acosf"] + 2) |x_i| + LIBM["expf"] + 2) 2^-23 relative on w_i, plus prior_i 4 2^-149 absolute
    where expf's result is subnormal or underflows (its ulps are absolute there).  With Δw_i that bound and
    ΔS = Σ Δw_i, the weight sum is within ΔS + ulp(S) and each posterior within (Δw_i + p_i ΔS) / S + 2 2^-23 p_i
    + ulp(p_i) (the float rounding of S and the division); the entropy within Σ |Δp_i| (|ln p_i| + 1) + Σ LIBM["logf"] p_i ulp(ln p_i) + 1e-6 |H|.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from test_pf_events_on_host import hs, host_imu, host_z, nan_states, states  # noqa: F401
from test_gpu_pf_exact import LIBM, ORG_REL, R, RESAMPLE_ROT_BAR, ulp

pytestmark = pytest.mark.gpu

F = np.float32
NOISE_ROT_BAR = RESAMPLE_ROT_BAR
DENORM = 4 * 2.0 ** -149
# a standard normal z = rad cos(phi) (or sin): logf halved by the square root, the root, cosf / sinf, one product
Z_REL = (LIBM["logf"] / 2 + 1 + LIBM["cosf"] + 1) * R
PARITY = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "pf_events_parity_test")
SIZES = [1, 1000, 65_536, 1 << 20]
SIG = (0.3, 0.05, 0.02, 1e3)


@pytest.fixture(scope="module")
def E():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def probs_of(n, seed=1):
    return np.random.default_rng(seed).uniform(0.1, 1.0, n).astype(F)


def host_redraw(hs, st, seed, call, sg):
    out = st.copy()
    hs.hostsim_pf_redraw(_p(out), len(out), seed, call, *sg)
    return out


def host_noise(hs, st, seed, call, sp, sr):
    out = st.copy()
    org = np.zeros((len(st), 6), F)
    hs.hostsim_pf_noise(_p(out), len(out), seed, call, _p(np.array(sp, F)), _p(np.array(sr, F)), _p(org))
    return out, org


def check_redraw(got, want, base):
    for f in ("pos", "rot", "odom_err_integ_lin", "odom_err_integ_ang"):
        assert got[f].tobytes() == base[f].tobytes(), f
    for f in ("noise_ll", "noise_la", "noise_aa", "noise_al"):
        w = want[f].astype(np.float64)
        d = np.abs(got[f].astype(np.float64) - w)
        assert (d <= ORG_REL * np.abs(w) + ulp(want[f])).all(), (f, d.max())


def check_noise(got, want, org):
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        assert (got[f] == 0).all()
    for f, cols in (("pos", (0, 1, 2)), ("odom_err_integ_lin", (0, 1, 2)), ("odom_err_integ_ang", (3, 4, 5))):
        for a, k in enumerate(cols):
            d = np.abs(got[f][:, a].astype(np.float64) - want[f][:, a])
            assert (d <= ulp(want[f][:, a]) + ORG_REL * np.abs(org[:, k])).all(), (f, a, d.max())
    rn = np.linalg.norm(want["rot"].astype(np.float64), axis=1, keepdims=True)
    d = np.abs(got["rot"].astype(np.float64) - want["rot"])
    assert (d <= NOISE_ROT_BAR * rn + ulp(want["rot"])).all(), d.max()


@pytest.mark.parametrize("n", SIZES)
def test_redraw_against_host_and_call_count(E, hs, n):  # noqa: F811
    st, pr = states(n, 21), probs_of(n)
    e = E.Engine((0,))
    e.particles_set(st, pr)
    cur = st
    for call in (1, 2):
        e.particles_redraw_odom_noise(*SIG, seed=7)
        got, gp = e.particles_get()
        check_redraw(got, host_redraw(hs, cur, 7, call, SIG), cur)
        assert gp.tobytes() == pr.tobytes()
        cur = got
    e.particles_set(st, pr)   # particles_set keeps the count: the third call draws call 3's numbers
    e.particles_redraw_odom_noise(*SIG, seed=7)
    check_redraw(e.particles_get()[0], host_redraw(hs, st, 7, 3, SIG), st)
    e.close()


@pytest.mark.parametrize("n", [1000, 1 << 20])
def test_redraw_draws_are_the_host_recomputation(E, hs, n):  # noqa: F811
    """With every sigma 1.0 the redraw stores the device's standard normals themselves (float(double(z) * 1.0) == z):
    each equals the host's z, recomputed from the documented Philox layout, within the bar of logf / cosf / sinf only.
    The Philox words and the uniforms are exact integer and float arithmetic on both sides, so a single different
    word would put its two draws far outside this bar."""
    st, pr = states(n, 28), probs_of(n)
    e = E.Engine((0,))
    e.particles_set(st, pr)
    for call in (1, 2):
        e.particles_redraw_odom_noise(1.0, 1.0, 1.0, 1.0, seed=2 ** 63 + 5)
        got = e.particles_get()[0]
        dev = np.stack([got["noise_ll"], got["noise_la"], got["noise_aa"], got["noise_al"]], 1).astype(np.float64)
        want = host_z(hs, n, 2 ** 63 + 5, call)
        d = np.abs(dev - want)
        assert (d <= Z_REL * np.abs(want) + ulp(want)).all(), (call, d.max())
    e.close()


@pytest.mark.parametrize("n", SIZES)
def test_noise_against_host_unnormalised(E, hs, n):  # noqa: F811
    st, pr = states(n, 22), probs_of(n)
    sp, sr = (0.5, 0.5, 0.1), (0.05, 0.05, 0.3)
    e = E.Engine((0,))
    e.particles_set(st, pr)
    e.particles_redraw_odom_noise(*SIG, seed=3)   # the node's order: the redraw, then the expansion noise discards it
    cur = e.particles_get()[0]
    e.particles_noise(sp, sr, seed=3)
    got, gp = e.particles_get()
    want, org = host_noise(hs, cur, 3, 1, sp, sr)
    check_noise(got, want, org)
    assert gp.tobytes() == pr.tobytes()
    assert np.abs(np.linalg.norm(got["rot"].astype(np.float64), axis=1) - 1).max() > 0.05
    e.particles_noise((0, 0, 0), (0, 0, 0), seed=3)   # zero sigma: exact (noise quaternion (0, 0, 0, 1)), call 2
    z = e.particles_get()[0]
    want0, _ = host_noise(hs, got, 3, 2, (0, 0, 0), (0, 0, 0))
    assert z.tobytes() == want0.tobytes()
    e.close()


def test_same_seed_byte_identical_and_calls_advance(E):
    st, pr = states(5000, 23), probs_of(5000)
    outs = []
    for _ in range(2):
        e = E.Engine((0,))
        e.particles_set(st, pr)
        snaps = []
        for _ in range(2):
            e.particles_redraw_odom_noise(*SIG, seed=11)
            e.particles_noise((0.1, 0.1, 0.1), (0.1, 0.1, 0.1), seed=11)
            snaps.append(e.particles_get()[0].tobytes())
        e.particles_redraw_odom_noise(*SIG, seed=11)
        snaps.append(e.particles_get()[0].tobytes())
        outs.append(snaps)
        e.close()
    assert outs[0] == outs[1]
    assert outs[0][0] != outs[0][1]


def imu_eps(lik, var):
    """eps_i of the module docstring where lik_i > 0, with x_i = diff_i^2 / sq2 = -ln(lik_i / a); 0 where lik_i == 0."""
    sg = np.float64(F(var))
    a = float(F(1.0 / np.sqrt(2.0 * np.pi * sg * sg)))
    pos = lik > 0
    x = np.zeros(len(lik))
    x[pos] = np.abs(np.log(lik[pos].astype(np.float64) / a))
    return np.where(pos, ((2 * LIBM["acosf"] + 2) * x + LIBM["expf"] + 2) * R, 0.0)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("acc,var", [((0.1, -0.05, 0.98), 0.3), ((0.0, 0.0, 9.81), 0.05)])
def test_imu_update_against_host(E, hs, n, acc, var):  # noqa: F811
    st = states(n, 24, scale=(0.98, 1.02))
    st["rot"][:, :2] *= 0.15   # tilts mostly within the likelihood's reach; at var 0.05 the widest underflow to 0
    pr = probs_of(n, 2)
    lik, _ = host_imu(hs, st, acc, var)
    assert np.isfinite(lik).all() and (lik > 0).any()
    e = E.Engine((0,))
    e.particles_set(st, pr)
    summ = e.particles_imu_update(acc, var)
    got_s, got_p = e.particles_get()
    assert got_s.tobytes() == st.tobytes()
    # w_i within eps_i w_i plus an absolute DENORM for results in or below the subnormal range (expf's ulps there are
    # absolute: 3 ulps of 2^-149 each side); the sum, its float rounding and the division as in the module docstring
    w = (pr * lik).astype(F).astype(np.float64)
    dw = imu_eps(lik, var) * w + pr.astype(np.float64) * DENORM
    S = w.sum()
    dS = dw.sum() + 1e-12 * S
    assert summ["kept"] == 1 and summ["match_ratio_min"] == 0.0 and summ["match_ratio_max"] == 0.0
    assert abs(summ["weight_sum"] - S) <= dS + float(ulp(F(S)))
    p = w / S
    d = np.abs(got_p.astype(np.float64) - p)
    assert (d <= (dw + p * dS) / S * 1.01 + 2 * R * p + ulp(F(p))).all(), d.max()
    nz = p > 0
    H = -(p[nz] * np.log(p[nz])).sum()
    bar = (d[nz] * (np.abs(np.log(p[nz])) + 1)).sum() + (LIBM["logf"] * p[nz] * ulp(np.log(p[nz]).astype(F))).sum() + 1e-6 * H
    assert abs(summ["entropy"] - H) <= bar + float(ulp(F(H)))
    assert got_p[summ["max_index"]] == got_p.max() and summ["max_index"] == int(np.argmax(got_p))
    e.close()


def test_imu_nan_and_all_zero_keep_the_prior(E, hs):  # noqa: F811
    e = E.Engine((0,))
    for s0, acc in nan_states(hs):
        st = states(4096, 25)
        st[1234] = s0
        pr = probs_of(4096, 3)
        lik, _ = host_imu(hs, st, acc, 0.1)
        assert np.isnan(lik[1234])
        e.particles_set(st, pr)
        summ = e.particles_imu_update(acc, 0.1)
        assert summ["kept"] == 0 and np.isnan(summ["weight_sum"]) and summ["entropy"] == 0
        assert e.particles_get()[1].tobytes() == pr.tobytes()
    st = np.zeros(300, synth.STATE)
    st["rot"] = [1.0, 0.0, 0.0, 0.0]
    pr = np.full(300, 1 / 300, F)
    e.particles_set(st, pr)
    summ = e.particles_imu_update((0, 0, 1), 0.01)
    assert summ["kept"] == 0 and summ["weight_sum"] == 0
    assert e.particles_get()[1].tobytes() == pr.tobytes()
    e.close()


def test_error_codes(E):
    L = E.load_library()
    e = E.Engine((0,))
    acc = np.array([0, 0, 1], F)
    s3 = np.zeros(3, F)
    summ = E.UpdateSummary()
    # no resident set yet
    assert L.mcl3dl_particles_redraw_odom_noise(e.h, 0.1, 0.1, 0.1, 0.1, 1) == -1
    assert L.mcl3dl_particles_noise(e.h, _p(s3), _p(s3), 1) == -1
    assert L.mcl3dl_particles_imu_update(e.h, _p(acc), 0.1, C.byref(summ)) == -1
    # null engine
    assert L.mcl3dl_particles_redraw_odom_noise(None, 0.1, 0.1, 0.1, 0.1, 1) == -1
    assert L.mcl3dl_particles_noise(None, _p(s3), _p(s3), 1) == -1
    assert L.mcl3dl_particles_imu_update(None, _p(acc), 0.1, C.byref(summ)) == -1
    st, pr = states(10, 26), probs_of(10)
    e.particles_set(st, pr)
    for bad in (-0.1, float("nan"), float("inf")):
        for k in range(4):
            sg = [0.1] * 4
            sg[k] = bad
            assert L.mcl3dl_particles_redraw_odom_noise(e.h, *sg, 1) == -1
        for k in range(6):
            v = np.full(6, 0.1, F)
            v[k] = bad
            assert L.mcl3dl_particles_noise(e.h, _p(v[:3].copy()), _p(v[3:].copy()), 1) == -1
    for bad in (0.0, -1.0, float("nan"), float("inf"), 1e-50, 1e300):   # float(acc_var) must be finite and positive
        assert L.mcl3dl_particles_imu_update(e.h, _p(acc), bad, C.byref(summ)) == -1
    assert L.mcl3dl_particles_noise(e.h, None, _p(s3), 1) == -1
    assert L.mcl3dl_particles_imu_update(e.h, None, 0.1, C.byref(summ)) == -1
    assert L.mcl3dl_particles_imu_update(e.h, _p(acc), 0.1, None) == -1
    # nothing above touched the set
    gs, gp = e.particles_get()
    assert gs.tobytes() == st.tobytes() and gp.tobytes() == pr.tobytes()
    e.close()


def test_redraw_then_cycle_equals_uploaded_set(E):
    """After a redraw, predict / resample / estimate give the same bytes as the same set uploaded with particles_set."""
    n = 70_000
    st, pr = states(n, 27, scale=(0.99, 1.01)), probs_of(n, 4)
    a = E.Engine((0,))
    a.particles_set(st, pr)
    a.particles_redraw_odom_noise(*SIG[:3], 0.01, seed=5)
    mid = a.particles_get()
    b = E.Engine((0,))
    b.particles_set(*mid)
    prev = np.zeros(1, synth.POSE)
    prev["qw"] = 1
    cur = prev.copy()
    cur["px"], cur["qz"], cur["qw"] = 0.3, np.sin(0.05), np.cos(0.05)
    outs = []
    for e in (a, b):
        e.particles_predict(prev, cur, 0.1, 10.0, 10.0)
        e.particles_resample((0.05, 0.05, 0.05), (0.01, 0.01, 0.02), 0.37, 99)
        est = e.particles_estimate(cur, 1.0, 1.0)
        s, p = e.particles_get()
        outs.append((s.tobytes(), p.tobytes(), est["mean_biased"].tobytes(), est["cov"].tobytes(), est["max_index"]))
        e.close()
    assert outs[0] == outs[1]


@pytest.mark.parametrize("args,resets", [(["300", "1.5", "4"], 4), (["300", "0", "4"], 0), (["3000", "1.5", "3"], 3)])
def test_adapter_parity(args, resets):
    """ParticleFilterB200's resident cycles with IMU updates between clouds, the odometry-noise redraw and expansion
    resetting (triggered on every cycle by match_ratio_thresh 1.5, never by the node's default 0) against the reference
    filter fed the same draws (oracle/pf_events_parity_test.cpp)."""
    if not os.path.exists(PARITY):
        pytest.skip("oracle/_ref/pf_events_parity_test not built (needs a checkout of the reference at build time)")
    r = subprocess.run([PARITY] + args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "PF EVENTS PARITY OK" in r.stdout
    assert "expansion resets: %d" % resets in r.stdout
