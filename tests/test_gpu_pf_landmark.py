"""The landmark update, the odometry-error reset and the published particle poses on the resident set (H100) against the
host build of their device functions (tests/hostsim/pf_landmark_hostsim.cpp), which tests/test_pf_landmark_on_host.py
holds bit for bit to the port and reference checkers.

Bars, derived as in tests/test_gpu_pf_events.py (LIBM, R there).  Everything in the landmark likelihood is explicit
round-to-nearest arithmetic except atan2f (roll, yaw), asinf (pitch) and expf:
  - x: the position differences are exact; roll and yaw within LIBM["atan2f"] ulp(x_j), pitch within LIBM["asinf"] ulp;
  - q = -0.5 x^T S x: the same float order on both sides, so the two values differ by at most the first-order change
    sum_j |g_j| dx_j (g = 0.5 (S + S^T) x) plus both sides' rounding, 2 gamma_12 * 0.5 sum_jk |x_j S_jk x_k|;
  - the likelihood a expf(q): |dq| + LIBM["expf"] + 1 relative ulps, the prior's product one more: eps_i on w_i, plus
    prior_i * a * 4 2^-149 absolute where expf's result is subnormal or underflows.
With dw_i that bound and dS = sum dw_i, the weight sum, the posteriors and the entropy follow the IMU update's bars.
The reset and the poses are exact arithmetic (the square root and the double division are correctly rounded), so they
are compared byte for byte.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from test_pf_landmark_on_host import covariance, host_landmark, hs, measured_pose, states  # noqa: F401
from test_gpu_pf_exact import LIBM, R, ulp

pytestmark = pytest.mark.gpu

F = np.float32
DENORM = 4 * 2.0 ** -149
G12 = 12 * 2.0 ** -24 / (1 - 12 * 2.0 ** -24)
PARITY = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "landmark_parity_test")
SIZES = [1, 1000, 65_536, 1 << 20]


@pytest.fixture(scope="module")
def E():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def probs_of(n, seed=1):
    return np.random.default_rng(seed).uniform(0.1, 1.0, n).astype(F)


def lik_eps(x, S):
    """The relative bar eps_i on each particle's likelihood (module docstring)."""
    x64, S64 = x.astype(np.float64), S.astype(np.float64)
    dx = np.zeros_like(x64)
    dx[:, 3] = LIBM["atan2f"] * ulp(x[:, 3])
    dx[:, 4] = LIBM["asinf"] * ulp(x[:, 4])
    dx[:, 5] = LIBM["atan2f"] * ulp(x[:, 5])
    g = 0.5 * x64 @ (S64 + S64.T)
    mag = 0.5 * np.einsum("ij,jk,ik->i", np.abs(x64), np.abs(S64), np.abs(x64))
    dq = (np.abs(g) * dx).sum(1) * 1.01 + (np.abs(S64).sum() * (dx ** 2).sum(1)) + 2 * G12 * mag
    return dq * 1.01 + (LIBM["expf"] + 2) * R


def check_update(summ, got_p, pr, lik, x, S, nd_a):
    w = (pr * lik).astype(F).astype(np.float64)
    dw = lik_eps(x, S) * w + pr.astype(np.float64) * max(float(nd_a), 1.0) * DENORM
    S_ = w.sum()
    dS = dw.sum() + 1e-12 * S_
    assert summ["kept"] == 1 and summ["match_ratio_min"] == 0.0 and summ["match_ratio_max"] == 0.0
    assert abs(summ["weight_sum"] - S_) <= dS + float(ulp(F(S_)))
    p = w / S_
    d = np.abs(got_p.astype(np.float64) - p)
    assert (d <= (dw + p * dS) / S_ * 1.01 + 2 * R * p + ulp(F(p))).all(), d.max()
    nz = p > 0
    H = -(p[nz] * np.log(p[nz])).sum()
    bar = (d[nz] * (np.abs(np.log(p[nz])) + 1)).sum() + (LIBM["logf"] * p[nz] * ulp(np.log(p[nz]).astype(F))).sum() + 1e-6 * H
    assert abs(summ["entropy"] - H) <= bar + float(ulp(F(H)))
    assert got_p[summ["max_index"]] == got_p.max() and summ["max_index"] == int(np.argmax(got_p))


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("case", ["near", "rotated"])
def test_landmark_update_against_host(E, hs, n, case):  # noqa: F811
    st, pr = states(n, 31), probs_of(n, 2)
    pr[1::7] = 0
    if case == "near":
        m, cov = measured_pose((0.1, -0.05, 0.02), (0.02, -0.01, 0.05, 0.998)), covariance(1)
    else:   # an un-normalised measured rotation with w < 0, a non-symmetric covariance
        m, cov = measured_pose((-0.2, 0.1, 0.0), (0.0, 0.05, -0.2, -1.03)), covariance(3, symmetric=False)
    nd_a, si = E.landmark_nd(cov)
    lik, x = host_landmark(hs, st, m, nd_a, si, with_x=True)
    assert np.isfinite(lik).all() and (pr * lik > 0).any()
    e = E.Engine((0,))
    e.particles_set(st, pr)
    summ = e.particles_landmark_update(m, nd_a, si)
    got_s, got_p = e.particles_get()
    assert got_s.tobytes() == st.tobytes()   # the states never change
    check_update(summ, got_p, pr, lik, x, si, nd_a)
    assert (got_p[1::7] == 0).all()
    e.close()


def test_landmark_nan_and_far_keep_the_prior(E, hs):  # noqa: F811
    e = E.Engine((0,))
    nd_a, si = E.landmark_nd(covariance(6))
    st, pr = states(4096, 32), probs_of(4096, 3)
    e.particles_set(st, pr)
    summ = e.particles_landmark_update(measured_pose((1e3, -1e3, 50), (0, 0, 0, 1)), nd_a, si)   # every weight is 0
    assert host_landmark(hs, st, measured_pose((1e3, -1e3, 50), (0, 0, 0, 1)), nd_a, si).max() == 0
    assert summ["kept"] == 0 and summ["weight_sum"] == 0 and summ["entropy"] == 0
    assert e.particles_get()[1].tobytes() == pr.tobytes()
    st[1234]["rot"] = [np.nan, 0, 0, 1]
    e.particles_set(st, pr)
    summ = e.particles_landmark_update(measured_pose((0.1, 0, 0), (0, 0, 0, 1)), nd_a, si)
    assert summ["kept"] == 0 and np.isnan(summ["weight_sum"]) and summ["entropy"] == 0
    gs, gp = e.particles_get()
    assert gp.tobytes() == pr.tobytes() and gs.tobytes() == st.tobytes()
    e.close()


@pytest.mark.parametrize("n", SIZES)
def test_reset_and_poses_exact(E, hs, n):  # noqa: F811
    st, pr = states(n, 33, scale=(0.5, 2.0)), probs_of(n, 4)
    e = E.Engine((0,))
    e.particles_set(st, pr)
    poses = e.particles_get_poses()
    want = np.zeros(n, synth.POSE)
    hs.hostsim_pf_poses(_p(st), n, _p(want))
    assert poses.tobytes() == want.tobytes()
    gs, gp = e.particles_get()
    assert gs.tobytes() == st.tobytes() and gp.tobytes() == pr.tobytes()   # get_poses reads the set only
    e.particles_reset_odom_err_integ()
    gs, gp = e.particles_get()
    want_s = st.copy()
    hs.hostsim_pf_reset_odom_err(_p(want_s), n)
    assert gs.tobytes() == want_s.tobytes() and gp.tobytes() == pr.tobytes()
    assert not np.signbit(gs["odom_err_integ_lin"]).any() and not np.signbit(gs["odom_err_integ_ang"]).any()
    e.close()


def test_poses_after_resize_and_update(E, hs):  # noqa: F811
    """get_poses follows the resident count through a resize and reads the set a landmark update left."""
    st, pr = states(5000, 34), probs_of(5000, 5)
    e = E.Engine((0,))
    e.particles_set(st, pr)
    e.particles_resize(3000)
    nd_a, si = E.landmark_nd(covariance(2))
    e.particles_landmark_update(measured_pose((0, 0, 0), (0, 0, 0, 1)), nd_a, si)
    gs, _ = e.particles_get()
    want = np.zeros(3000, synth.POSE)
    hs.hostsim_pf_poses(_p(gs), 3000, _p(want))
    assert e.particles_get_poses().tobytes() == want.tobytes()
    e.close()


def test_error_codes(E):
    L = E.load_library()
    nd_a, si = E.landmark_nd(covariance(1))
    prm = E.LandmarkParams()
    prm.measured[7] = 1.0
    prm.nd_a = float(nd_a)
    C.memmove(prm.sigma_inv, np.ascontiguousarray(si, F).ctypes.data, 144)
    summ = E.UpdateSummary()
    out = np.zeros(10, synth.POSE)
    e = E.Engine((0,))
    # no resident set yet
    assert L.mcl3dl_particles_landmark_update(e.h, C.byref(prm), C.byref(summ)) == -1
    assert L.mcl3dl_particles_reset_odom_err_integ(e.h) == -1
    assert L.mcl3dl_particles_get_poses(e.h, _p(out), 10) == -1
    # null engine
    assert L.mcl3dl_particles_landmark_update(None, C.byref(prm), C.byref(summ)) == -1
    assert L.mcl3dl_particles_reset_odom_err_integ(None) == -1
    assert L.mcl3dl_particles_get_poses(None, _p(out), 10) == -1
    st, pr = states(10, 35), probs_of(10)
    e.particles_set(st, pr)
    assert L.mcl3dl_particles_landmark_update(e.h, None, C.byref(summ)) == -1
    assert L.mcl3dl_particles_landmark_update(e.h, C.byref(prm), None) == -1
    assert L.mcl3dl_particles_get_poses(e.h, None, 10) == -1
    for n in (9, 11, 0):   # the count must be the resident count
        assert L.mcl3dl_particles_get_poses(e.h, _p(np.zeros(12, synth.POSE)), n) == -1
    for bad in (float("nan"), float("inf"), -float("inf")):
        for k in (0, 1, 2, 4, 5, 6, 7):   # every pose value but _pad
            p2 = E.LandmarkParams.from_buffer_copy(prm)
            p2.measured[k] = bad
            assert L.mcl3dl_particles_landmark_update(e.h, C.byref(p2), C.byref(summ)) == -1
        p2 = E.LandmarkParams.from_buffer_copy(prm)
        p2.nd_a = bad
        assert L.mcl3dl_particles_landmark_update(e.h, C.byref(p2), C.byref(summ)) == -1
        for k in (0, 7, 35):
            p2 = E.LandmarkParams.from_buffer_copy(prm)
            p2.sigma_inv[k] = bad
            assert L.mcl3dl_particles_landmark_update(e.h, C.byref(p2), C.byref(summ)) == -1
    # nothing above touched the set
    gs, gp = e.particles_get()
    assert gs.tobytes() == st.tobytes() and gp.tobytes() == pr.tobytes()
    p2 = E.LandmarkParams.from_buffer_copy(prm)
    p2.measured[3] = float("nan")   # _pad is not read
    assert L.mcl3dl_particles_landmark_update(e.h, C.byref(p2), C.byref(summ)) == 0
    # a multi-device engine (two contexts on one GPU)
    two = E.Engine((0, 0))
    assert L.mcl3dl_particles_landmark_update(two.h, C.byref(prm), C.byref(summ)) == -1
    assert L.mcl3dl_particles_reset_odom_err_integ(two.h) == -1
    assert L.mcl3dl_particles_get_poses(two.h, _p(out), 10) == -1
    two.close()
    e.close()


def test_adapter_parity():
    """ParticleFilterB200 through the node's sequence (a resident cycle, cbLandmark with the reference's own
    NormalLikelihoodNd, a pose-jump reset, the published poses) against the reference filter
    (oracle/landmark_parity_test.cpp)."""
    if not os.path.exists(PARITY):
        pytest.skip("oracle/_ref/landmark_parity_test not built (needs a checkout of the reference at build time)")
    r = subprocess.run([PARITY, "3000", "3"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "LANDMARK PARITY OK" in r.stdout
