"""The landmark update, the odometry-error reset and the published particle poses without a GPU: the device functions of
mcl_3dl_b200/csrc/pf_funcs.cuh, compiled for the host by tests/hostsim/pf_landmark_hostsim.cpp, equal both CPU checkers
bit for bit — the port (oracle/pf_landmark_oracle.cpp) and the reference tier (oracle/pf_landmark_ref_driver.cpp:
cbLandmark's measure_func with the reference's State6DOF::operator-, Quat::inv and Quat::getRPY inside
pf::ParticleFilter::measure, the node's reset lambda through pf::ParticleFilter::predict, publishParticles' normalize).
All three call the host's libm.  The quadratic form's fixed order is also held to the exact value of -0.5 x^T S x."""
import ctypes as C
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from mcl_3dl_b200 import engine, synth
from oracle import pf_landmark_checker as lc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "pf_landmark_hostsim.cpp")
F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pflhs") / "libpflhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_pf_landmark.argtypes = [vp, sz, vp, C.c_float, vp, vp, vp]
    L.hostsim_pf_landmark.restype = None
    L.hostsim_pf_nd6_exponent.argtypes = [vp, vp]
    L.hostsim_pf_nd6_exponent.restype = C.c_float
    L.hostsim_pf_reset_odom_err.argtypes = [vp, sz]
    L.hostsim_pf_reset_odom_err.restype = None
    L.hostsim_pf_poses.argtypes = [vp, sz, vp]
    L.hostsim_pf_poses.restype = None
    return L


@pytest.fixture(scope="module")
def port():
    lc.build("port")
    return lc.PfLandmarkChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not lc.build("reference"):
        pytest.skip("reference checker not built (no reference checkout)")
    return lc.PfLandmarkChecker("reference")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def states(n, seed, scale=(0.9, 1.1), spread=0.3):
    """Positions around the origin, non-unit rotations (half of them with w < 0), every other field nonzero."""
    rng = np.random.default_rng(seed)
    st = np.zeros(n, synth.STATE)
    st["pos"] = rng.normal(0, spread, (n, 3))
    q = rng.normal(0, 1, (n, 4))
    q[:, :3] *= 0.3 * spread
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[::2] *= -1
    st["rot"] = q * rng.uniform(*scale, (n, 1))
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        st[f] = rng.normal(0, 0.1, n)
    st["odom_err_integ_lin"] = rng.normal(0, 0.2, (n, 3))
    st["odom_err_integ_ang"] = rng.normal(0, 0.2, (n, 3))
    st["odom_err_integ_lin"][::3, 1] = -0.0
    return st


def covariance(seed, scales=(0.5, 0.5, 0.3, 0.3, 0.3, 0.4), symmetric=True):
    """A 6x6 covariance as the message's 36 doubles (row-major as written, read column-major by cbLandmark)."""
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 1, (6, 6)) * 0.3 + np.eye(6)
    c = (a @ a.T) * np.outer(scales, scales)
    if not symmetric:
        c = c + np.triu(np.full((6, 6), 0.01 * min(scales) ** 2), 1)
    return c.reshape(36)


def measured_pose(pos, rot):
    m = np.zeros(1, synth.POSE)
    m["px"], m["py"], m["pz"] = pos
    m["qx"], m["qy"], m["qz"], m["qw"] = rot
    return m


def same(a, b):
    """Bit for bit, except that a NaN only has to be a NaN (its sign and payload depend on the compiler's negation)."""
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and a[~na].tobytes() == b[~nb].tobytes()


def host_landmark(hs, st, measured, nd_a, sigma_inv, with_x=False):
    """The host build's likelihoods (and, with_x, each particle's x [n, 6])."""
    lik = np.zeros(len(st), F)
    x = np.zeros((len(st), 6), F) if with_x else None
    m = lc.measured7(measured)
    hs.hostsim_pf_landmark(_p(np.ascontiguousarray(st)), len(st), _p(m), nd_a,
                           _p(np.ascontiguousarray(sigma_inv, dtype=F).reshape(36)), _p(lik), lc._ptr(x))
    return (lik, x) if with_x else lik


def check_landmark(hs, port, ref, st, probs, measured, nd_a, sigma_inv):
    lik = host_landmark(hs, st, measured, nd_a, sigma_inv)
    p_port, l_port, k_port, s_port, e_port = port.landmark(st, probs, measured, nd_a, sigma_inv)
    p_ref, l_ref, k_ref, s_ref, e_ref = ref.landmark(st, probs, measured, nd_a, sigma_inv)
    assert same(lik, l_port) and same(lik, l_ref)
    assert p_port.tobytes() == p_ref.tobytes() and k_port == k_ref
    assert same([s_port, e_port], [s_ref, e_ref])
    if not k_ref:
        assert p_ref.tobytes() == np.asarray(probs, F).tobytes()   # the prior, untouched
    return lik, k_ref


@pytest.mark.parametrize("n", [1, 1000])
@pytest.mark.parametrize("cov_seed,symmetric", [(1, True), (2, True), (3, False)])
def test_landmark_equals_both_checkers(hs, port, ref, n, cov_seed, symmetric):
    st = states(n, 5)
    probs = np.random.default_rng(6).uniform(0.1, 1.0, n).astype(F)
    nd_a, si = engine.landmark_nd(covariance(cov_seed, symmetric=symmetric))
    for pos, rot in [((0.0, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0)), ((0.3, -0.2, 0.1), (0.05, -0.02, 0.1, 0.99)),
                     ((-0.5, 0.4, 0.0), (0.0, 0.0, -0.3, -1.05))]:   # the last one un-normalised, w < 0
        lik, kept = check_landmark(hs, port, ref, st, probs, measured_pose(pos, rot), nd_a, si)
        assert kept and np.isfinite(lik).all() and (lik > 0).any()


def test_landmark_identity_rotations_and_measured_at_a_particle(hs, port, ref):
    st = np.zeros(4, synth.STATE)
    st["rot"] = [[0, 0, 0, 1], [0, 0, 0, -1], [0, 0, 0, 1.2], [0, 0, 0, -0.8]]
    nd_a, si = engine.landmark_nd(covariance(4))
    lik, kept = check_landmark(hs, port, ref, st, np.full(4, 0.25, F), measured_pose((0, 0, 0), (0, 0, 0, 1)), nd_a, si)
    # x = 0 (a w < 0 rotation has roll = yaw = atan2(0, 1) = 0 and pitch asin(0)): likelihood = a * expf(0) = a
    assert kept and (lik == F(nd_a)).all()


def test_landmark_pitch_clamp_and_angle_wraps(hs, port, ref):
    """Pitch differences at +-pi/2 where getRPY's t2 clamps to +-1, roll and yaw differences on both sides of +-pi."""
    c, s = np.cos(np.pi / 4), np.sin(np.pi / 4)
    rots = [[0, s, 0, c], [0, -s, 0, c]]
    rots += [list(np.array(r) * 1.01) for r in rots]   # |t2| = 1.0201 before the clamp
    for ang in (np.pi - 1e-3, np.pi + 1e-3, -np.pi + 1e-3, np.pi):
        rots += [[np.sin(ang / 2), 0, 0, np.cos(ang / 2)], [0, 0, np.sin(ang / 2), np.cos(ang / 2)]]
    st = np.zeros(len(rots), synth.STATE)
    st["rot"] = rots
    st["pos"] = np.random.default_rng(7).normal(0, 0.2, (len(rots), 3))
    nd_a, si = engine.landmark_nd(covariance(5, scales=(1, 1, 1, 2, 2, 2)))
    probs = np.full(len(rots), 1 / len(rots), F)
    for mrot in [(0, 0, 0, 1), (0, 0, 0, 0.97)]:
        lik, kept = check_landmark(hs, port, ref, st, probs, measured_pose((0, 0, 0), mrot), nd_a, si)
        assert kept and np.isfinite(lik).all()


def test_landmark_zero_priors_far_landmark_and_nan(hs, port, ref):
    st = states(64, 8)
    nd_a, si = engine.landmark_nd(covariance(6))
    probs = np.random.default_rng(9).uniform(0.1, 1.0, 64).astype(F)
    probs[::4] = 0
    lik, kept = check_landmark(hs, port, ref, st, probs, measured_pose((0.1, 0, 0), (0, 0, 0, 1)), nd_a, si)
    assert kept
    post = port.landmark(st, probs, measured_pose((0.1, 0, 0), (0, 0, 0, 1)), nd_a, si)[0]
    assert (post[::4] == 0).all()
    # a landmark far from every particle: every weight underflows to 0, the update is discarded
    lik, kept = check_landmark(hs, port, ref, st, probs, measured_pose((1e3, -1e3, 50), (0, 0, 0, 1)), nd_a, si)
    assert (lik == 0).all() and not kept
    # one NaN rotation: its likelihood is NaN and the whole update is discarded
    st[17]["rot"] = [np.nan, 0, 0, 1]
    lik, kept = check_landmark(hs, port, ref, st, probs, measured_pose((0.1, 0, 0), (0, 0, 0, 1)), nd_a, si)
    assert np.isnan(lik[17]) and np.isfinite(np.delete(lik, 17)).all() and not kept


def test_landmark_near_singular_covariance(hs, port, ref):
    """Eigenvalues from 1e-6 to 1: sigma_inv entries near 1e6, still finite."""
    rng = np.random.default_rng(10)
    qm, _ = np.linalg.qr(rng.normal(0, 1, (6, 6)))
    cov = (qm * np.array([1e-6, 1e-3, 0.1, 0.5, 1.0, 1.0])) @ qm.T
    nd_a, si = engine.landmark_nd(cov.reshape(36))
    assert np.isfinite(si).all() and np.abs(si).max() > 1e5
    st = states(300, 11, spread=1e-3)
    probs = np.full(300, 1 / 300, F)
    check_landmark(hs, port, ref, st, probs, measured_pose((0, 0, 0), (0, 0, 0, 1)), nd_a, si)


def test_landmark_nd_helper():
    cov = covariance(12, symmetric=False)
    nd_a, si = engine.landmark_nd(cov)
    sigma = cov.reshape(6, 6, order="F").astype(F).astype(np.float64)   # column-major: the array's transpose
    assert np.allclose(si.astype(np.float64) @ sigma, np.eye(6), atol=1e-4)
    want = 1.0 / ((2 * np.pi) ** 3 * np.sqrt(np.linalg.det(sigma)))
    assert abs(nd_a - want) <= 1e-5 * want


def exact_exponent(x, S):
    fx = [Fraction(float(v)) for v in x]
    fS = [[Fraction(float(S[j, k])) for k in range(6)] for j in range(6)]
    return -Fraction(1, 2) * sum(fx[j] * fS[j][k] * fx[k] for j in range(6) for k in range(6))


def test_quadratic_form_order_within_gamma12(hs):
    """The fixed order's value is within gamma_12 * 0.5 * sum_jk |x_j S_jk x_k| of the exact -0.5 x^T S x: twelve
    roundings at most lie on any term's path (the product with S, five sums, the product with x, five sums).  The bound
    holds for every summation order, so it also bounds the distance to the order Eigen would take."""
    u = 2.0 ** -24
    g12 = 12 * u / (1 - 12 * u)
    rng = np.random.default_rng(13)
    worst = 0.0
    for t in range(300):
        x = (rng.normal(0, 1, 6) * 10.0 ** rng.uniform(-3, 2, 6)).astype(F)
        if t % 3 == 0:
            a = rng.normal(0, 1, (6, 6))
            S = (a @ a.T).astype(F)
        else:
            S = (rng.normal(0, 1, (6, 6)) * 10.0 ** rng.uniform(-2, 4)).astype(F)
        got = Fraction(float(hs.hostsim_pf_nd6_exponent(_p(x), _p(np.ascontiguousarray(S.reshape(36))))))
        want = exact_exponent(x, S)
        mag = Fraction(1, 2) * sum(abs(Fraction(float(x[j])) * Fraction(float(S[j, k])) * Fraction(float(x[k])))
                                   for j in range(6) for k in range(6))
        err = abs(got - want)
        assert err <= Fraction(g12) * mag, (t, float(err), float(mag))
        worst = max(worst, float(err / mag) if mag else 0.0)
    assert worst > 0   # the bound is exercised, not trivially met by exact results


def test_reset_and_poses_equal_both_checkers(hs, port, ref):
    st = states(1000, 14, scale=(0.5, 2.0))
    st["rot"][3] = [0, 0, 0, -1]
    st["rot"][4] = [0, 0, 0, 1e-3]
    got = st.copy()
    hs.hostsim_pf_reset_odom_err(_p(got), len(got))
    assert got.tobytes() == port.reset_odom_err(st).tobytes() == ref.reset_odom_err(st).tobytes()
    assert (got["odom_err_integ_lin"] == 0).all() and not np.signbit(got["odom_err_integ_lin"]).any()
    assert (got["odom_err_integ_ang"] == 0).all() and not np.signbit(got["odom_err_integ_ang"]).any()
    for f in ("pos", "rot", "noise_ll", "noise_la", "noise_al", "noise_aa"):
        assert got[f].tobytes() == st[f].tobytes()
    poses = np.zeros(len(st), synth.POSE)
    hs.hostsim_pf_poses(_p(st), len(st), _p(poses))
    assert poses.tobytes() == port.poses(st).tobytes() == ref.poses(st).tobytes()
    assert (poses["_pad"] == 0).all()
    n = np.sqrt(sum(poses[k].astype(np.float64) ** 2 for k in ("qx", "qy", "qz", "qw")))
    assert np.abs(n - 1).max() < 1e-6
    assert poses["px"].tobytes() == st["pos"][:, 0].copy().tobytes()


def test_new_entry_points_reject_a_null_engine():
    L = engine.load_library()
    prm = engine.LandmarkParams()
    summ = engine.UpdateSummary()
    out = np.zeros(4, synth.POSE)
    assert L.mcl3dl_particles_landmark_update(None, C.byref(prm), C.byref(summ)) == -1
    assert L.mcl3dl_particles_reset_odom_err_integ(None) == -1
    assert L.mcl3dl_particles_get_poses(None, _p(out), 4) == -1
