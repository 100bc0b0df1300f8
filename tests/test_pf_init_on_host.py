"""The initial seed of the resident set without a GPU: pf_init_state of mcl_3dl_b200/csrc/pf_funcs.cuh, compiled for the
host by tests/hostsim/pf_init_hostsim.cpp, equals both CPU checkers bit for bit given the same standard normals — the
port (oracle/pf_init_oracle.cpp) and the reference tier (oracle/pf_init_ref_driver.cpp: the reference's own
initUsingNoiseGenerator, generateNoise, setMean / getRPY, Quat(rpy) and MultivariateNoiseGenerator's mean_vec_ +
norm_transform_ * random).  The draws themselves are recomputed here from the counter layout include/mcl3dl_b200.h
documents (event word 3), with glibc's logf / cosf / sinf, which the host build calls too."""
import ctypes as C
import ctypes.util
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import engine, synth
from oracle import pf_init_checker as pic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "pf_init_hostsim.cpp")
F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("pfihs") / "libpfihs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hostsim_pf_init.argtypes = [C.c_size_t, C.c_int, vp, vp, vp, C.c_uint64, C.c_uint32, vp, vp, vp]
    L.hostsim_pf_init.restype = None
    return L


@pytest.fixture(scope="module")
def port():
    pic.build("port")
    return pic.PfInitChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not pic.build("reference"):
        pytest.skip("reference checker not built (no reference checkout)")
    return pic.PfInitChecker("reference")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host_init(hs, n, mean6, seed, call, sigma=None, T=None):
    """-> (states, probs, z) of the host build of mcl3dl_particles_init."""
    mean6 = np.ascontiguousarray(mean6, F)
    sg = np.zeros(6, F) if sigma is None else np.ascontiguousarray(sigma, F)
    t = np.zeros(36, F) if T is None else np.ascontiguousarray(T, F).reshape(36)
    st, pr, z = np.zeros(n, synth.STATE), np.zeros(n, F), np.zeros((n, 6), F)
    hs.hostsim_pf_init(n, int(T is not None), _p(mean6), _p(sg), _p(t), seed, call, _p(st), _p(pr), _p(z))
    return st, pr, z


# ------------------------------------------------------------------ the draws, recomputed from the documented layout
_M = C.CDLL(ctypes.util.find_library("m"))
for _f in ("logf", "cosf", "sinf"):
    getattr(_M, _f).argtypes = [C.c_float]
    getattr(_M, _f).restype = C.c_float


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


def init_z(seed, index, call):
    a, b = philox((index, call, 0, 3), seed), philox((index, call, 1, 3), seed)
    return np.array(box_muller(a[0], a[1]) + box_muller(a[2], a[3]) + box_muller(b[0], b[1]), F)


def pose7(pos, rpy):
    """x y z qx qy qz qw of a position and the unit quaternion of (roll, pitch, yaw), as float32."""
    r, p, y = (np.float64(v) / 2 for v in rpy)
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    q = [sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy]
    return np.array(list(pos) + q, F)


def check_tiers(hs, checkers, n, pose, seed, call, sigma=None, cov=None, T=None):
    """The host build against every checker tier, bit for bit; returns (states, probs, mean6, T)."""
    mean6 = checkers[0].mean(pose)
    for c in checkers[1:]:
        assert c.mean(pose).tobytes() == mean6.tobytes(), c.kind
    if cov is not None and T is None:
        T = engine.noise_transform(cov)
    st, pr, z = host_init(hs, n, mean6, seed, call, sigma=sigma, T=T)
    for i in range(min(n, 64)):
        assert z[i].tobytes() == init_z(seed, i, call).tobytes(), i
    assert np.all(pr == F(1.0 / n))
    for c in checkers:
        cs, cp = c.init(pose, z, sigma=sigma, norm_transform=T)
        assert cs.tobytes() == st.tobytes(), c.kind
        assert cp.tobytes() == pr.tobytes(), c.kind
    return st, pr, mean6, T


def tiers(port, request):
    out = [port]
    if pic.build("reference"):
        out.append(request.getfixturevalue("ref"))
    return out


def test_draws_use_their_own_event_word(hs):
    """event 3 is not resampling's (0) or the expansion noise's (2) stream of the same (seed, index, call)"""
    z = init_z(7, 5, 1)
    for ev in (0, 2):
        a, b = philox((5, 1, 0, ev), 7), philox((5, 1, 1, ev), 7)
        other = np.array(box_muller(a[0], a[1]) + box_muller(a[2], a[3]) + box_muller(b[0], b[1]), F)
        assert not np.array_equal(z, other)


@pytest.mark.parametrize("n", [1, 1000])
def test_diagonal_zero_sigmas_and_negative_zero_mean(hs, port, request, n):
    pose = np.array([-0.0, 2.5, -0.0, 0.0, 0.0, 0.0, 1.0], F)
    st, _, mean6, _ = check_tiers(hs, tiers(port, request), n, pose, 11, 1, sigma=np.zeros(6, F))
    # every component is the mean: pos keeps the sign of -0.0, the angular integral is rpy - rpy = +0
    assert np.signbit(st["pos"][:, 0]).all() and np.signbit(st["odom_err_integ_lin"][:, 2]).all()
    assert (st["pos"][:, 1] == F(2.5)).all()
    assert not np.signbit(st["odom_err_integ_ang"]).any() and (st["odom_err_integ_ang"] == 0).all()
    assert (st["rot"] == np.array([0, 0, 0, 1], F)).all()


@pytest.mark.parametrize("call", [1, 3])
def test_diagonal_configured_start(hs, port, request, call):
    """MCL3dlNode::configure's pf_->init(initial_pose, initial_pose_std): some sigmas 0, others not"""
    pose = pose7((1.5, -3.0, 0.2), (0.01, -0.02, 1.2))
    sigma = np.array([0.5, 0.5, 0.0, 0.0, 0.0, 0.2], F)
    st, _, mean6, _ = check_tiers(hs, tiers(port, request), 2000, pose, 0x5eed, call, sigma=sigma)
    assert (st["pos"][:, 2] == mean6[2]).all()
    # the reference quirk, kept: odom_err_integ_lin_ is the position, mean included
    assert st["odom_err_integ_lin"].tobytes() == st["pos"].tobytes()
    assert (st["odom_err_integ_ang"][:, :2] == 0).all()
    assert (st[["noise_ll", "noise_la", "noise_al", "noise_aa"]].tolist() == [(0, 0, 0, 0)] * len(st))


def rviz_cov():
    """RViz's 2-D pose estimate: x, y and yaw only; the rows (and columns) of z, roll and pitch are zero"""
    c = np.zeros((6, 6))
    c[0, 0], c[1, 1], c[5, 5] = 0.25, 0.25, 0.06853891945200942
    return c.reshape(36)


def test_multivariate_rviz_pose_estimate(hs, port, request):
    pose = pose7((4.0, -1.0, 0.0), (0.0, 0.0, 2.0))
    checkers = tiers(port, request)
    T = engine.noise_transform(rviz_cov())
    assert (T[2] == 0).all() and (T[3] == 0).all() and (T[4] == 0).all()
    if len(checkers) > 1:
        Tr = checkers[1].transform(rviz_cov())
        assert (Tr[2] == 0).all() and (Tr[3] == 0).all() and (Tr[4] == 0).all()
    st, _, mean6, _ = check_tiers(hs, checkers, 3000, pose, 99, 1, T=T)
    assert (st["pos"][:, 2] == mean6[2]).all()
    assert (st["odom_err_integ_ang"][:, :2] == 0).all()
    assert np.std(st["pos"][:, 0]) > 0.3 and np.std(st["odom_err_integ_ang"][:, 2]) > 0.1


def dense_cov(seed=3):
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 1, (6, 6))
    return (a @ a.T * 0.05 + np.eye(6) * 0.01).reshape(36)


def test_multivariate_dense_covariance(hs, port, request):
    pose = pose7((0.3, 0.2, 0.1), (0.2, -0.1, -0.7))
    checkers = tiers(port, request)
    check_tiers(hs, checkers, 4096, pose, 2 ** 63 + 12345, 2, cov=dense_cov())
    if len(checkers) > 1:   # the reference's own setCovariance (shim_mv's solver) through the same path
        check_tiers(hs, checkers, 500, pose, 5, 1, T=checkers[1].transform(dense_cov()))


def test_multivariate_reads_the_lower_triangle(hs, port, request):
    """cov(i, j) = covariance[j + i * 6] (row-major); the solver reads only the lower triangle"""
    c = dense_cov(8).reshape(6, 6)
    skew = c.copy()
    skew[np.triu_indices(6, 1)] += 0.3   # upper triangle changed only
    assert engine.noise_transform(skew).tobytes() == engine.noise_transform(c).tobytes()
    checkers = tiers(port, request)
    if len(checkers) > 1:
        assert checkers[1].transform(skew.reshape(36)).tobytes() == checkers[1].transform(c.reshape(36)).tobytes()
    # the transpose reads another lower triangle
    assert engine.noise_transform(skew.T).tobytes() != engine.noise_transform(c).tobytes()
    check_tiers(hs, checkers, 700, pose7((1, 1, 1), (0, 0, 0)), 21, 1, cov=skew.reshape(36))


@pytest.mark.parametrize("rpy", [(0.0, 0.0, 3.14159), (0.0, 0.0, -3.14159), (0.3, 1.5707, 0.2), (-0.1, -1.5707, -2.0),
                                 (3.1, 0.0, 0.0)])
@pytest.mark.parametrize("mv", [False, True])
def test_angles_near_the_wrap_and_the_pitch_pole(hs, port, request, rpy, mv):
    pose = pose7((0.0, 0.0, 0.0), rpy)
    if mv:
        st, _, mean6, _ = check_tiers(hs, tiers(port, request), 1500, pose, 17, 1, cov=dense_cov(4))
    else:
        st, _, mean6, _ = check_tiers(hs, tiers(port, request), 1500, pose, 17, 1, sigma=np.full(6, 0.3, F))
    # the angular integral is org - mean, not wrapped: near +-pi it reaches past pi
    assert np.isfinite(st["odom_err_integ_ang"]).all() and np.isfinite(st["rot"]).all()


def test_n_one_and_probability_rule(hs, port, request):
    for n in (1, 3, 7, 65537):
        _, pr, _ = host_init(hs, n, np.zeros(6, F), 1, 1, sigma=np.ones(6, F))
        assert pr.tobytes() == np.full(n, np.float32(1.0 / np.float64(n)), F).tobytes()
    check_tiers(hs, tiers(port, request), 1, pose7((1, 2, 3), (0.1, 0.2, 0.3)), 4, 9, sigma=np.full(6, 0.1, F))
    check_tiers(hs, tiers(port, request), 1, pose7((1, 2, 3), (0.1, 0.2, 0.3)), 4, 9, cov=dense_cov())


def test_negative_eigenvalue_gives_a_non_finite_transform():
    c = np.diag([0.1, 0.1, 0.1, 0.1, 0.1, -0.01]).reshape(36)
    assert not np.isfinite(engine.noise_transform(c)).all()
