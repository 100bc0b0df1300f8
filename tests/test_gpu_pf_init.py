"""mcl3dl_particles_init on an H100: the initial seed of the resident set (the configured start's
DiagonalNoiseGenerator and cbPosition's MultivariateNoiseGenerator) against the host build of pf_init_state and the
port checker (tests/test_pf_init_on_host.py holds those to the reference's own code bit for bit).

Bars, derived as in tests/test_gpu_pf_exact.py (LIBM, R there):
  - the device's standard normals: with mean 0 and every sigma 1 the seed stores them (pos = z * 1 + 0, odom_err_integ_ang
    = org - 0), and each equals the host's z, recomputed from the documented Philox layout, within Z_REL |z| + ulp(z)
    (logf / cosf / sinf only; the Philox words and uniforms are exact, so one different word would be far outside);
  - given those same z, position, both integrals and the probability are exact: the port checker fed the device's z
    gives the same bytes;
  - the rotation is Quat(rpy) of the same org with the device's sinf / cosf: within NOISE_ROT_BAR (a sum of products of
    three libm values, the bar of the expansion noise's rotation, which also covers a quaternion product).
The sample mean and covariance at 1 M particles are held to T T^T within six standard errors, derived from N."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import synth
from oracle import pf_init_checker as pic
from test_gpu_pf_events import NOISE_ROT_BAR, Z_REL
from test_gpu_pf_exact import ulp
from test_pf_init_on_host import dense_cov, hs, host_init, pose7, rviz_cov  # noqa: F401

pytestmark = pytest.mark.gpu
PARITY = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "init_parity_test")
SIZES = [1, 1000, 65_536, 1 << 20]
F = np.float32


@pytest.fixture(scope="module")
def E():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(scope="module")
def port():
    pic.build("port")
    return pic.PfInitChecker("port")


def device_z(E, n, seed):
    """The device's standard normals of init call 1 (a fresh engine): mean 0 and sigma 1 store them."""
    e = E.Engine((0,))
    e.particles_init(n, np.zeros(6, F), seed, sigma=np.ones(6, F))
    st, _ = e.particles_get()
    e.close()
    return np.concatenate([st["pos"], st["odom_err_integ_ang"]], 1)


def init_once(E, n, mean6, seed, **gen):
    e = E.Engine((0,))
    e.particles_init(n, mean6, seed, **gen)
    st, pr = e.particles_get()
    e.close()
    return st, pr


def check_given_z(got, gp, want, wp):
    """pos, the integrals and the probability exact; rot within NOISE_ROT_BAR"""
    for f in ("pos", "odom_err_integ_lin", "odom_err_integ_ang", "noise_ll", "noise_la", "noise_al", "noise_aa"):
        assert got[f].tobytes() == want[f].tobytes(), f
    assert gp.tobytes() == wp.tobytes()
    d = np.abs(got["rot"].astype(np.float64) - want["rot"])
    assert (d <= NOISE_ROT_BAR + ulp(want["rot"])).all(), d.max()


@pytest.mark.parametrize("n", SIZES)
def test_device_normals_are_the_host_recomputation(E, hs, n):  # noqa: F811
    z = device_z(E, n, 2 ** 63 + 77).astype(np.float64)
    _, _, want = host_init(hs, n, np.zeros(6, F), 2 ** 63 + 77, 1, sigma=np.ones(6, F))
    d = np.abs(z - want)
    assert (d <= Z_REL * np.abs(want) + ulp(want)).all(), d.max()


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("gen", ["diagonal", "rviz", "dense"])
def test_seed_against_the_port_given_the_device_normals(E, port, n, gen):
    seed = 0xC0FFEE + n
    z = device_z(E, n, seed)
    pose = pose7((1.5, -2.0, 0.25), (0.05, -1.2, 3.1))
    mean6 = port.mean(pose)
    if gen == "diagonal":
        kw = dict(sigma=np.array([0.5, 0.5, 0.0, 0.0, 0.1, 0.3], F))
        want, wp = port.init(pose, z, sigma=kw["sigma"])
    else:
        from mcl_3dl_b200 import engine
        T = engine.noise_transform(rviz_cov() if gen == "rviz" else dense_cov())
        kw = dict(norm_transform=T)
        want, wp = port.init(pose, z, norm_transform=T)
    got, gp = init_once(E, n, mean6, seed, **kw)
    check_given_z(got, gp, want, wp)
    if gen == "rviz":   # z, roll and pitch are the mean exactly
        assert (got["pos"][:, 2] == mean6[2]).all() and (got["odom_err_integ_ang"][:, :2] == 0).all()


@pytest.mark.parametrize("seed", [3, 2 ** 40 + 1])
def test_sample_moments_at_one_million(E, seed):
    from mcl_3dl_b200 import engine
    n = 1 << 20
    T = engine.noise_transform(dense_cov(5)).astype(np.float64)
    mean6 = np.array([1.0, -2.0, 0.5, 0.1, -0.2, 0.3], F)
    st, pr = init_once(E, n, mean6, seed, norm_transform=T)
    x = np.concatenate([st["pos"], st["odom_err_integ_ang"].astype(np.float64) + mean6[3:]], 1).astype(np.float64)
    S = T @ T.T
    sd = np.sqrt(np.diag(S))
    m = x.mean(0)
    assert (np.abs(m - mean6) <= 6 * sd / np.sqrt(n)).all(), (m - mean6) / (sd / np.sqrt(n))
    c = np.cov(x, rowvar=False)
    se = np.sqrt((np.outer(np.diag(S), np.diag(S)) + S * S) / n)
    assert (np.abs(c - S) <= 6 * se).all(), np.max(np.abs(c - S) / se)
    assert np.all(pr == F(1.0 / n))


def test_call_count_determinism_and_seeds(E):
    n = 5000
    sg = dict(sigma=np.full(6, 0.2, F))
    first, _ = init_once(E, n, np.zeros(6, F), 11, **sg)
    again, _ = init_once(E, n, np.zeros(6, F), 11, **sg)
    other, _ = init_once(E, n, np.zeros(6, F), 12, **sg)
    assert first.tobytes() == again.tobytes()
    assert not np.array_equal(first["pos"], other["pos"])
    e = E.Engine((0,))
    e.particles_init(n, np.zeros(6, F), 11, **sg)
    assert e.particles_get()[0].tobytes() == first.tobytes()
    e.particles_set(*e.particles_get())         # particles_set does not reset init's count
    e.particles_init(n, np.zeros(6, F), 11, **sg)
    second = e.particles_get()[0]
    assert not np.array_equal(second["pos"], first["pos"])
    e.close()
    # the other entry points keep their own counts: noise after init draws noise call 1, as after an upload
    outs = []
    for upload in (False, True):
        e = E.Engine((0,))
        if upload:
            e.particles_set(first, np.full(n, F(1.0 / n)))
        else:
            e.particles_init(n, np.zeros(6, F), 11, **sg)
        e.particles_noise((0.1, 0.1, 0.1), (0.01, 0.01, 0.01), 5)
        e.particles_resample((0.05, 0.05, 0.05), (0.01, 0.01, 0.02), 0.37, 99)
        outs.append(e.particles_get()[0].tobytes())
        e.close()
    assert outs[0] == outs[1]


def test_count_grows_from_nothing_shrinks_and_grows(E):
    e = E.Engine((0,))
    for n in (1000, 10, 200_000, 3):
        e.particles_init(n, np.zeros(6, F), 1, sigma=np.ones(6, F))
        st, pr = e.particles_get()
        assert len(st) == n and np.all(pr == F(1.0 / n)) and np.isfinite(st["pos"]).all()
    # after a resize the next init takes the count it is given
    e.particles_resize(50)
    e.particles_init(77, np.zeros(6, F), 1, sigma=np.ones(6, F))
    assert len(e.particles_get()[0]) == 77
    e.close()


def test_init_then_cycle_equals_uploaded_seed(E):
    """Init followed by predict, measure_update, resample and estimate gives the same bytes as particles_set of the
    downloaded seed followed by the same calls."""
    s = synth.scene(20_000, 64, 32, 4, seed=81)
    n = 4096
    a = E.Engine((0,))
    a.particles_init(n, np.array([0.5, 0.5, 0.0, 0.0, 0.0, 0.3], F), 8, sigma=np.array([1.0, 1.0, 0.05, 0.01, 0.01, 0.3], F))
    seed_set = a.particles_get()
    b = E.Engine((0,))
    b.particles_set(*seed_set)
    prev = np.zeros(1, synth.POSE)
    prev["qw"] = 1
    cur = prev.copy()
    cur["px"], cur["qz"], cur["qw"] = 0.3, np.sin(0.05), np.cos(0.05)
    outs = []
    for e in (a, b):
        e.set_map(s["map"], E.LikParams(dist_weight=(1, 1, 5)), E.beam_params_from_reference(num_points_default=4))
        e.particles_predict(prev, cur, 0.1, 10.0, 10.0)
        summ = e.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.0)
        e.particles_resample((0.05, 0.05, 0.05), (0.01, 0.01, 0.02), 0.37, 99)
        est = e.particles_estimate(cur, 1.0, 1.0)
        st, pr = e.particles_get()
        outs.append((st.tobytes(), pr.tobytes(), est["mean_biased"].tobytes(), est["cov"].tobytes(), est["max_index"],
                     summ["kept"], summ["weight_sum"]))
        e.close()
    assert outs[0][:6] == outs[1][:6] and outs[0][6] == outs[1][6]


def test_errors_leave_the_set_untouched(E):
    L = E.load_library()
    e = E.Engine((0,))
    e.particles_init(100, np.zeros(6, F), 1, sigma=np.ones(6, F))
    st, pr = e.particles_get()

    def call(n=100, mv=0, mean=None, sigma=None, T=None, h=True, prm=True):
        p = E.InitParams()
        p.multivariate = mv
        for k, v in enumerate(np.zeros(6) if mean is None else mean):
            p.mean[k] = v
        for k, v in enumerate(np.ones(6) if sigma is None else sigma):
            p.sigma[k] = v
        for k, v in enumerate(np.eye(6).reshape(36) if T is None else np.asarray(T).reshape(36)):
            p.norm_transform[k] = v
        return L.mcl3dl_particles_init(e.h if h else None, n, C.byref(p) if prm else None, 1)

    assert call(h=False) == -1
    assert call(prm=False) == -1
    assert call(n=0) == -1
    assert call(n=1 << 31) == -1
    assert call(mv=2) == -1 and call(mv=-1) == -1
    assert call(mean=[0, 0, np.nan, 0, 0, 0]) == -1 and call(mean=[np.inf, 0, 0, 0, 0, 0]) == -1
    assert call(sigma=[0, 0, 0, -0.1, 0, 0]) == -1 and call(sigma=[0, np.nan, 0, 0, 0, 0]) == -1
    assert call(sigma=[0, 0, 0, 0, 0, np.inf]) == -1
    T = np.eye(6)
    T[3, 2] = np.nan
    assert call(mv=1, T=T) == -1
    # a diagonal seed ignores the transform, a multivariate one the sigmas
    from mcl_3dl_b200 import engine
    assert not np.isfinite(engine.noise_transform(np.diag([1, 1, 1, 1, 1, -1.0]).reshape(36))).all()
    gs, gp = e.particles_get()
    assert gs.tobytes() == st.tobytes() and gp.tobytes() == pr.tobytes()
    assert call(mv=0, T=T) == 0 and call(mv=1, sigma=[-1, np.nan, 0, 0, 0, 0]) == 0
    e.close()
    # a multi-device engine is refused, as for every resident-set call
    import torch
    if torch.cuda.device_count() > 1:
        m = E.Engine((0, 1))
        p = E.InitParams()
        assert L.mcl3dl_particles_init(m.h, 10, C.byref(p), 1) == -1
        m.close()


@pytest.mark.parametrize("args", [[], ["4096"]])
def test_adapter_parity(args):
    """ParticleFilterB200's initResident (the configured start), initUsingCovarianceResident + reset + posesResident
    (cbPosition), a predict / measure / resample cycle, a seed of an enlarged set and a refused covariance, against the
    reference filter with the device's draws replayed (oracle/init_parity_test.cpp)."""
    if not os.path.exists(PARITY):
        pytest.skip("oracle/_ref/init_parity_test not built (needs a checkout of the reference at build time)")
    r = subprocess.run([PARITY] + args, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "INIT PARITY OK" in r.stdout
