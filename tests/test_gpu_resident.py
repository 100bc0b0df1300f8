"""Resident particle set (scope row f3, mcl3dl_particles_*): predict, measure + weight update, resample on the device.

"""
import numpy as np
import pytest

from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(scope="module")
def cc():
    from oracle import cpu_checker
    cpu_checker.build("port")
    return cpu_checker


def make_states(n, seed, scene=None):
    rng = np.random.default_rng(seed)
    st = np.zeros(n, dtype=synth.STATE)
    if scene is not None:
        st["pos"] = np.stack([scene["particles"]["px"], scene["particles"]["py"], scene["particles"]["pz"]], axis=1)[:n]
        st["rot"] = np.stack([scene["particles"][k] for k in ("qx", "qy", "qz", "qw")], axis=1)[:n]
    else:
        st["pos"] = rng.uniform(-10, 10, (n, 3))
        q = rng.normal(0, 1, (n, 4))
        st["rot"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    for f in ("noise_ll", "noise_la", "noise_al", "noise_aa"):
        st[f] = rng.normal(0, 0.05, n)
    st["odom_err_integ_lin"] = rng.normal(0, 0.1, (n, 3))
    st["odom_err_integ_ang"] = rng.normal(0, 0.1, (n, 3))
    return st


def fields_close(a, b, rtol, atol):
    for f in a.dtype.names:
        assert np.allclose(a[f], b[f], rtol=rtol, atol=atol), f


def test_set_get_round_trip(eng_mod):
    e = eng_mod.Engine((0,))
    st = make_states(1000, 1)
    prob = np.random.default_rng(2).uniform(0, 1, 1000).astype(np.float32)
    e.particles_set(st, prob)
    got_s, got_p = e.particles_get()
    assert got_s.tobytes() == st.tobytes() and np.array_equal(got_p, prob)
    e.close()


@pytest.mark.parametrize("turn", [0.3, -2.9, 0.0])
def test_predict_matches_oracle(eng_mod, cc, turn):
    """Device sinf/cosf differ from glibc's by a few ulp: 1e-5 relative on the rotation, exact elsewhere in practice."""
    port = cc.CpuChecker("port")
    e = eng_mod.Engine((0,))
    st = make_states(5000, 3)
    prev = synth.make_poses(np.array([[1.0, 2.0, 0.1]]), synth.quat_from_rpy(np.array([[0.02, -0.01, 0.4]])))
    cur = synth.make_poses(np.array([[1.2, 2.1, 0.1]]), synth.quat_from_rpy(np.array([[0.01, 0.03, 0.4 + turn]])))
    e.particles_set(st, np.full(len(st), 1.0 / len(st), np.float32))
    e.particles_predict(prev, cur, 0.1, 10.0, 10.0)
    got, _ = e.particles_get()
    want = port.motion_predict(prev, cur, 0.1, 10.0, 10.0, st.copy())
    fields_close(got, want.view(synth.STATE), rtol=1e-5, atol=1e-6)
    e.close()


def test_measure_update_matches_host_path(eng_mod):
    """The resident update equals mcl3dl_measure_update fed with the same poses, priors and odometry-error factors."""
    s = synth.scene(60_000, 700, 64, 8, seed=141)
    lik = eng_mod.LikParams(dist_weight=(1, 1, 5))
    beam = eng_mod.beam_params_from_reference(num_points_default=8, dda_grid_size=0.2)
    e = eng_mod.Engine((0,))
    e.set_map(s["map"], lik, beam)
    st = make_states(700, 5, scene=s)
    prior = np.random.default_rng(6).uniform(0.1, 1.0, 700).astype(np.float32)
    sigma = np.float32(0.4)
    # NormalLikelihood(sigma)(|odom_err_integ_lin|), include/mcl_3dl/nd.h:45-53, in float as the reference computes it
    a = np.float32(1.0 / np.sqrt(2.0 * np.pi * float(sigma) * float(sigma)))
    sq2 = np.float32(float(sigma) * float(sigma) * 2.0)
    lin = st["odom_err_integ_lin"]
    x = np.sqrt((lin[:, 0] * lin[:, 0] + lin[:, 1] * lin[:, 1]).astype(np.float32) + lin[:, 2] * lin[:, 2]).astype(np.float32)
    extra = (a * np.exp((-x * x / sq2).astype(np.float32)).astype(np.float32)).astype(np.float32)
    want_post, want_summ, _ = e.measure_update(s["particles"][:700], s["lik"], s["beam"], s["origins"], prior, extra_likelihood=extra)
    e.particles_set(st, prior)
    summ = e.particles_measure_update(s["lik"], s["beam"], s["origins"], float(sigma))
    _, post = e.particles_get()
    assert summ["kept"] == want_summ["kept"] == 1
    assert np.allclose(post, want_post, rtol=2e-5, atol=1e-12)          # device expf vs numpy's
    assert abs(summ["entropy"] - want_summ["entropy"]) < 1e-4 * abs(want_summ["entropy"])
    assert summ["match_ratio_min"] == want_summ["match_ratio_min"] and summ["match_ratio_max"] == want_summ["match_ratio_max"]
    # without the odometry term the two paths are bit-identical
    want_post, want_summ, _ = e.measure_update(s["particles"][:700], s["lik"], s["beam"], s["origins"], prior)
    e.particles_set(st, prior)
    summ = e.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.0)
    _, post = e.particles_get()
    assert np.array_equal(post, want_post) and summ["max_index"] == want_summ["max_index"]
    e.close()


def test_measure_update_keeps_the_prior_when_nothing_survives(eng_mod):
    s = synth.scene(20_000, 64, 32, 4, seed=81)
    e = eng_mod.Engine((0,))
    e.set_map(s["map"], eng_mod.LikParams(dist_weight=(1, 1, 5)), eng_mod.beam_params_from_reference(num_points_default=4))
    st = make_states(64, 9, scene=s)
    st["pos"][:, 0] += np.float32(1e4)                                    # nothing matches: every weight is zero
    prior = np.full(64, 1.0 / 64, np.float32)
    e.particles_set(st, prior)
    summ = e.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.0)
    _, post = e.particles_get()
    assert summ["kept"] == 0 and np.array_equal(post, prior)
    e.close()


@pytest.mark.parametrize("n,frac", [(64, 0.37), (5000, 0.0), (65536, 0.999)])
def test_resample_picks_are_the_reference_systematic_picks(eng_mod, n, frac):
    """sigma = 0 for the plain copies, a real sigma for the statistics of the duplicates."""
    e = eng_mod.Engine((0,))
    rng = np.random.default_rng(n)
    prob = (rng.uniform(0.2, 1.0, n) ** 2).astype(np.float32)            # skewed, but no weight small enough to vanish
    prob /= prob.sum(dtype=np.float32)                                   # in the float prefix sum (ties: see test_hostsim)
    st = make_states(n, 11)
    st["pos"][:, 0] = np.arange(n, dtype=np.float32)                     # x = the source index, to read the picks back
    e.particles_set(st, prob)
    sp, sr = np.array([0.05, 0.05, 0.01], np.float32), np.array([0.0, 0.0, 0.02], np.float32)
    e.particles_resample(sp, sr, frac, seed=42)
    out, out_p = e.particles_get()
    accum = np.zeros(n, np.float32)
    a = np.float32(0)
    for i in range(n):                                                   # pf.h:189-194: sequential float sum
        a = np.float32(a + prob[i])
        accum[i] = a
    assert (np.diff(accum) > 0).all()
    pstep = np.float32(a / np.float32(n))
    pscan = (pstep * np.arange(n, dtype=np.float32) + np.float32(np.float32(frac) * pstep)).astype(np.float32)
    ss = np.searchsorted(accum, pscan, side="left")
    found = ss < n                                                       # past the end: the last particle found (pf.h:208-212)
    src = np.where(found, ss, ss[found][-1] if found.any() else 0)
    dup = np.concatenate([[ss[0] == 0], ss[1:] == ss[:-1]]) & found
    plain = ~dup
    assert out[plain].tobytes() == st[src[plain]].tobytes()             # copies are bit-identical
    assert np.all(out_p == np.float32(1.0 / n))
    if dup.sum() > 200:
        d = out["pos"][dup] - st["pos"][src[dup]]
        assert np.abs(d[:, 0]).max() < 6 * sp[0]                        # still next to the particle they were copied from
        assert 0.8 * sp[0] < d[:, 0].std() < 1.2 * sp[0] and abs(d[:, 0].mean()) < 0.2 * sp[0]
        assert (out["noise_ll"][dup] == 0).all()
        assert np.allclose(np.linalg.norm(out["rot"][dup], axis=1), 1.0, atol=1e-5)
    e.close()


@pytest.mark.parametrize("n,with_prev", [(64, True), (5000, False), (65536, True)])
def test_estimate_matches_the_filter(eng_mod, cc, n, with_prev):
    """mcl3dl_particles_estimate == pf_->bias + expectationBiased + max + covariance(1.0, 1.0) of the reference filter
    (the oracle port, pinned bit for bit to the reference build by tests/test_oracle_golden.py).  The device sums in
    double with a fixed tree, the reference sequentially in float: 1e-4 relative is the bar."""
    port = cc.CpuChecker("port")
    rng = np.random.default_rng(n)
    st = make_states(n, 21)
    st["pos"] = rng.normal([3.0, -4.0, 0.5], [0.3, 0.2, 0.05], (n, 3))
    st["rot"] = synth.quat_from_rpy(rng.normal([0.01, -0.02, 2.9], [0.02, 0.02, 0.2], (n, 3)))   # yaw wraps past pi
    st["rot"] *= (1.0 + rng.normal(0, 1e-3, (n, 1))).astype(np.float32)                          # rot_ is not exactly unit
    prob = rng.uniform(0.1, 1.0, n).astype(np.float32)
    prob /= prob.sum(dtype=np.float64).astype(np.float32) * np.float32(1.001)     # total < 1: the reference adds every particle
    prev = synth.make_poses([[3.1, -4.0, 0.5]], synth.quat_from_rpy([[0.0, 0.0, 2.95]])) if with_prev else None
    e = eng_mod.Engine((0,))
    e.particles_set(st, prob)
    got = e.particles_estimate(prev, 0.2, 0.25)
    mean, best, cov = port.pf_estimate(prob, st.view(cc.MOTION_STATE), prev, 0.2, 0.25)
    assert got["max_index"] == best == int(np.argmax(prob))
    assert got["max_state"]["px"][0] == st["pos"][best, 0] and got["max_state"]["qw"][0] == st["rot"][best, 3]
    for f in ("px", "py", "pz"):
        assert abs(got["mean_biased"][f][0] - mean[f][0]) < 1e-4 * max(1.0, abs(mean[f][0])), f
    for f in ("qx", "qy", "qz", "qw"):
        assert abs(got["mean_biased"][f][0] - mean[f][0]) < 2e-5, f
    assert np.allclose(got["cov"], cov, rtol=2e-3, atol=1e-7)
    assert np.allclose(got["cov"], got["cov"].T) and (np.diag(got["cov"]) > 0).all()
    e.close()


def test_cycle_predict_measure_resample(eng_mod):
    """Three localisation cycles on the device: the weight mass moves to the particles near the true pose."""
    s = synth.scene(60_000, 2000, 96, 8, seed=151)
    e = eng_mod.Engine((0,))
    e.set_map(s["map"], eng_mod.LikParams(dist_weight=(1, 1, 5)), eng_mod.beam_params_from_reference(num_points_default=8))
    st = make_states(2000, 13, scene=s)
    st["noise_ll"] = st["noise_la"] = st["noise_al"] = st["noise_aa"] = 0
    e.particles_set(st, np.full(2000, 1.0 / 2000, np.float32))
    still = synth.make_poses(np.zeros((1, 3)), np.array([[0, 0, 0, 1.0]]))
    ent = []
    for k in range(3):
        e.particles_predict(still, still, 0.1, 10.0, 10.0)
        summ = e.particles_measure_update(s["lik"], s["beam"], s["origins"], 0.0)
        assert summ["kept"] == 1
        ent.append(summ["entropy"])
        e.particles_resample(np.full(3, 0.01, np.float32), np.array([0, 0, 0.005], np.float32), 0.5, seed=7 + k)
    est = e.particles_estimate(None)
    out, prob = e.particles_get()
    assert np.linalg.norm([est["mean_biased"]["px"][0] - out["pos"][:, 0].mean(), est["mean_biased"]["py"][0] - out["pos"][:, 1].mean()]) < 1e-3
    d = np.linalg.norm(out["pos"][:, :2] - np.asarray(s["truth_pos"])[:2], axis=1)
    d0 = np.linalg.norm(st["pos"][:, :2] - np.asarray(s["truth_pos"])[:2], axis=1)
    assert np.median(d) < np.median(d0)
    e.close()
