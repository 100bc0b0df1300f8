"""The bodies of tests/test_gpu_pf_exact.py executed on the HOST through tests/fake_engine.py (the resident particle set
run by the product's per-particle functions compiled for the host), with the SM count of an H100 SXM (132).  This
checks the case generators, the exact-sum machinery and the near-boundary assertions without a GPU; the device then
only has its kernels, folds and plumbing to get right."""
from fractions import Fraction

import numpy as np
import pytest

import fake_engine
import test_gpu_pf_exact as T
from test_hostsim import hostsim  # noqa: F401  (builds tests/hostsim/libhostsim.so)

SM = 132


@pytest.mark.parametrize("n,kind", T.PREDICT_CASES)
def test_predict(hostsim, n, kind):  # noqa: F811
    T.predict_case(fake_engine, SM, n, kind)


def test_predict_cutoff_floats():
    T.test_predict_cutoff_floats_straddle_the_threshold()


@pytest.mark.parametrize("i,n", list(enumerate(T.RESAMPLE_SIZES)))
def test_resample(hostsim, i, n):  # noqa: F811
    T.resample_case(fake_engine, SM, n, T.FRACS[i % 3], T.SEEDS[i % 3])


@pytest.mark.parametrize("kind,n", [("ties", 4097), ("total3.7", 1025), ("total1e-30", 4097), ("one", 17)])
def test_resample_weights(hostsim, kind, n):  # noqa: F811
    T.test_resample_weights(fake_engine, SM, hostsim, kind, n)


def test_resample_past_the_end_sweep(hostsim):  # noqa: F811
    T.test_resample_past_the_end_sweep(fake_engine, SM, hostsim)


def test_resample_three_calls(hostsim):  # noqa: F811
    T.test_resample_three_calls(fake_engine, SM, hostsim)


# (2^20 particles: the sequential sum's bound γ_n is too wide for the equalities; the device's tree depth is ~560)
@pytest.mark.parametrize("n,ties,with_prev", [c for c in T.ESTIMATE_CASES if c[0] != (0, 1 << 20)])
def test_estimate(hostsim, n, ties, with_prev):  # noqa: F811
    T.estimate_case(fake_engine, SM, n, ties, with_prev)


def test_estimate_cancelling_sums(hostsim):  # noqa: F811
    T.estimate_case(fake_engine, SM, 4099, far=True)   # (the sequential bound γ_n is too wide at the device's sizes)


@pytest.mark.parametrize("path", ["measure_update", "resident"])
@pytest.mark.parametrize("P,ties", [c for c in T.FOLD_CASES if c[0] != (3, 7)])
def test_weight_fold(hostsim, P, ties, path):  # noqa: F811
    T.fold_case(fake_engine, SM, P, ties, path)


def test_weight_fold_total_rounds_up(hostsim):  # noqa: F811
    T.fold_case(fake_engine, SM, 8192, "none", "resident", round_up=True)


def test_weight_fold_with_odometry_factor(hostsim):  # noqa: F811
    T.fold_case(fake_engine, SM, 8193, "none", "resident", sigma=0.4)


def test_cycle(hostsim):  # noqa: F811
    T.cycle_case(fake_engine, SM, n=3000)


@pytest.mark.parametrize("n,with_prev", [(5000, False), (20_000, True)])
def test_exported_terms_reproduce_the_host_estimate(hostsim, n, with_prev):  # noqa: F811
    """The exact sums of hostsim_pf_est_terms / hostsim_pf_cov_terms fed through hostsim_pf_est_finish give
    hostsim_pf_estimate's results, whose sums are sequential doubles: within γ_n of the exact sums, so equal after the
    rounding to float wherever to_f32's margin holds, and within one ulp for the rotation."""
    L = T.hs()
    st, prob, _, _ = T.estimate_inputs(n, "none", 1, SM)
    prev = T.synth.make_poses([[3.1, -4.0, 0.5]], T.synth.quat_from_rpy([[0.0, 0.0, 2.95]])) if with_prev else None
    got = fake_engine.Engine()
    got.particles_set(st, prob)
    est = got.particles_estimate(prev, 0.2, 0.25)
    bias, terms = np.zeros(n, np.float32), np.zeros((n, 20), np.float32)
    assert L.hostsim_pf_est_terms(T._ptr(prob), T._ptr(st), n, T._ptr(prev), 0.2, 0.25, T._ptr(bias), T._ptr(terms)) == 0
    S, A = T.col_sums(terms)
    g = T.gamma(n)
    assert np.float32(est["weight_sum_biased"]) == T.to_f32(S[0], g * Fraction(A[0]))
    for a, f in enumerate(("px", "py", "pz")):
        assert est["mean_biased"][f][0] == T.to_f32(S[1 + a] / S[0], T.ratio_err(S[1 + a], A[1 + a], S[0], A[0], n))
    v = np.array([float(s) for s in S])
    mpos, mrot, epos, erpy = (np.zeros(k, np.float32) for k in (3, 4, 3, 3))
    L.hostsim_pf_est_finish(T._ptr(v), T._ptr(mpos), T._ptr(mrot), T._ptr(epos), T._ptr(erpy))
    q = np.array([est["mean_biased"][f][0] for f in ("qx", "qy", "qz", "qw")], np.float32)
    assert (np.abs(q.astype(np.float64) - mrot) <= T.ulp(mrot)).all()
    d, t2 = np.zeros((n, 6), np.float32), np.zeros((n, 22), np.float32)
    assert L.hostsim_pf_cov_terms(T._ptr(prob), T._ptr(st), n, T._ptr(epos), T._ptr(erpy), T._ptr(d), T._ptr(t2)) == 0
    Cs, CA = T.col_sums(t2)
    t = 1
    for j in range(6):
        for k in range(j, 6):
            assert est["cov"][j, k] == T.to_f32(Cs[t] / Cs[0], T.ratio_err(Cs[t], CA[t], Cs[0], CA[0], n)), (j, k)
            t += 1
