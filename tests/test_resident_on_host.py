"""The bodies of tests/test_gpu_resident.py executed on the HOST: tests/fake_engine.py implements the resident particle
set with the product's per-thread device functions compiled for the host (tests/hostsim).  If these pass here, a failure
of the same test on the H100 can only come from the kernels or the engine's plumbing around those functions."""
import pytest

import fake_engine
import test_gpu_resident as T
from test_hostsim import hostsim  # noqa: F401  (builds tests/hostsim/libhostsim.so)


@pytest.fixture(scope="module")
def cc():
    from oracle import cpu_checker
    cpu_checker.build("port")
    return cpu_checker


def test_set_get(hostsim):  # noqa: F811
    T.test_set_get_round_trip(fake_engine)


@pytest.mark.parametrize("turn", [0.3, -2.9, 0.0])
def test_predict(hostsim, cc, turn):  # noqa: F811
    T.test_predict_matches_oracle(fake_engine, cc, turn)


def test_measure_update(hostsim):  # noqa: F811
    T.test_measure_update_matches_host_path(fake_engine)


def test_measure_update_keeps_prior(hostsim):  # noqa: F811
    T.test_measure_update_keeps_the_prior_when_nothing_survives(fake_engine)


@pytest.mark.parametrize("n,frac", [(64, 0.37), (5000, 0.0), (65536, 0.999)])
def test_resample(hostsim, n, frac):  # noqa: F811
    T.test_resample_picks_are_the_reference_systematic_picks(fake_engine, n, frac)


@pytest.mark.parametrize("n,with_prev", [(64, True), (5000, False), (65536, True)])
def test_estimate(hostsim, cc, n, with_prev):  # noqa: F811
    T.test_estimate_matches_the_filter(fake_engine, cc, n, with_prev)


def test_cycle(hostsim):  # noqa: F811
    T.test_cycle_predict_measure_resample(fake_engine)
