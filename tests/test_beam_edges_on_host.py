"""The beam edge worlds (tests/beam_edge_worlds.py) through the per-ray device functions compiled for the host, against the
reference build (oracle/_ref/libmcl3dl_ref.so): records and per-ray status bit for bit, for both casters.  This proves
the worlds and their expectations before tests/test_gpu_beam_edges.py holds the kernels to the same reference."""
import numpy as np
import pytest

import beam_edge_worlds as W
from mcl_3dl_b200 import engine
from oracle import cpu_checker as cc

STATUS_CODES = {0, 1, 2, 3}  # short, hit, long, total reflection


@pytest.fixture(scope="module")
def ref():
    if not cc.available("reference"):
        pytest.skip("oracle/_ref/libmcl3dl_ref.so not built (needs a checkout of the reference at build time)")
    return cc.CpuChecker("reference")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    return W.load_hostsim(tmp_path_factory.mktemp("beam_edges"))


def reference(ref, w, caster):
    cpu = ref.create(w["map"], cc.lik_params(dist_weight=w["dist_weight"]), cc.beam_raw(**W.beam_kwargs(w, caster)))
    cpu.set_tally(True)
    rec = cpu.measure(w["poses"], None, w["scan"], w["origins"])
    st = cpu.beam_status(w["poses"], w["scan"], w["origins"]) if len(w["scan"]) else np.zeros((len(w["poses"]), 0), np.uint8)
    cpu.close()
    return rec, st


@pytest.mark.parametrize("name,caster", W.cases())
def test_edge_world_on_host_equals_reference(ref, hs, name, caster):
    w = W.world(name)
    want, want_st = reference(ref, w, caster)
    beam = engine.beam_params_from_reference(**W.beam_kwargs(w, caster))
    lik = engine.LikParams(dist_weight=w["dist_weight"])
    got, st, work = hs(w["map"], w["poses"], w["scan"], w["origins"], beam, lik, near=(2, 1))
    for f in ("score_beam", "n_short", "n_hit", "n_long"):
        assert np.array_equal(got[f], want[f]), f
    assert st.tobytes() == want_st.tobytes()
    assert set(np.unique(st)) <= STATUS_CODES
    assert (got["n_short"] + got["n_hit"] + got["n_long"] + (st == 3).sum(axis=1) == len(w["scan"])).all()
    if len(w["scan"]):
        assert work[0] > 0


def test_edge_worlds_reach_their_edges(ref, hs):
    """The worlds are not vacuous: every status occurs under both casters, the score underflows to the floor, a
    filtered first point in a DDA cell lets a later one collide, and the KD caster's second search comes back empty."""
    seen = {c: set() for c in W.CASTERS}
    floors = 0
    for name, caster in W.cases():
        w = W.world(name)
        rec, st = reference(ref, w, caster)
        seen[caster] |= set(np.unique(st).tolist())
        floors += int((rec["score_beam"] == np.float32(w["beam"].get("beam_likelihood_min", 0.2))).sum())
    assert seen["dda"] == STATUS_CODES and seen["kd"] == STATUS_CODES
    assert floors > 0
    # labels: a filtered point that comes first in its DDA cell hides the cell's later label-1 points (rays through the
    # x = +1 wall go on, LONG), while the label-1 wall at x = -1 (== filter_label_max) stops rays
    w = W.world("labels")
    _, st = reference(ref, w, "dda")
    plus_x = (w["scan"]["x"] > 1.2) & (np.abs(w["scan"]["y"]) < 0.5) & (np.abs(w["scan"]["z"]) < 0.3)
    minus_x = (w["scan"]["x"] < -1.2) & (np.abs(w["scan"]["y"]) < 0.5) & (np.abs(w["scan"]["z"]) < 0.3)
    assert plus_x.any() and (st[:, plus_x] == 2).all()
    assert minus_x.any() and (st[:, minus_x] <= 1).any()
    # kd_sin_one: where the empty second search leaves sin_angle = 1, oblique rays collide as SHORT / HIT that are total
    # reflections with unit metric weights (the second search then finds the floor)
    w = W.world("kd_sin_one")
    _, st = reference(ref, w, "kd")
    _, st_unit = reference(ref, dict(w, dist_weight=(1.0, 1.0, 1.0)), "kd")
    assert ((st <= 1) & (st_unit == 3)).sum() >= 6
