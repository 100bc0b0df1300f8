"""The ray markers (mcl3dl_beam_cast) without a GPU: the per-thread device functions (cast_ray_at / cast_ray_kd_at and the
kernel's pose, transform and origin steps) compiled for the host, the port checker and the reference's own marker loop
(oracle/beam_cast_api.h) agree record for record, bit for bit, for both casters, on every world of
tests/beam_cast_worlds.py and from every pose in it."""
import numpy as np
import pytest

import beam_cast_worlds as B
import beam_edge_worlds as W
from mcl_3dl_b200 import engine
from oracle import beam_cast_checker as bc
from oracle import cpu_checker as cc


@pytest.fixture(scope="module")
def port():
    return bc.BeamCastChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not bc.available("reference"):
        pytest.skip("oracle/_ref/libmcl3dl_beam_cast_ref.so not built (needs a checkout of the reference at build time)")
    return bc.BeamCastChecker("reference")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    return B.load_hostsim(tmp_path_factory.mktemp("beam_cast"))


def checker_rays(checker, w, caster):
    m = checker.create(w["map"], cc.lik_params(dist_weight=w["dist_weight"]), cc.beam_raw(**W.beam_kwargs(w, caster)))
    out = [m.beam_cast(w["poses"][i], w["scan"], w["origins"]) for i in range(len(w["poses"]))]
    m.close()
    return out


def host_rays(hs, w, caster):
    beam = engine.beam_params_from_reference(**W.beam_kwargs(w, caster))
    lik = engine.LikParams(dist_weight=w["dist_weight"])
    return [hs(w, i, beam, lik) for i in range(len(w["poses"]))]


@pytest.mark.parametrize("name,caster", B.cases())
def test_host_build_port_and_reference_agree(port, ref, hs, name, caster):
    w = B.world(name)
    want = checker_rays(ref, w, caster)
    got_port = checker_rays(port, w, caster)
    got_host = host_rays(hs, w, caster)
    for i, r in enumerate(want):
        assert got_port[i].tobytes() == r.tobytes(), "port, pose %d" % i
        assert got_host[i].tobytes() == r.tobytes(), "host build, pose %d" % i
        lng = r["status"] == 2
        assert np.isnan(r["pos"][lng]).all() and np.isfinite(r["pos"][~lng]).all()


def test_worlds_reach_the_deciding_step_edges(ref):
    """Not vacuous: every status occurs under both casters, first and last cast steps decide rays, rays leave the grid
    and start outside the DDA box (LONG), and filtered pillars let rays go on to a wall behind them."""
    seen = {c: set() for c in W.CASTERS}
    first = {c: 0 for c in W.CASTERS}
    last = {c: 0 for c in W.CASTERS}
    for name, caster in B.cases():
        w = B.world(name)
        for r in checker_rays(ref, w, caster):
            seen[caster] |= set(np.unique(r["status"]).tolist())
            k, n_last = B.decided_step(r, w, caster)
            hit = r["status"] != 2
            first[caster] += int((hit & (k == 1)).sum())
            last[caster] += int((hit & (k == n_last)).sum())
    assert seen["dda"] == {0, 1, 2, 3} and seen["kd"] == {0, 1, 2, 3}
    assert min(first.values()) > 0 and min(last.values()) > 0, (first, last)
    # begin outside the DDA box, ends far beyond the grid: LONG with a NaN position
    w = B.world("map_box")
    r = checker_rays(ref, w, "dda")
    assert (r[0]["status"] == 2).all()  # the first particle sits outside the box
    assert all(np.isnan(x["pos"][x["status"] == 2]).all() for x in r)
    # a filtered pillar in front of a wall: without the label filter the same rays stop earlier
    moved = 0
    for s in B.SEEDS:
        w = B.world("room_%d" % s)
        for caster in W.CASTERS:
            filt = checker_rays(ref, w, caster)
            unfilt = checker_rays(ref, dict(w, beam=dict(w["beam"], filter_label_max=0xFFFFFFFF)), caster)
            for a, b in zip(filt, unfilt):
                both = (a["status"] != 2) & (b["status"] != 2)
                da = np.linalg.norm(a["pos"] - a["begin"], axis=1)
                db = np.linalg.norm(b["pos"] - b["begin"], axis=1)
                moved += int((both & (da > db + 0.05)).sum())
    assert moved > 0


def test_port_rejects_a_label_beyond_the_origins(port):
    w = B.world("steps")
    m = port.create(w["map"], cc.lik_params(), cc.beam_raw())
    scan = w["scan"].copy()
    scan["label"][3] = len(w["origins"])
    with pytest.raises(RuntimeError):
        m.beam_cast(w["poses"][0], scan, w["origins"])
    m.close()
