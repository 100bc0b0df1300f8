"""Both beam kernels (kernels.cuh: beam_kernel_pl, beam_kernel_dq) held to the reference build (oracle/_ref/libmcl3dl_ref.so)
byte for byte, with both ray casters:

- the edge worlds of tests/beam_edge_worlds.py, each kernel forced through MCL3DL_BEAM (read at engine creation);
- the launch shapes: engine.cu's pick_pl_shape and the dq kernel's rays-per-item rule are restated below from the
  device's SM count, and the (particles, rays) of every case are chosen so that it reaches the shape it names - every
  chunks-per-group value, one and several CTAs per particle group (with a ray count that is not a multiple of a CTA's
  rays), 64 rays per lane, particle counts one above and one below a warp multiple, the dq item sizes 1, 3, 16 and the
  default, and both sides of the job size where the default selection switches kernels.  Large jobs are compared with
  the reference on a strided particle sample and with the host-compiled device functions on every particle;
- the scratch the kernels leave behind (tickets, partial and queue counters, tallies): shape A, then B, then A again;
- measure, beam_status, measure_device and the records of measure_update on the same inputs;
- the work counters of mcl3dl_read_stats (beam_cells_stepped / _occupied / beam_points_tested), which bench.py turns
  into the beam kernel's roofline figure: equal to the host-compiled device functions' counts on the same inputs, with
  the engine's own near-field dilations, in every case above.  The KD caster's points tested depend on how far the NN
  field reaches: by default it covers the caster's second search and the host build's field does not, so there the
  default engine's count is held equal across kernels and launch shapes, and an engine with MCL3DL_NNF_KD_R2=0 (the
  host build's field) is held to all three host counts and to the same records.
"""
import numpy as np
import pytest

import beam_edge_worlds as W
from mcl_3dl_b200 import synth
from oracle import cpu_checker as cc

pytestmark = pytest.mark.gpu

PL_WARPS = 8      # kernels.cuh: kPlWarps = kBlockThreads / 32
CTAS_PER_SM = 4   # the beam kernels' __launch_bounds__(kBlockThreads, 4): resident CTAs per SM
DQ_MIN_JOB = 262144  # engine.cu launch_beam: P * N from which the default selection takes the dq kernel
BEAM_FIELDS = ("score_beam", "n_short", "n_hit", "n_long")


def pl_shape(P, N, sm):
    """engine.cu: pick_pl_shape -> (ppl, cb, cpg)."""
    groups = (P + 31) // 32
    slots = sm * CTAS_PER_SM

    def ctas_for(ppl):
        chunks = max((N + ppl - 1) // ppl, 1)
        cpg = PL_WARPS
        while cpg > 1 and cpg // 2 >= chunks:
            cpg //= 2
        cb = (chunks + PL_WARPS - 1) // PL_WARPS if cpg == PL_WARPS else 1
        gpc = PL_WARPS // cpg
        return (groups + gpc - 1) // gpc * cb, (ppl, cb, cpg)

    ppl = min(max((N * groups + slots * PL_WARPS - 1) // max(slots * PL_WARPS, 1), 1), 64)
    n, sh = ctas_for(ppl)
    while slots < n < 3 * slots and ppl < 64:
        ppl += 1
        n, sh = ctas_for(ppl)
    return sh


def dq_ppl(P, N, sm, forced=0):
    """engine.cu: launch_beam_dq's rays per item (MCL3DL_BEAM_DQ_PPL = forced, 0: from the job size)."""
    warps = sm * CTAS_PER_SM * PL_WARPS
    groups = (P + 31) // 32
    ppl = forced if forced else (N * groups + 4 * warps - 1) // (4 * warps)
    return min(max(ppl, 1), 16)


@pytest.fixture(scope="module")
def E():
    from mcl_3dl_b200 import engine
    return engine


@pytest.fixture(scope="module")
def sm():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def ref():
    if not cc.available("reference"):
        pytest.skip("oracle/_ref/libmcl3dl_ref.so not built (needs a checkout of the reference at build time)")
    return cc.CpuChecker("reference")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    return W.load_hostsim(tmp_path_factory.mktemp("gpu_beam_edges"))


@pytest.fixture
def make(E, monkeypatch):
    engines = []

    def make(w, caster, **env):
        for k in ("MCL3DL_BEAM", "MCL3DL_BEAM_DQ_PPL", "MCL3DL_NEAR_K", "MCL3DL_NEAR_KD_K", "MCL3DL_NNF", "MCL3DL_NNF_KD_R2",
                  "MCL3DL_NN_CELL_FACTOR"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng = E.Engine((0,))
        engines.append(eng)
        eng.set_map(w["map"], E.LikParams(dist_weight=w["dist_weight"]), E.beam_params_from_reference(**W.beam_kwargs(w, caster)))
        return eng
    yield make
    for eng in engines:
        eng.close()


_REF, _HOST = {}, {}


def reference(ref, w, caster, rows):
    """Reference records and status of the particles `rows` (cached per world, caster and rows)."""
    key = (w["name"], caster, tuple(rows))
    if key not in _REF:
        cpu = ref.create(w["map"], cc.lik_params(dist_weight=w["dist_weight"]), cc.beam_raw(**W.beam_kwargs(w, caster)))
        cpu.set_tally(True)
        poses = w["poses"][list(rows)]
        rec = cpu.measure(poses, None, w["scan"], w["origins"])
        st = cpu.beam_status(poses, w["scan"], w["origins"]) if len(w["scan"]) else np.zeros((len(poses), 0), np.uint8)
        cpu.close()
        _REF[key] = (rec, st)
    return _REF[key]


def host(hs, E, eng, w, caster):
    """Records, status and beam work counters of the host-compiled device functions, with the engine's dilations."""
    info = eng.near_field_info()
    key = (w["name"], caster, info[0][0], info[1][0])
    if key not in _HOST:
        beam = E.beam_params_from_reference(**W.beam_kwargs(w, caster))
        _HOST[key] = hs(w["map"], w["poses"], w["scan"], w["origins"], beam, E.LikParams(dist_weight=w["dist_weight"]),
                        near=(info[0][0], info[1][0]))
    return _HOST[key]


def counters(eng):
    s = eng.read_stats()
    return s["beam_cells_stepped"], s["beam_cells_occupied"], s["beam_points_tested"]


def run(eng, w):
    """measure and beam_status, each with freshly zeroed counters -> (records, status, counters of each call)."""
    eng.collect_stats(True)
    rec = eng.measure(w["poses"], None, w["scan"], w["origins"]).copy()
    c_rec = counters(eng)
    st, c_st = np.zeros((len(w["poses"]), 0), np.uint8), c_rec
    if len(w["scan"]):
        eng.collect_stats(True)
        st = eng.beam_status(w["poses"], w["scan"], w["origins"])
        c_st = counters(eng)
    eng.collect_stats(False)
    return rec, st, c_rec, c_st


def sample(P, k=48):
    return np.unique(np.linspace(0, P - 1, min(P, k)).round().astype(int))


_KD_TESTED = {}  # world -> points tested by the KD caster with the engine's default NN field


def check(ref, hs, E, make, eng, w, caster, env):
    """The engine's records, status and counters against the reference (strided sample) and the host build (all).
    With the KD caster the engine's default NN field also covers the second search, so its count of points tested is
    held to the same count under every kernel and launch shape; an engine on the same env with MCL3DL_NNF_KD_R2=0 (the
    host build's field) must return the same records and all three of the host build's counters."""
    rec, st, c_rec, c_st = run(eng, w)
    h_rec, h_st, h_work = host(hs, E, eng, w, caster)
    rows = sample(len(w["poses"]))
    want, want_st = reference(ref, w, caster, rows)
    for f in BEAM_FIELDS:
        assert np.array_equal(rec[f][rows], want[f]), f
    assert st[rows].tobytes() == want_st.tobytes()
    assert rec.tobytes() == h_rec.tobytes()
    assert st.tobytes() == h_st.tobytes()
    assert c_st == c_rec, (c_rec, c_st)
    if caster == "dda":
        assert c_rec == h_work, (c_rec, h_work)
        return rec, st
    assert c_rec[:2] == h_work[:2], (c_rec, h_work)  # cells stepped and occupied do not depend on the field
    assert _KD_TESTED.setdefault(w["name"], c_rec[2]) == c_rec[2], (w["name"], c_rec, _KD_TESTED[w["name"]])
    narrow = make(w, caster, **dict(env, MCL3DL_NNF_KD_R2="0"))
    rec_n, st_n, c_n, c_n_st = run(narrow, w)
    assert rec_n.tobytes() == rec.tobytes() and st_n.tobytes() == st.tobytes()
    assert c_n == h_work and c_n_st == h_work, (c_n, c_n_st, h_work)
    narrow.close()
    return rec, st


# ------------------------------------------------------------------ edge worlds
@pytest.mark.parametrize("kernel", ["pl", "dq"])
@pytest.mark.parametrize("name,caster", W.cases())
def test_edge_world_equals_reference(ref, hs, E, make, name, caster, kernel):
    w = W.world(name)
    env = {"MCL3DL_BEAM": kernel}
    eng = make(w, caster, **env)
    check(ref, hs, E, make, eng, w, caster, env)


# ------------------------------------------------------------------ launch shapes
_POOL_P, _POOL_N = 40_000, 512


def shape_world(P, N):
    """The first P particles and N rays of one fixed tracking scene in the room of the edge worlds (no duplicate map
    points): particles within decimetres of each other, rays 0.3 ... 1.6 m from two origins - SHORT, HIT and LONG."""
    rng = np.random.default_rng(2024)
    pos = rng.uniform((-0.4, -0.4, -0.2), (0.4, 0.4, 0.2), (_POOL_P, 3))
    quat = synth.quat_from_rpy(rng.normal(0, 0.05, (_POOL_P, 3)) + np.array([0, 0, 0.3]))
    d = rng.normal(0, 1, (_POOL_N, 3)) * np.array([1, 1, 0.4])
    scan = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.3, 1.6, (_POOL_N, 1))
    w = W.world("lattice")
    return dict(w, name="shape_%d_%d" % (P, N), poses=synth.make_poses(pos[:P], quat[:P]),
                scan=synth.make_points(scan[:N], np.arange(N) % 2), origins=np.array([[0.0, 0.0, 0.1], [0.05, -0.02, 0.0]],
                                                                                    np.float32),
                beam=dict(w["beam"], num_points_default=24))


def ppl64_job(sm):
    """The smallest job of this device on which pick_pl_shape reaches 64 rays per lane: with 8 * 63 + 1 rays a CTA
    covers a particle group only at ppl = 64, and one group more than half the resident CTAs keeps the grid between one
    and three waves while ppl climbs."""
    N = 8 * 63 + 1
    P = 32 * (sm * CTAS_PER_SM // 2 + 1) - 1
    return P, N


def shape_cases(sm):
    """(id, P, N, env, what the case must reach)."""
    P64, N64 = ppl64_job(sm)
    pl = {"MCL3DL_BEAM": "pl"}
    dq = {"MCL3DL_BEAM": "dq"}
    return [
        ("pl_cpg1", 33, 1, pl, lambda s: s[2] == 1),
        ("pl_cpg2", 31, 2, pl, lambda s: s[2] == 2),
        ("pl_cpg4", 64, 3, pl, lambda s: s[2] == 4),
        ("pl_cpg8_cb1", 65, 7, pl, lambda s: s[2] == 8 and s[1] == 1),
        ("pl_cb3", 31, 21, pl, lambda s: s[1] == 3 and 21 % (8 * s[0])),
        ("pl_cb_many", 1025, 300, pl, lambda s: s[1] >= 3 and 300 % (8 * s[0])),
        ("pl_ppl64", P64, N64, pl, lambda s: s[0] == 64),
        ("dq_default", 1025, 300, dq, None),
        ("dq_default_big", P64, N64, dq, lambda p: p > 1),
        ("dq_ppl1", 1025, 300, dict(dq, MCL3DL_BEAM_DQ_PPL="1"), lambda p: p == 1),
        ("dq_ppl3", 1025, 301, dict(dq, MCL3DL_BEAM_DQ_PPL="3"), lambda p: p == 3),
        ("dq_ppl16", 63, 300, dict(dq, MCL3DL_BEAM_DQ_PPL="16"), lambda p: p == 16),
        ("auto_below", 513, 511, {}, None),  # P * N = 262 143: pl
        ("auto_at", 512, 512, {}, None),     # P * N = 262 144: dq
    ]


SHAPE_IDS = ["pl_cpg1", "pl_cpg2", "pl_cpg4", "pl_cpg8_cb1", "pl_cb3", "pl_cb_many", "pl_ppl64", "dq_default",
             "dq_default_big", "dq_ppl1", "dq_ppl3", "dq_ppl16", "auto_below", "auto_at"]


def reached(case, sm):
    cid, P, N, env, _ = case
    if env.get("MCL3DL_BEAM") == "pl":
        return pl_shape(P, N, sm)
    if env.get("MCL3DL_BEAM") == "dq":
        return dq_ppl(P, N, sm, int(env.get("MCL3DL_BEAM_DQ_PPL", "0")))
    return None


@pytest.mark.parametrize("caster", W.CASTERS)
@pytest.mark.parametrize("cid", SHAPE_IDS)
def test_launch_shape_equals_reference(ref, hs, E, make, sm, cid, caster):
    case = next(c for c in shape_cases(sm) if c[0] == cid)
    _, P, N, env, want = case
    if want is not None:
        assert want(reached(case, sm)), (cid, reached(case, sm))
    if cid.startswith("auto"):
        assert (P * N >= DQ_MIN_JOB) == (cid == "auto_at")
    w = shape_world(P, N)
    eng = make(w, caster, **env)
    check(ref, hs, E, make, eng, w, caster, env)


def test_launch_shapes_cover_the_selection(sm):
    """On this device the cases above reach every chunks-per-group value, one and three or more CTAs per group (with a
    ray count that is not a multiple of a CTA's rays), 64 rays per lane, P % 32 = 1 and 31, and dq items of 1, 3 and 16
    rays besides the default."""
    cases = shape_cases(sm)
    assert [c[0] for c in cases] == SHAPE_IDS
    pl = [(c, reached(c, sm)) for c in cases if c[3].get("MCL3DL_BEAM") == "pl"]
    assert {s[2] for _, s in pl} == {1, 2, 4, 8}
    assert any(s[1] == 1 for _, s in pl) and any(s[1] >= 3 and c[2] % (8 * s[0]) for c, s in pl)
    assert any(s[0] == 64 for _, s in pl)
    assert {c[1] % 32 for c in cases} >= {1, 31}
    dq = {reached(c, sm) for c in cases if c[3].get("MCL3DL_BEAM") == "dq"}
    assert dq >= {1, 3, 16} and len(dq) >= 4
    print("SM count %d; pl (ppl, cb, cpg): %s; dq ppl: %s" % (sm, sorted({s for _, s in pl}), sorted(dq)))


# ------------------------------------------------------------------ scratch left between calls
@pytest.mark.parametrize("caster", W.CASTERS)
@pytest.mark.parametrize("env,a,b", [({"MCL3DL_BEAM": "pl"}, (31, 21), (1025, 300)),
                                     ({"MCL3DL_BEAM": "dq", "MCL3DL_BEAM_DQ_PPL": "3"}, (65, 7), (1025, 301)),
                                     ({}, (512, 512), (31, 21))])
def test_scratch_is_left_at_zero(ref, hs, E, make, sm, env, a, b, caster):
    """Shape A, then B, then A again on one engine: tickets, partials, tallies and the queue that a call leaves behind
    must not change the next call's records."""
    wa, wb = shape_world(*a), shape_world(*b)
    eng = make(wa, caster, **env)
    first = check(ref, hs, E, make, eng, wa, caster, env)
    check(ref, hs, E, make, eng, wb, caster, env)
    again = check(ref, hs, E, make, eng, wa, caster, env)
    assert first[0].tobytes() == again[0].tobytes() and first[1].tobytes() == again[1].tobytes()


@pytest.mark.parametrize("caster", W.CASTERS)
@pytest.mark.parametrize("P,N", [(1025, 300), (513, 511)])
def test_entry_points_agree(E, make, P, N, caster):
    """measure, beam_status, measure_device and measure_update's records on the same inputs."""
    import torch
    w = shape_world(P, N)
    eng = make(w, caster)
    rec = eng.measure(w["poses"], None, w["scan"], w["origins"]).copy()
    st = eng.beam_status(w["poses"], w["scan"], w["origins"])
    counts = np.stack([(st == 0).sum(1), (st == 1).sum(1), (st == 2).sum(1)], axis=1)
    assert np.array_equal(counts, np.stack([rec["n_short"], rec["n_hit"], rec["n_long"]], axis=1))
    dev = torch.device("cuda:0")
    d_p = torch.from_numpy(np.frombuffer(w["poses"].tobytes(), np.uint8).copy()).to(dev)
    d_b = torch.from_numpy(np.frombuffer(w["scan"].tobytes(), np.uint8).copy()).to(dev)
    d_o = torch.from_numpy(w["origins"].reshape(-1).copy()).to(dev)
    d_out = torch.zeros(P * synth.RESULT.itemsize, dtype=torch.uint8, device=dev)
    eng.measure_device(d_p.data_ptr(), P, 0, 0, d_b.data_ptr(), N, d_o.data_ptr(), len(w["origins"]), d_out.data_ptr())
    torch.cuda.synchronize()
    assert d_out.cpu().numpy().tobytes() == rec.tobytes()
    _, _, rec_u = eng.measure_update(w["poses"], None, w["scan"], w["origins"], np.full(P, 1.0 / P, np.float32),
                                     want_records=True)
    assert rec_u.tobytes() == rec.tobytes()
