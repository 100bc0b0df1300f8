"""The normal-weighted sampler without a GPU.
  - reference == port: the reference's own PointCloudSamplerWithNormal (oracle/_ref, against oracle/shim_ns) and the
    port restatement give the same sampled points bit for bit, over seeds, every branch of the max_weight ladder, the
    non-finite case and the edge sizes.
  - host build == port: the ns_* functions of mcl_3dl_b200/csrc/scan_funcs.cuh compiled for the host
    (tests/hostsim/normal_sampler_hostsim.cpp) give the port's neighbour counts exactly, its normals within
    1 - |n . n'| <= 1e-9 where the eigengap allows, and weights within one unit of q.
  - the neighbour grid keeps every neighbour at cell boundaries, and the draw rule draws in proportion to q."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

from mcl_3dl_b200 import engine, synth
from oracle import normal_sampler_checker as nc
import normal_sampler_worlds as W

F = np.float32


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    return W.load_hostsim(tmp_path_factory.mktemp("nshost"))


@pytest.fixture(scope="module")
def port():
    nc.build("port")
    return nc.NormalSamplerChecker("port")


@pytest.fixture(scope="module")
def ref():
    if not nc.build("reference"):
        pytest.skip("reference checker not built (no reference checkout)")
    return nc.NormalSamplerChecker("reference")


def cloud(n, seed):
    rng = np.random.default_rng(seed)
    xyz = np.c_[rng.uniform(-2, 2, n), rng.uniform(-2, 2, n), 0.05 * rng.standard_normal(n)]
    xyz[: n // 3, 2] = xyz[: n // 3, 0] * 0.8  # a tilted patch, so the normals differ
    p = np.zeros(n, synth.POINT)
    p["x"], p["y"], p["z"] = xyz.T.astype(F)
    p["label"] = np.arange(n) % 7
    return p


# eigenvalue ratios sqrt(l2 / l1): 1 (below 2: max_weight 1), 3 (interpolated), 10 (above 5: max_weight), and 0 / 0
COVS = {"flat": np.diag([0.2, 0.2, 0.1]), "interp": np.diag([0.9, 0.1, 0.05]), "strong": np.diag([1.0, 0.01, 0.002]),
        "dense": np.array([[0.5, -0.2, 0.05], [-0.2, 0.3, 0.01], [0.05, 0.01, 0.02]]), "zero": np.zeros((3, 3))}


@pytest.mark.parametrize("case", sorted(COVS))
def test_reference_equals_port(ref, port, case):
    pts = cloud(400, 1)
    n = len(pts)
    nums = (1,) if case == "zero" else (0, 1, 37, n - 1, n, n + 5)  # zero: NaN weights, only num = 1 ends
    for seed in (0, 1, 12345):
        for num in nums:
            for rot in ((0, 0, 0, 1), (0.2, -0.1, 0.4, 0.87)):
                a, ca = port.sample(pts, COVS[case], rot, num, seed)
                b, _ = ref.sample(pts, COVS[case], rot, num, seed)
                assert a.tobytes() == b.tobytes(), (case, seed, num)
                assert len(a) == (min(num, n))
    e, _ = ref.sample(np.zeros(0, synth.POINT), COVS["strong"], (0, 0, 0, 1), 5, 0)
    assert len(e) == 0


def _params(vals, vec, rot, **kw):
    sp = engine.NormalSamplerParams()
    prm = dict(engine.NORMAL_SAMPLER_DEFAULTS, **kw)
    for k in engine.NORMAL_SAMPLER_DEFAULTS:
        setattr(sp, k, prm[k])
    sp.eigen_values[:] = list(vals)
    sp.eigen_vector[:] = list(vec)
    sp.mean_rot[:] = list(rot)
    return sp


@pytest.mark.parametrize("case", sorted(COVS))
def test_host_constants_equal_the_port(hs, port, case):
    pts = cloud(50, 2)
    for rot in ((0, 0, 0, 1), (0.2, -0.1, 0.4, 0.87), (0.0, 0.0, 0.0, 2.0)):
        vals, vecs = port.eigen(COVS[case].astype(F))
        mw, fpc, sh = W.consts(hs, _params(vals, vecs[:, 2], rot))
        _, c = port.sample(pts, COVS[case], rot, 1, 0)   # one draw: the zero case's NaN weights end after it
        want_mw = c[0] if np.isfinite(c[0]) else 1.0   # the non-finite rule
        assert mw == want_mw
        assert fpc.tobytes() == c[1:].astype(F).tobytes()
        assert sh == 32 - int(np.ceil(np.log2(max(1.0, mw))))
    assert W.consts(hs, _params((0, 0, 0), (0, 0, 1), (0, 0, 0, 1)))[0] == 1.0
    assert W.consts(hs, _params((1, 1, 4), (0, 0, 1), (0, 0, 0, 1), perform_weighting_ratio=2.0, max_weight_ratio=2.0))[0] == 1.0


@pytest.mark.parametrize("name", W.WORLDS)
def test_host_build_equals_port(hs, port, name):
    pts = W.world(name)[::2]
    fpc = np.array([0.6, 0.0, 0.8], F)
    for mw in (5.0, 1.0, 0.5, 3.7):
        sh = 32 - int(np.ceil(np.log2(max(1.0, mw))))
        rc, nrm, cnt, q = W.host_normals(hs, pts, 0.4, fpc, mw, sh)
        assert rc == 0
        p_nrm, p_cnt = port.normals(pts, 0.4)
        assert np.array_equal(cnt, p_cnt)
        fin = np.isfinite(p_nrm[:, 0])
        assert np.array_equal(fin, np.isfinite(nrm[:, 0]))
        assert np.array_equal(fin, cnt >= 3)
        assert np.allclose(np.linalg.norm(nrm[fin].astype(np.float64), axis=1), 1.0, atol=1e-6)
        gap = W.eigengap(pts, 0.4)
        good = fin & (gap >= 1e-3)
        a = nrm[good].astype(np.float64)
        b = p_nrm[good].astype(np.float64)
        a /= np.linalg.norm(a, axis=1)[:, None]
        b /= np.linalg.norm(b, axis=1)[:, None]
        assert (1.0 - np.abs((a * b).sum(1)) <= 1e-9).all()
        want = np.maximum(1, np.rint(port.weights(nrm, fpc, mw) * np.ldexp(1.0, sh))).astype(np.int64)
        assert np.abs(want - q.astype(np.int64)).max(initial=0) <= 1
        assert q.max(initial=0) <= 2 ** 32
        assert (q[~fin] == np.uint64(np.ldexp(1.0, sh))).all()   # NaN normal: weight 1


def test_acos_against_libm(hs):
    a = np.r_[np.linspace(0, 1, 200001), 0.5, np.nextafter(0.5, 1), 1.0 - 2.0 ** -52, 2.0 ** -30]
    out = np.zeros_like(a)
    hs.hostsim_ns_acos(a.ctypes.data_as(C.c_void_p), len(a), out.ctypes.data_as(C.c_void_p))
    ref = np.arccos(a)
    assert np.all(np.abs(out - ref) <= 4 * np.spacing(np.maximum(ref, 1e-300)) + 1e-16)


@pytest.mark.parametrize("r", (0.4, 0.25, 1.0))
@pytest.mark.parametrize("base", (0.0, 3.3, -7.9, 250.0, -1000.0))
def test_grid_keeps_neighbours_at_cell_edges(hs, port, r, base):
    """Pairs at r (1 -/+ 2^-20) apart straddle the grid's cell boundaries on each axis, at positive and negative
    coordinates: the neighbour counts equal the brute-force ones."""
    edge, inv, mn_b, div, cells = C.c_float(0), np.zeros(3, F), np.zeros(3, np.int32), np.zeros(3, np.uint32), C.c_uint32(0)
    lo, hi = np.full(3, base - 5, F), np.full(3, base + 5, F)
    assert hs.hostsim_ns_lattice(r, lo.ctypes.data_as(C.c_void_p), hi.ctypes.data_as(C.c_void_p), C.byref(edge),
                                 inv.ctypes.data_as(C.c_void_p), mn_b.ctypes.data_as(C.c_void_p),
                                 div.ctypes.data_as(C.c_void_p), C.byref(cells)) == 1
    e = float(edge.value)
    assert r * (1 + 2 ** -11) < e <= r * (1 + 2 ** -9)
    xyz = [lo, hi]
    k0 = int(np.floor((base - 1) / e))
    for c in range(k0, k0 + 6):
        b = F(c * e)  # near a cell boundary
        for d in (F(r * (1 - 2 ** -20)), F(r * (1 + 2 ** -20))):
            for axis in range(3):
                for off in (F(-1e-6), F(0), F(1e-6), F(-d / 2), F(d / 3)):
                    p = np.full(3, base, F)
                    q = p.copy()
                    p[axis] = F(b + off)
                    q[axis] = F(p[axis] + d)
                    xyz += [p, q]
    xyz = np.array(xyz, F)
    pts = np.zeros(len(xyz), synth.POINT)
    pts["x"], pts["y"], pts["z"] = xyz.T
    rc, _, cnt, _ = W.host_normals(hs, pts, r, np.zeros(3, F), 1.0, 32)
    assert rc == 0
    _, p_cnt = port.normals(pts, r)
    assert np.array_equal(cnt, p_cnt)
    assert cnt.max() >= 2


def test_draw_rule_frequencies(hs):
    rng = np.random.default_rng(7)
    q = rng.integers(1, 2 ** 32, 50, dtype=np.uint64)
    q[:5] = [1, 2 ** 32, 2 ** 31, 3, 2 ** 30]
    cum = np.ascontiguousarray(np.cumsum(q, dtype=np.uint64))
    idx = W.host_draws(hs, cum, 2024, 0, 0, 1_000_000)
    f = np.bincount(idx, minlength=len(q))
    expect = q.astype(np.float64) / float(cum[-1]) * len(idx)
    keep = expect >= 5
    chi2 = (((f - expect) ** 2) / expect)[keep].sum()
    assert stats.chi2.sf(chi2, keep.sum() - 1) > 1e-3
    assert f[0] <= 1   # probability 2^-37 per draw


def test_restated_selection_is_distinct_and_in_draw_order(hs):
    q = np.ones(100, np.uint64) * np.uint64(2 ** 20)
    q[7] = np.uint64(2 ** 28)
    idx, rounds, draws = W.restate_sample(hs, q, 60, 5, 1)
    assert len(np.unique(idx)) == 60 and idx[0] == W.host_draws(hs, np.cumsum(q, dtype=np.uint64), 5, 1, 0, 1)[0]
    assert rounds == 1 and draws == 2048
