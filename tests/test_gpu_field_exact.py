"""Field mode bit for bit: the node volume, the corner layout, the trilinear lookup and whole scans, against the numpy
float32 restatement of tests/field_restate.py.

Field mode is inexact only against the exact nearest-neighbour distance; the kernels themselves are deterministic float
code (-fmad=false), so each step is held to its restatement exactly:
1. every node of the volume field_nodes_kernel builds, on maps with regular, wide and overflow NN-field cells, at three
   dist_weights and for each NN-field radius (likelihood only, DDA beam, KD beam with and without its second search);
   the node volume is the device NN field's only per-query output, and every node lies on a voxel corner;
2. one eval per record over an uploaded volume of random values: field_expand_kernel's corner order and pitch and
   field_dist's cell index, fractions and bounds, at nodes, one coordinate ulp either side of them, the upper faces,
   outside the lattice, past int range and at NaN;
3. whole scans at every launch shape of lik_kernel_field (TPP 8 .. 256, the staged and the global scan): match_cnt bit
   for bit, score_like within test_gpu_lik_exact.py's bar for the particle-major kernels' summation order, from the
   per-point terms of the same device functions compiled for the host (tests/hostsim/field_hostsim.cpp);
4. restaging after set_map, map_append and switching the mode off and on: the same bytes as a fresh engine;
5. the error codes of field_upload and field_mode.
Check (1) of test_gpu_field.py (sampled node distances within a tolerance) is superseded by 1. here; its check (2), the
deviation of field-mode scores from the exact nearest-neighbour scores, stays the reported, loosely bounded measure.
"""
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import field_restate as FR
from mcl_3dl_b200 import synth
from test_field_on_host import SRC, load, random_volume
from test_gpu_lik_exact import TPP_NF, U, depth, exact_row_sums

pytestmark = pytest.mark.gpu
F = np.float32
R, FLAT, W = 0.2, 0.05, 5.0
DWS = [(1, 1, 1), (1, 1, 5), (0.7, 1.3, 2.9)]
BEAMS = [FR.LIK, FR.DDA, FR.KD_R2, FR.KD_R1]
BLOCK, NF_U, NF_MINB = 256, 4, 4     # kBlockThreads, kNfU, kNfCtasPerSm
MAX_STAGED = 200 * 1024 // 2         # lik_kernel_field stages scans of up to kMaxStagedBytes / 2
ERR_INVALID_ARG, ERR_NO_MAP, ERR_TOO_LARGE = -1, -2, -5


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fieldhs") / "libfieldhs.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return load(so)


@pytest.fixture
def make_engine(eng_mod, monkeypatch):
    """Engines with the given environment (read at creation), closed after the test."""
    made = []

    def make(devices=(0,), **env):
        for k in ("MCL3DL_NNF", "MCL3DL_LIK_SHARE", "MCL3DL_LIK_MODE", "MCL3DL_NNF_KD_R2", "MCL3DL_FIELD_MAX_MB"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        e = eng_mod.Engine(devices)
        made.append(e)
        return e
    yield make
    for e in made:
        e.close()


def beam_params(eng_mod, beam):
    if beam == FR.LIK:
        return None
    return eng_mod.beam_params_from_reference(num_points_default=8, dda_grid_size=0.2,
                                              use_raycast_using_dda=beam == FR.DDA)


def engine_for(make_engine, eng_mod, xyz, dw, beam, **env):
    if beam == FR.KD_R1:
        env["MCL3DL_NNF_KD_R2"] = "0"
    e = make_engine(**env)
    e.set_map(synth.make_points(xyz), eng_mod.LikParams(W, R, FLAT, dw), beam_params(eng_mod, beam))
    return e


# ------------------------------------------------------------------ maps
def surface_map():
    """A voxel-filtered surface map (floor, ceiling, walls; one point per 0.1 m voxel): regular NN-field cells."""
    mp, _ = synth.warehouse_map(8000, seed=5)
    return np.stack([mp["x"], mp["y"], mp["z"]], axis=1).astype(F)


def wide_map():
    """The sparse volume of test_gpu_parity.py::test_wide_cells_of_the_nn_field: wide cells."""
    return np.random.default_rng(92).uniform(0.0, 1.0, (600, 3)).astype(F)


def dense_map():
    """A dense raw cloud (test_selection_overflow_cells): overflow cells."""
    pts = np.random.default_rng(91).uniform(0.0, 1.0, (120_000, 3)).astype(F)
    return np.vstack([pts, [[-0.5, -0.5, -0.5], [1.5, 1.5, 1.5]]]).astype(F)


def box_map():
    """600 random points in a 1 x 0.6 x 0.3 box: a lattice with three different extents."""
    return (np.random.default_rng(93).uniform(0.0, 1.0, (600, 3)) * [1.0, 0.6, 0.3]).astype(F)


MAPS = {"surface": surface_map, "wide": wide_map, "dense": dense_map}


def lattice_of(e, xyz, dw, beam):
    """The engine's lattice, checked against the restated one; returns (origin, edge, node dims, inv_e, clamp)."""
    _, org, edge, dims = e.field_nodes(download=False)
    clamp = FR.field_radius(R, beam)
    want_dims, want_org, want_edge, inv_e = FR.lattice(xyz, dw, clamp)
    assert dims == want_dims and org.tobytes() == want_org.tobytes() and F(edge) == want_edge
    assert F(F(1) / inv_e) == F(edge)   # the restated inv_e is the one behind the returned edge
    return org, F(edge), dims, inv_e, clamp


# ------------------------------------------------------------------ 1. every node
@pytest.mark.parametrize("beam", BEAMS)
@pytest.mark.parametrize("dw", DWS)
@pytest.mark.parametrize("name", list(MAPS))
def test_every_node(eng_mod, make_engine, name, dw, beam):
    xyz = MAPS[name]()
    e = engine_for(make_engine, eng_mod, xyz, dw, beam)
    info = e.nn_field_info()
    if name == "dense":
        assert info["overflow_cells"] > 0   # nodes whose search falls back to the CSR window search
    elif dw == (1, 1, 1) and beam != FR.KD_R2:   # (the KD search's wider field overflows a few cells of every map)
        assert info["overflow_cells"] == 0
        if name == "wide":
            assert info["wide_cells"] > 0
    e.field_mode(True)
    org, edge, dims, inv_e, clamp = lattice_of(e, xyz, dw, beam)
    nodes = e.field_nodes()[0]
    want = FR.node_values(FR.rescaled(xyz, dw), org, edge, dims, clamp)
    bad = np.argwhere(nodes.view(np.uint32) != want.view(np.uint32))
    print("%s dw=%s %s: %d nodes (%d inside the clamp), field %s; %d differ"
          % (name, dw, beam, nodes.size, int((want < clamp).sum()), info, len(bad)))
    assert len(bad) == 0, (len(bad), [(tuple(b), nodes[tuple(b)], want[tuple(b)]) for b in bad[:4]])
    assert (want < clamp).sum() > 100 and (want == clamp).any()


# ------------------------------------------------------------------ 2. one eval per record
def one_eval_poses(q_pos):
    """Particles at q_pos with the identity rotation: with the one-point scan (0, 0, 0) each record is one eval at
    float(q_pos * dist_weight) (test_field_on_host.py::test_one_eval_per_record)."""
    return synth.make_poses(q_pos, np.tile(np.array([0, 0, 0, 1], F), (len(q_pos), 1)))


@pytest.mark.parametrize("dw", [(1, 1, 1), (1, 1, 5)])
def test_lookup_one_eval_per_record(eng_mod, make_engine, dw):
    xyz = box_map()
    e = engine_for(make_engine, eng_mod, xyz, dw, FR.KD_R2)   # clamp 0.27 > match_dist_min: matches and misses
    e.field_mode(True)
    org, edge, dims, inv_e, clamp = lattice_of(e, xyz, dw, FR.KD_R2)
    assert len(set(dims)) == 3
    rng = np.random.default_rng(301)
    V = random_volume(rng, (dims[0] - 1, dims[1] - 1, dims[2] - 1), clamp, FLAT)
    e.field_upload(V)
    assert e.field_nodes()[0].tobytes() == V.tobytes()
    q = FR.edge_queries(dims, org, edge, inv_e, rng, n=20000)
    pos = (q / np.asarray(dw, F)).astype(F)
    pos = np.vstack([pos, [[np.nan, np.nan, np.nan], [np.nan, 0.5, 0.1]]]).astype(F)
    got = e.measure(one_eval_poses(pos), synth.make_points(np.zeros((1, 3), F)), None, None)
    qs = (pos * np.asarray(dw, F)).astype(F)
    score, cnt = FR.one_eval_records(V, org, inv_e, clamp, qs, R, FLAT, W)
    bad = np.nonzero((got["score_like"].view(np.uint32) != score.view(np.uint32)) | (got["match_cnt"] != cnt))[0]
    assert len(bad) == 0, (len(bad), qs[bad[:4]], got[bad[:4]], score[bad[:4]], cnt[bad[:4]])
    assert got["match_cnt"][-2:].tolist() == [0, 0] and got["score_like"][-2:].tolist() == [0.0, 0.0]   # NaN: no match
    # the lookup's edges were reached: tx on node 0, both sides of the upper faces, outside, matches and misses
    t = ((qs[:-2] - org).astype(F) * inv_e).astype(F)
    n = np.array(dims) - 1
    assert (t == 0).any(axis=0).all() and ((t < n) & (t > n - 1e-3)).any(axis=0).all()
    assert ((t >= n) & (t < n + 1e-3)).any(axis=0).all() and (t > 2.0 ** 31).any(axis=0).all()
    assert 1000 < cnt.sum() < len(cnt) - 1000


# ------------------------------------------------------------------ 3. whole scans at every launch shape
def pick_tpp_nf(P, N, sm):
    """engine.cu pick_tpp_nf."""
    slots = sm * NF_MINB

    def ctas(t):
        return (P * t + BLOCK - 1) // BLOCK
    tpp = 8
    while tpp < BLOCK and tpp * NF_U < N:
        tpp *= 2
    while tpp < BLOCK and tpp < N and ctas(tpp) * 2 <= sm:
        tpp *= 2
    while tpp > 8 and slots < ctas(tpp) < 2 * slots:
        tpp //= 2
    return tpp


def field_shape(P, N, sm):
    """launch_lik_field_t: (TPP, STAGED, more groups than CTAs)."""
    tpp = pick_tpp_nf(P, N, sm)
    ppb = BLOCK // tpp
    groups = (P + ppb - 1) // ppb
    grid = max(1, min(groups, sm * NF_MINB))
    return tpp, N * 16 <= MAX_STAGED and (ppb >= 4 or groups > grid), groups > grid


SHAPES = [(1, 1), (37, 1), (1, 96), (2000, 48), (300, 32), (301, 64), (300, 128), (300, 256), (100, 512),
          (100, 1024), (2000, 1024), (40000, 16), (50, 7000), (3000, 7000), (64, 0)]


@pytest.fixture(scope="module")
def shape_scene():
    return synth.scene(20_000, 40000, 7000, 0, seed=311)


def check_scan(hs, got, poses, scan, V, org, inv_e, clamp, dw):
    """The records of a whole scan: match_cnt bit for bit, score_like within gamma_D * sum |T| of the exact sum S
    (test_gpu_lik_exact.py's bar for lik_kernel_nf, whose lane and reduction order lik_kernel_field shares); T and M
    from the host build of the device functions over the same node volume.  Returns the number of matches."""
    P, N = len(poses), len(scan)
    if N == 0:
        assert np.all(got["score_like"] == 1.0) and np.all(got["match_cnt"] == 0)
        return 0
    cells = FR.expand(V)
    dims = np.array([V.shape[2] - 1, V.shape[1] - 1, V.shape[0] - 1], np.int32)
    T, M = np.zeros((P, N), F), np.zeros((P, N), np.uint8)
    p = np.ascontiguousarray(poses)
    s = np.ascontiguousarray(scan)
    hs.hostsim_field_terms(p.ctypes.data, P, s.ctypes.data, N, cells.ctypes.data, dims.ctypes.data,
                           np.asarray(org, F).ctypes.data, F(inv_e), F(clamp), np.asarray(dw, F).ctypes.data,
                           F(R), F(FLAT), F(W), T.ctypes.data, M.ctypes.data)
    M = M.astype(bool)
    assert np.array_equal(got["match_cnt"], M.sum(axis=1).astype(np.uint32))
    S = exact_row_sums(T)
    A = exact_row_sums(np.abs(T))
    D = depth(N, TPP_NF)
    g = D * U / (1 - D * U)
    for i in range(P):
        assert abs(Fraction(float(got["score_like"][i])) - S[i]) <= g * A[i], (i, float(got["score_like"][i]), float(S[i]))
    return int(M.sum())


@pytest.mark.parametrize("volume", ["device", "random"])
def test_launch_shapes(eng_mod, make_engine, hs, sm_count, shape_scene, volume):
    s = shape_scene
    xyz = np.stack([s["map"]["x"], s["map"]["y"], s["map"]["z"]], axis=1).astype(F)
    dw = (1, 1, 5)
    e = engine_for(make_engine, eng_mod, xyz, dw, FR.KD_R2)
    e.field_mode(True)
    org, edge, dims, inv_e, clamp = lattice_of(e, xyz, dw, FR.KD_R2)
    if volume == "random":
        e.field_upload(random_volume(np.random.default_rng(312), (dims[0] - 1, dims[1] - 1, dims[2] - 1), clamp, FLAT))
    V = e.field_nodes()[0]
    shapes = [field_shape(P, N, sm_count) for P, N in SHAPES]
    assert {t for t, _, _ in shapes} == set(TPP_NF)
    assert {st for _, st, _ in shapes} == {True, False} and any(w for _, _, w in shapes)
    matched = evals = 0
    for (P, N), sh in zip(SHAPES, shapes):
        poses, scan = s["particles"][:P], s["lik"][:N]
        got = e.measure(poses, scan, None, None)
        try:
            matched += check_scan(hs, got, poses, scan, V, org, inv_e, clamp, dw)
        except AssertionError as err:
            raise AssertionError("P=%d N=%d (TPP, staged, waves) = %s: %s" % (P, N, sh, err)) from None
        evals += P * N
    print("%s volume: shapes %s, %d of %d evals matched" % (volume, shapes, matched, evals))
    assert 0 < matched < evals


# ------------------------------------------------------------------ 4. restaging
def fresh(make_engine, eng_mod, xyz, dw, poses, scan):
    e = engine_for(make_engine, eng_mod, xyz, dw, FR.KD_R2)
    e.field_mode(True)
    out = (e.field_nodes()[0].tobytes(), e.measure(poses, scan, None, None).tobytes())
    e.close()
    return out


def test_restaging(eng_mod, make_engine):
    dw = (1, 1, 5)
    s = synth.scene(20_000, 500, 300, 0, seed=321)
    big = np.stack([s["map"]["x"], s["map"]["y"], s["map"]["z"]], axis=1).astype(F)
    lo, hi = big.min(axis=0), big.max(axis=0)
    small = big[(big[:, 0] < lo[0] + 0.6 * (hi[0] - lo[0]))]
    poses, scan = s["particles"], s["lik"]

    def state(e):
        return e.field_nodes()[0].tobytes(), e.measure(poses, scan, None, None).tobytes()
    e = engine_for(make_engine, eng_mod, small, dw, FR.KD_R2)
    e.field_mode(True)
    assert state(e) == fresh(make_engine, eng_mod, small, dw, poses, scan)
    dims_small = e.field_nodes(download=False)[3]
    # a larger map: the lattice grows, the pitched node volume is allocated anew
    e.set_map(synth.make_points(big), eng_mod.LikParams(W, R, FLAT, dw), beam_params(eng_mod, FR.KD_R2))
    assert e.field_nodes(download=False)[3][0] > dims_small[0]
    assert state(e) == fresh(make_engine, eng_mod, big, dw, poses, scan)
    # an append inside the map's box (the incremental NN-field update), then one past it (the full rebuild)
    rng = np.random.default_rng(322)
    inner = (lo + rng.uniform(0.2, 0.8, (300, 3)) * (hi - lo)).astype(F)
    assert e.map_append(synth.make_points(inner))["incremental"] == 1
    cur = np.vstack([big, inner])
    assert state(e) == fresh(make_engine, eng_mod, cur, dw, poses, scan)
    outer = (hi + rng.uniform(0.0, 0.5, (100, 3))).astype(F)
    assert e.map_append(synth.make_points(outer))["incremental"] == 0
    cur = np.vstack([cur, outer])
    want = fresh(make_engine, eng_mod, cur, dw, poses, scan)
    assert state(e) == want
    # off: the exact search; on again: the same volume and records
    e.field_mode(False)
    exact = engine_for(make_engine, eng_mod, cur, dw, FR.KD_R2)
    assert e.measure(poses, scan, None, None).tobytes() == exact.measure(poses, scan, None, None).tobytes()
    e.field_mode(True)
    assert state(e) == want


def test_restaging_on_two_devices(eng_mod, make_engine):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    dw = (1, 1, 5)
    s = synth.scene(20_000, 500, 300, 0, seed=331)
    xyz = np.stack([s["map"]["x"], s["map"]["y"], s["map"]["z"]], axis=1).astype(F)
    e = make_engine(devices=(0, 1))
    e.set_map(s["map"], eng_mod.LikParams(W, R, FLAT, dw), beam_params(eng_mod, FR.KD_R2))
    e.field_mode(True)
    nodes, rec = fresh(make_engine, eng_mod, xyz, dw, s["particles"], s["lik"])
    assert e.field_nodes()[0].tobytes() == nodes
    assert e.measure(s["particles"], s["lik"], None, None).tobytes() == rec


# ------------------------------------------------------------------ 5. errors
def test_errors(eng_mod, make_engine):
    e = make_engine()
    with pytest.raises(eng_mod.EngineError) as err:
        e.field_upload(np.zeros((4, 4, 4), F))
    assert err.value.code == ERR_NO_MAP
    xyz = surface_map()
    dw = (1, 1, 5)
    e.set_map(synth.make_points(xyz), eng_mod.LikParams(W, R, FLAT, dw), None)
    e.field_mode(True)
    _, _, _, dims = e.field_nodes(download=False)
    for bad in [(dims[2], dims[1], dims[0] + 1), (dims[2] - 1, dims[1], dims[0]), (dims[0], dims[1], dims[2])]:
        with pytest.raises(eng_mod.EngineError) as err:
            e.field_upload(np.zeros(bad, F))
        assert err.value.code == ERR_INVALID_ARG
    # a volume above MCL3DL_FIELD_MAX_MB: TOO_LARGE, and the engine keeps serving exact records
    s = synth.scene(20_000, 200, 96, 0, seed=341)
    small = make_engine(MCL3DL_FIELD_MAX_MB="1")
    small.set_map(synth.make_points(xyz), eng_mod.LikParams(W, R, FLAT, dw), None)
    cells = np.prod([d - 1 for d in dims])
    assert cells * 32 > 1 << 20
    with pytest.raises(eng_mod.EngineError) as err:
        small.field_mode(True)
    assert err.value.code == ERR_TOO_LARGE
    exact = make_engine()
    exact.set_map(synth.make_points(xyz), eng_mod.LikParams(W, R, FLAT, dw), None)
    want = exact.measure(s["particles"], s["lik"], None, None)
    assert small.measure(s["particles"], s["lik"], None, None).tobytes() == want.tobytes()
