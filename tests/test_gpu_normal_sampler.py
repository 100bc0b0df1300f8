"""The normal-weighted sampler on the device (include/mcl3dl_b200.h: mcl3dl_scan_sample_with_normal): the normals,
neighbour counts and fixed-point weights equal the host build of the same functions bit for bit
(tests/hostsim/normal_sampler_hostsim.cpp) and the brute-force port within the stated bars; the samples equal a
restatement of the draw rule over the downloaded weights byte for byte; the call replaces only the sampled scans; every
error leaves the previous samples in place."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from mcl_3dl_b200 import engine, synth
from oracle import normal_sampler_checker as nc
import normal_sampler_worlds as W

pytestmark = pytest.mark.gpu

CLIP = dict(lik_clip=(0.5, 10.0, -2.0, 2.0), beam_clip=(0.5, 4.0, -2.0, 2.0))
COV = np.diag([0.5, 0.02, 0.01, 0.01, 0.01, 0.01])  # ratio 5: max_weight 5


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    return W.load_hostsim(tmp_path_factory.mktemp("nsgpu"))


@pytest.fixture(scope="module")
def port():
    nc.build("port")
    return nc.NormalSamplerChecker("port")


@pytest.fixture(scope="module")
def eng():
    e = engine.Engine((0,))
    yield e
    e.close()


def prepare(eng, name, lik_num=96, beam_num=3, downsample=None):
    raw = W.world(name)
    ds = (0.0, 0.0, 0.0) if name == "nan" else (downsample or (0.1, 0.1, 0.1))
    return eng.scan_prepare(raw, engine.ScanParams(downsample=ds, lik_num_points=lik_num, beam_num_points=beam_num, seed=3,
                                                   **CLIP))


def params_of(cov, rot=(0, 0, 0, 1), **kw):
    w, v = np.linalg.eigh(np.abs(np.asarray(cov, np.float64)[:3, :3]))
    sp = engine.NormalSamplerParams()
    prm = dict(engine.NORMAL_SAMPLER_DEFAULTS, **kw)
    for k in engine.NORMAL_SAMPLER_DEFAULTS:
        setattr(sp, k, prm[k])
    sp.eigen_values[:] = list(w)
    sp.eigen_vector[:] = list(v[:, 2])
    sp.mean_rot[:] = list(rot)
    return sp


@pytest.mark.parametrize("name", W.WORLDS)
def test_normals_equal_the_host_build_and_the_port(eng, hs, port, name):
    prepare(eng, name)
    rot = (0.1, -0.2, 0.3, 0.9)
    info = eng.scan_sample_with_normal(rot, COV, None, 96, 3, seed=5)
    mw, fpc, sh = W.consts(hs, params_of(COV, rot))
    assert info["max_weight"] == mw and info["weight_shift"] == sh
    assert info["fpc_local"].tobytes() == fpc.tobytes()
    for which in (0, 1):
        clipped = eng.scan_get(1 + which)
        nrm, cnt, q = eng.scan_normals(which)
        assert len(nrm) == len(clipped)
        rc, h_nrm, h_cnt, h_q = W.host_normals(hs, clipped, 0.4, fpc, mw, sh)
        assert rc == 0
        assert np.array_equal(cnt, h_cnt)
        assert nrm.tobytes() == h_nrm.tobytes()
        assert np.array_equal(q, h_q)
        assert info["n_normal"][which] == int(np.isfinite(nrm[:, 0]).sum())
        p_nrm, p_cnt = port.normals(clipped, 0.4)
        assert np.array_equal(cnt, p_cnt)
        fin = np.isfinite(p_nrm[:, 0])
        assert np.array_equal(fin, np.isfinite(nrm[:, 0]))
        assert np.allclose(np.linalg.norm(nrm[fin].astype(np.float64), axis=1), 1.0, atol=1e-6)
        gap = W.eigengap(clipped, 0.4)
        good = fin & (gap >= 1e-3)
        a = nrm[good].astype(np.float64)
        b = p_nrm[good].astype(np.float64)
        a /= np.linalg.norm(a, axis=1)[:, None]  # directions: the float storage's length error is not an angle
        b /= np.linalg.norm(b, axis=1)[:, None]
        dots = np.abs((a * b).sum(1))
        assert (1.0 - dots <= 1e-9).all(), (1.0 - dots).max()
        # the weights of the same normals: the device's acos against std::acos, within one unit of q
        want = np.maximum(1, np.rint(port.weights(nrm, fpc, mw) * np.ldexp(1.0, sh))).astype(np.int64)
        assert np.abs(want - q.astype(np.int64)).max(initial=0) <= 1


@pytest.mark.parametrize("name", ("floor_walls", "outliers", "nan"))
def test_samples_equal_the_draw_rule(eng, hs, name):
    info = prepare(eng, name)
    n = [info["n_lik_clipped"], info["n_beam_clipped"]]
    for nums in ([0, 0], [1, 1], [n[0] - 1, n[1] - 1], n, [n[0] + 5, n[1] + 5], [96, 3]):
        nums = [max(0, int(v)) for v in nums]
        got = eng.scan_sample_with_normal((0, 0, 0.2, 0.98), COV, None, nums[0], nums[1], seed=11)
        for which in (0, 1):
            clipped = eng.scan_get(1 + which)
            _, _, q = eng.scan_normals(which)
            idx, rounds, draws = W.restate_sample(hs, q, nums[which], 11, which)
            sample = eng.scan_get(3 + which)
            assert sample.tobytes() == clipped[idx].tobytes(), (nums, which)
            assert got["rounds"][which] == rounds and got["draws"][which] == draws
            assert [got["n_lik"], got["n_beam"]][which] == len(idx)


def test_skewed_weights_need_several_rounds(eng, hs):
    info = prepare(eng, "floor_walls", downsample=(0.05, 0.05, 0.05))
    n = info["n_lik_clipped"]
    num = n - 2
    got = eng.scan_sample_with_normal((0, 0, 0, 1), np.diag([1.0, 0.001, 0.0005]), {"max_weight": 50.0}, num, 0, seed=2)
    _, _, q = eng.scan_normals(0)
    idx, rounds, draws = W.restate_sample(hs, q, num, 2, 0)
    assert rounds >= 2 and got["rounds"][0] == rounds and got["draws"][0] == draws
    assert eng.scan_get(3).tobytes() == eng.scan_get(1)[idx].tobytes()
    assert got["n_beam"] == 0 and len(eng.scan_get(4)) == 0


def test_empty_clipped_cloud(eng):
    far = W.world("cylinder")
    far["x"] += 100.0
    eng.scan_prepare(far, engine.ScanParams(lik_num_points=96, beam_num_points=3, **CLIP))
    got = eng.scan_sample_with_normal((0, 0, 0, 1), COV, None, 96, 3, seed=1)
    assert got["n_lik"] == 0 and got["n_beam"] == 0 and got["n_normal"] == [0, 0]
    assert len(eng.scan_get(3)) == 0 and len(eng.scan_normals(0)[0]) == 0


def test_prepared_update_and_untouched_state(eng):
    s = synth.scene(30_000, 64, 96, 3, seed=4)
    eng.set_map(s["map"], engine.LikParams(dist_weight=(1, 1, 5)),
                engine.beam_params_from_reference(num_points_default=3, dda_grid_size=0.2))
    st = np.zeros(64, dtype=synth.STATE)
    st["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], axis=1)
    st["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], axis=1)
    prior = np.full(64, 1.0 / 64, np.float32)
    raw = np.concatenate([s["map"][:20000], W.world("floor_walls")])
    raw["label"] = 0
    eng.scan_prepare(raw, engine.ScanParams(lik_num_points=96, beam_num_points=3, seed=9, **CLIP))
    before = [eng.scan_get(k).tobytes() for k in range(3)]
    eng.particles_set(st, prior)
    res_before = [a.tobytes() for a in eng.particles_get()]
    eng.scan_sample_with_normal((0, 0, 0, 1), COV, None, 96, 3, seed=4)
    assert [eng.scan_get(k).tobytes() for k in range(3)] == before
    assert [a.tobytes() for a in eng.particles_get()] == res_before
    lik, beam = eng.scan_get(3), eng.scan_get(4)
    origins = np.zeros((1, 3), np.float32)
    a = eng.particles_measure_update_prepared(origins, 0.0)
    got_a = [x.tobytes() for x in eng.particles_get()]
    eng.particles_set(st, prior)
    b = eng.particles_measure_update(lik, beam, origins, 0.0)
    assert a == b
    assert [x.tobytes() for x in eng.particles_get()] == got_a


def test_errors_leave_the_previous_samples(eng):
    fresh = engine.Engine((0,))
    with pytest.raises(engine.EngineError) as e:
        fresh.scan_sample_with_normal((0, 0, 0, 1), COV)   # no scan_prepare
    assert e.value.code == -1
    with pytest.raises(engine.EngineError):
        fresh.scan_normals(0)
    fresh.close()
    prepare(eng, "cylinder")
    eng.scan_sample_with_normal((0, 0, 0, 1), COV, None, 50, 3, seed=8)
    keep = [eng.scan_get(3).tobytes(), eng.scan_get(4).tobytes(), eng.scan_normals(0)[2].tobytes()]
    # a null engine or null params, through the C ABI itself
    L = eng.L
    info = engine.NormalSamplerInfo()
    assert L.mcl3dl_scan_sample_with_normal(None, C.byref(params_of(COV)), C.byref(info)) == -1
    assert L.mcl3dl_scan_sample_with_normal(eng.h, None, C.byref(info)) == -1
    n = C.c_size_t(0)
    assert L.mcl3dl_scan_normals(None, 0, None, None, None, 0, C.byref(n)) == -1
    assert [eng.scan_get(3).tobytes(), eng.scan_get(4).tobytes(), eng.scan_normals(0)[2].tobytes()] == keep
    ev = np.linalg.eigh(np.abs(COV[:3, :3]))
    bad = [dict(params={"normal_search_range": 0.0}), dict(params={"normal_search_range": float("inf")}),
           dict(params={"max_weight": 0.0}), dict(params={"max_weight": float("nan")}),
           dict(params={"perform_weighting_ratio": float("nan")}), dict(params={"max_weight_ratio": float("inf")}),
           dict(vals=(0.0, float("nan"), 1.0)), dict(vec=(0.0, float("inf"), 1.0)), dict(rot=(0.0, 0.0, float("nan"), 1.0))]
    for b in bad:
        with pytest.raises(engine.EngineError) as e:
            eng.scan_sample_with_normal_eigen(b.get("rot", (0, 0, 0, 1)), b.get("vals", ev[0]), b.get("vec", ev[1][:, 2]),
                                              b.get("params"), 50, 3, 8)
        assert e.value.code == -1, b
        assert [eng.scan_get(3).tobytes(), eng.scan_get(4).tobytes(), eng.scan_normals(0)[2].tobytes()] == keep
    # an outlier far out in an unbounded clip window: the neighbour grid would need 2^31 cells or more
    raw = W.world("cylinder")
    far = raw[:2].copy()
    far["x"] = (3.0e4, -3.0e4)
    far["y"] = (3.0e4, -3.0e4)
    far["z"] = (1.0e4, -1.0e4)
    eng.scan_prepare(np.concatenate([raw, far]), engine.ScanParams(lik_num_points=50, beam_num_points=3, seed=3,
                                                                   lik_clip=(0.0, 1e9, -1e9, 1e9), beam_clip=CLIP["beam_clip"]))
    keep = [eng.scan_get(3).tobytes(), eng.scan_get(4).tobytes()]   # the uniform sampler's scans
    with pytest.raises(engine.EngineError) as e:
        eng.scan_sample_with_normal((0, 0, 0, 1), COV, None, 50, 3, seed=8)
    assert e.value.code == -5
    assert [eng.scan_get(3).tobytes(), eng.scan_get(4).tobytes()] == keep
    with pytest.raises(engine.EngineError):
        eng.scan_normals(2)


def test_adapter_parity_program():
    """MeasurementBatcher::sampleWithNormalPrepared with the reference filter's expectation() and covariance(1.0, 1.0)
    against the port: max_weight, fpc_local, the weight shift, neighbour counts, weights and both samples
    (oracle/normal_sampler_parity_test.cpp)."""
    exe = nc.lib_path("parity")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/normal_sampler_parity_test not built (needs a checkout of the reference at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "NORMAL SAMPLER PARITY OK" in r.stdout
