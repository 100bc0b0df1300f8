"""mcl3dl_match_output on an H100: the node's matched / unmatched clouds (src/mcl_3dl.cpp:761-805) equal, byte for byte,
the points the CPU checkers classify, transformed by mcl3dl_cpu_transform_point (the port always, the reference's own
loop where build() made oracle/_ref/libmcl3dl_match_ref.so).  Non-finite transformed points are compared as non-finite: the device and x86 write
different NaN payloads.  Workloads: the node's defaults on the synthetic c2-sized map with off-map points injected, and
1-1.5 m chunks where the chunk rule changes classes relative to a search over every map point."""
import os
import subprocess

import numpy as np
import pytest

from oracle import cpu_checker as cc
from oracle import match_checker as mc
from mcl_3dl_b200 import engine, synth
from test_match_output_cpu import match_scene, transformed, global_classes, MATCHED, UNMATCHED

pytestmark = pytest.mark.gpu


def expected(cpu_map, port, pose, pts, match_dist, unmatch_dist):
    cls = cpu_map.match_output(pose, pts, match_dist, unmatch_dist)
    xyz = transformed(port, pose, pts)
    out = cc.points(xyz, pts["label"])
    return out[cls == MATCHED], out[cls == UNMATCHED], cls


def assert_same_cloud(got, want):
    assert len(got) == len(want)
    g = np.stack([got["x"], got["y"], got["z"]], 1)
    w = np.stack([want["x"], want["y"], want["z"]], 1)
    fin = np.all(np.isfinite(w), axis=1)
    assert got[fin].tobytes() == want[fin].tobytes()
    assert np.array_equal(np.isnan(g), np.isnan(w))
    assert np.array_equal(g[~np.isnan(g)], w[~np.isnan(w)])
    assert np.array_equal(got["label"], want["label"])


def checkers():
    out = [mc.MatchChecker("port")]
    if mc.available("reference"):
        out.append(mc.MatchChecker("reference"))
    return out


@pytest.fixture(scope="module")
def port():
    return cc.CpuChecker("port")


@pytest.fixture(scope="module")
def c2():
    """The node's defaults on a c2-sized map (1 M points, dist_weight (1, 1, 5), map_chunk 20, max_search_radius 0.2)."""
    mp, pose, pts = match_scene(seed=5, n_map=1_000_000, n_scan=20_000, n_off=2000, n_nan=6)
    eng = engine.Engine((0,))
    eng.set_map(mp, engine.LikParams(dist_weight=(1, 1, 5)), None)
    yield eng, mp, pose, pts
    eng.close()


def test_c2_defaults_equal_checkers(c2, port):
    eng, mp, pose, pts = c2
    got_m, got_u = eng.match_output(pose, pts, 0.1, 0.5, 20.0, 0.2)
    for chk in checkers():
        want_m, want_u, cls = expected(chk.create(mp, cc.lik_params(dist_weight=(1, 1, 5)), 20.0, 0.2), port, pose, pts,
                                       0.1, 0.5)
        assert np.bincount(cls, minlength=3).min() > 0
        assert_same_cloud(got_m, want_m)
        assert_same_cloud(got_u, want_u)


@pytest.mark.parametrize("chunk_length,weights,seed", [(1.0, (1, 1, 1), 0), (1.5, (1, 1, 5), 1)])
def test_small_chunks_equal_checkers(port, chunk_length, weights, seed):
    mp, pose, pts = match_scene(seed)
    eng = engine.Engine((0,))
    eng.set_map(mp, engine.LikParams(dist_weight=weights), None)
    got_m, got_u = eng.match_output(pose, pts, 0.1, 0.5, chunk_length, 0.2)
    for chk in checkers():
        want_m, want_u, cls = expected(chk.create(mp, cc.lik_params(dist_weight=weights), chunk_length, 0.2), port, pose,
                                       pts, 0.1, 0.5)
        assert_same_cloud(got_m, want_m)
        assert_same_cloud(got_u, want_u)
    glob = global_classes(mp, transformed(port, pose, pts), weights, 0.1, 0.5)
    assert np.count_nonzero(glob != cls) > 0  # the chunk rule decided some classes
    eng.close()


def test_prepared_cloud_equals_host_cloud(port):
    mp, pose, pts = match_scene(2)
    eng = engine.Engine((0,))
    eng.set_map(mp, engine.LikParams(), engine.beam_params_from_reference())
    finite = pts[np.isfinite(pts["x"]) & np.isfinite(pts["y"]) & np.isfinite(pts["z"])]
    eng.scan_prepare(finite, engine.ScanParams(downsample=(0.05, 0.05, 0.05)))
    ds = eng.scan_get(0)
    assert 0 < len(ds) < len(finite)
    for chunk in (20.0, 1.0):
        a = eng.match_output(pose, None, 0.1, 0.5, chunk, 0.2)
        b = eng.match_output(pose, ds, 0.1, 0.5, chunk, 0.2)
        assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
        assert len(a[0]) and len(a[1])
    eng.close()


def test_errors():
    mp = cc.points([[0.5, 0.5, 0.5], [1.0, 1.0, 1.0]])
    pose = cc.poses([0, 0, 0], [0, 0, 0, 1])
    eng = engine.Engine((0,))
    with pytest.raises(engine.EngineError) as e:
        eng.match_output(pose, mp)
    assert e.value.code == -2  # no map
    eng.set_map(mp, None, engine.beam_params_from_reference())
    with pytest.raises(engine.EngineError) as e:
        eng.match_output(pose, mp)
    assert e.value.code == -1  # no likelihood grid
    eng.set_map(mp, engine.LikParams(), None)
    for kw in (dict(chunk_length=0.0), dict(chunk_length=-1.0), dict(chunk_length=0.4, unmatch_dist=0.5)):
        with pytest.raises(engine.EngineError) as e:
            eng.match_output(pose, mp, **kw)
        assert e.value.code == -1, kw
    with pytest.raises(engine.EngineError) as e:
        eng.match_output(pose, None)  # no prepared scan
    assert e.value.code == -1
    m, u = eng.match_output(pose, mp, chunk_length=0.5, unmatch_dist=0.5)  # radius == chunk length is allowed
    assert len(m) == 2 and len(u) == 0
    L, h = eng.L, eng.h
    import ctypes as C
    n = C.c_size_t(0)
    mpar = engine.MatchParams(0.1, 0.5, 20.0, 0.2)
    assert L.mcl3dl_match_output(None, pose.ctypes.data, mp.ctypes.data, 2, C.byref(mpar), None, C.byref(n), None, C.byref(n)) == -1
    assert L.mcl3dl_match_output(h, None, mp.ctypes.data, 2, C.byref(mpar), None, C.byref(n), None, C.byref(n)) == -1
    assert L.mcl3dl_match_output(h, pose.ctypes.data, mp.ctypes.data, 2, None, None, C.byref(n), None, C.byref(n)) == -1
    assert L.mcl3dl_match_output(h, pose.ctypes.data, mp.ctypes.data, 2, C.byref(mpar), None, None, None, C.byref(n)) == -1
    assert L.mcl3dl_match_output(h, pose.ctypes.data, mp.ctypes.data, 2, C.byref(mpar), None, C.byref(n), None, None) == -1
    # count only
    n_m, n_u = C.c_size_t(9), C.c_size_t(9)
    assert L.mcl3dl_match_output(h, pose.ctypes.data, mp.ctypes.data, 2, C.byref(mpar), None, C.byref(n_m), None,
                                 C.byref(n_u)) == 0
    assert (n_m.value, n_u.value) == (2, 0)
    eng.close()


def test_no_disturbance_of_measure_and_resident_update():
    """measure records and particles_measure_update_prepared results are byte-identical with and without an interleaved
    match_output, and the call is counted in the launch counter."""
    s = synth.scene(50_000, 256, 96, 8, seed=3)
    mp_, pose, pts = match_scene(4)

    def run(interleave):
        eng = engine.Engine((0,))
        eng.set_map(s["map"], engine.LikParams(dist_weight=(1, 1, 5)), engine.beam_params_from_reference())
        rec = [eng.measure(s["particles"], s["lik"], s["beam"], s["origins"])]
        n0 = eng.kernel_launches()
        if interleave:
            eng.match_output(pose, pts, 0.1, 0.5, 20.0, 0.2)
            assert eng.kernel_launches() > n0
        rec.append(eng.measure(s["particles"], s["lik"], s["beam"], s["origins"]))
        n = len(s["particles"])
        states = np.zeros(n, dtype=synth.STATE)
        states["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], 1)
        states["rot"] = np.stack([s["particles"]["qx"], s["particles"]["qy"], s["particles"]["qz"], s["particles"]["qw"]], 1)
        eng.particles_set(states, np.full(n, 1.0 / n, np.float32))
        raw = np.concatenate([s["lik"], s["beam"]])
        eng.scan_prepare(raw, engine.ScanParams(downsample=(0.0, 0.0, 0.0), lik_num_points=64, beam_num_points=4))
        if interleave:
            eng.match_output(pose, pts, 0.1, 0.5, 20.0, 0.2)
            eng.match_output(pose, None, 0.1, 0.5, 20.0, 0.2)
        summ = eng.particles_measure_update_prepared(s["origins"])
        st, prob = eng.particles_get()
        out = [r.tobytes() for r in rec] + [repr(sorted(summ.items())), st.tobytes(), prob.tobytes()]
        eng.close()
        return out

    assert run(False) == run(True)


def test_match_parity_program():
    """The reference's ChunkedKdtree loop vs the C++ adapter's matchOutput, in one process (oracle/_ref)."""
    exe = mc.lib_path("parity")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/match_parity_test not built (no reference checkout at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "MATCH OUTPUT PARITY OK" in r.stdout
