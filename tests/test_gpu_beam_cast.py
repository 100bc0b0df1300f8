"""The ray markers on the device (mcl3dl_beam_cast, beam_cast_kernel) against the host build of the same device functions and
the CPU checkers of oracle/beam_cast_api.h, byte for byte; its statuses against mcl3dl_beam_status; the prepared-scan
path, map appends, a multi-device engine and the error codes; and the parity program of the C++ adapter
(oracle/_ref/beam_cast_parity_test)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import beam_cast_worlds as B
import beam_edge_worlds as W
from mcl_3dl_b200 import engine, synth
from oracle import beam_cast_checker as bc
from oracle import cpu_checker as cc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    if not bc.available("reference"):
        pytest.skip("oracle/_ref/libmcl3dl_beam_cast_ref.so not built (needs a checkout of the reference at build time)")
    return bc.BeamCastChecker("reference")


@pytest.fixture(scope="module")
def port():
    return bc.BeamCastChecker("port")


@pytest.fixture(scope="module")
def hs(tmp_path_factory):
    return B.load_hostsim(tmp_path_factory.mktemp("beam_cast_gpu"))


def staged(w, caster, devices=(0,)):
    eng = engine.Engine(devices)
    eng.set_map(w["map"], engine.LikParams(dist_weight=w["dist_weight"]),
                engine.beam_params_from_reference(**W.beam_kwargs(w, caster)))
    return eng


def test_record_layout_matches_header():
    assert engine.BEAM_RAY.itemsize == 40 and bc.BEAM_RAY == engine.BEAM_RAY
    assert [engine.BEAM_RAY.fields[k][1] for k in ("begin", "end", "pos", "status")] == [0, 12, 24, 36]


@pytest.mark.parametrize("name,caster", B.cases())
def test_kernel_equals_host_build_and_reference(ref, hs, name, caster):
    w = B.world(name)
    eng = staged(w, caster)
    m = ref.create(w["map"], cc.lik_params(dist_weight=w["dist_weight"]), cc.beam_raw(**W.beam_kwargs(w, caster)))
    beam = engine.beam_params_from_reference(**W.beam_kwargs(w, caster))
    lik = engine.LikParams(dist_weight=w["dist_weight"])
    for i in range(len(w["poses"])):
        got = eng.beam_cast(w["poses"][i], w["scan"], w["origins"])
        want = m.beam_cast(w["poses"][i], w["scan"], w["origins"])
        assert got.tobytes() == want.tobytes(), "pose %d" % i
        assert got.tobytes() == hs(w, i, beam, lik).tobytes(), "pose %d" % i
        # the statuses are mcl3dl_beam_status's for the same pose and rays
        if len(w["scan"]):
            st = eng.beam_status(w["poses"][i:i + 1], w["scan"], w["origins"])[0]
            assert np.array_equal(st, got["status"].astype(np.uint8))
    m.close()
    eng.close()


def _room_scan(n, seed):
    rng = np.random.default_rng(seed)
    d = rng.normal(0, 1, (n, 3))
    xyz = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.2, 3.0, (n, 1))
    return synth.make_points(xyz.astype(np.float32), (np.arange(n) % 2).astype(np.uint32))


@pytest.mark.parametrize("caster", W.CASTERS)
@pytest.mark.parametrize("n", [1, 255, 257, 1000, 5000])
def test_launch_shapes(ref, caster, n):
    w = B.world("room_%d" % (1 if caster == "kd" else 2))
    eng = staged(w, caster)
    m = ref.create(w["map"], cc.lik_params(dist_weight=w["dist_weight"]), cc.beam_raw(**W.beam_kwargs(w, caster)))
    scan = _room_scan(n, n)
    got = eng.beam_cast(w["poses"][1], scan, w["origins"])
    assert len(got) == n
    assert got.tobytes() == m.beam_cast(w["poses"][1], scan, w["origins"]).tobytes()
    m.close()
    eng.close()


@pytest.mark.parametrize("caster", W.CASTERS)
def test_prepared_scan_equals_host_scan(caster):
    w = B.world("room_3")
    eng = staged(w, caster)
    raw = _room_scan(4000, 9)
    eng.scan_prepare(raw, engine.ScanParams(downsample=(0.05, 0.05, 0.05), beam_clip=(0.3, 10.0, -5.0, 5.0), lik_num_points=8,
                                            beam_num_points=300, seed=3))
    for k in range(2):
        if k:  # the normal-weighted sampler's scans replace the prepared ones
            eng.scan_sample_with_normal((0, 0, 0, 1), np.diag([0.1, 0.1, 0.01]), lik_num_points=8, beam_num_points=200,
                                        seed=4)
        scan = eng.scan_get(4)
        assert len(scan) > 50
        for i in range(len(w["poses"])):
            a = eng.beam_cast(w["poses"][i], None, w["origins"])
            b = eng.beam_cast(w["poses"][i], scan, w["origins"])
            assert a.tobytes() == b.tobytes()
    eng.close()


@pytest.mark.parametrize("caster", W.CASTERS)
def test_after_map_append_equals_fresh_engine(caster):
    w = B.world("room_4")
    eng = staged(w, caster)
    xyz = np.stack([w["map"]["x"], w["map"]["y"], w["map"]["z"]], axis=1)
    lo, hi = xyz.min(axis=0), xyz.max(axis=0)
    rng = np.random.default_rng(44)
    inner = synth.make_points((lo + rng.uniform(0.2, 0.8, (300, 3)) * (hi - lo)).astype(np.float32))
    outer = synth.make_points((hi + rng.uniform(0.0, 0.5, (100, 3))).astype(np.float32))
    cur = w["map"]
    for patch, incremental in ((inner, 1), (outer, 0)):
        assert eng.map_append(patch)["incremental"] == incremental
        cur = np.concatenate([cur, patch])
        fresh = staged(dict(w, map=cur), caster)
        for i in range(len(w["poses"])):
            assert eng.beam_cast(w["poses"][i], w["scan"], w["origins"]).tobytes() == \
                fresh.beam_cast(w["poses"][i], w["scan"], w["origins"]).tobytes()
        fresh.close()
    eng.close()


@pytest.mark.parametrize("caster", W.CASTERS)
def test_multi_device_engine_host_scans(caster):
    """Engine((0, 0)) is two device contexts on one H100: host scans run on device 0 and equal a one-device engine's."""
    w = B.world("room_1")
    one, two = staged(w, caster), staged(w, caster, (0, 0))
    for i in range(len(w["poses"])):
        assert two.beam_cast(w["poses"][i], w["scan"], w["origins"]).tobytes() == \
            one.beam_cast(w["poses"][i], w["scan"], w["origins"]).tobytes()
    with pytest.raises(engine.EngineError) as e:
        two.beam_cast(w["poses"][0], None, w["origins"])  # the prepared form is single-device only
    assert e.value.code == -1
    one.close()
    two.close()


def _raw_cast(eng, pose, pts, origins, out, capacity):
    n = C.c_size_t(12345)
    rc = eng.L.mcl3dl_beam_cast(eng.h, engine._ptr(pose) if pose is not None else None,
                                pts.ctypes.data if pts is not None else None, len(pts) if pts is not None else 0,
                                engine._ptr(origins), len(origins), engine._ptr(out) if out is not None else None, capacity,
                                C.byref(n))
    return rc, n.value


def test_errors():
    w = B.world("steps")
    pose = w["poses"][:1]
    scan = w["scan"][:10].copy()
    origins = w["origins"]
    out = np.zeros(10, engine.BEAM_RAY)
    eng = engine.Engine((0,))
    assert _raw_cast(eng, pose, scan, origins, out, 10)[0] == -2  # before set_map
    assert eng.L.mcl3dl_beam_cast(None, engine._ptr(pose), engine._ptr(scan), 10, engine._ptr(origins), 1,
                                  engine._ptr(out), 10, C.byref(C.c_size_t(0))) == -1
    eng.set_map(w["map"], engine.LikParams(), None)
    assert _raw_cast(eng, pose, scan, origins, out, 10)[0] == -1  # no beam params
    eng.set_map(w["map"], None, engine.beam_params_from_reference(use_raycast_using_dda=True))
    assert _raw_cast(eng, pose, scan, origins, out, 10) == (0, 10)  # DDA needs no likelihood grid
    eng.set_map(w["map"], engine.LikParams(), engine.beam_params_from_reference(use_raycast_using_dda=False))
    assert _raw_cast(eng, None, scan, origins, out, 10)[0] == -1  # no pose
    assert eng.L.mcl3dl_beam_cast(eng.h, engine._ptr(pose), engine._ptr(scan), 10, engine._ptr(origins), 1,
                                  engine._ptr(out), 10, None) == -1  # no n_out
    assert _raw_cast(eng, pose, scan, origins, None, 10)[0] == -1  # no out with rays to write
    assert _raw_cast(eng, pose, scan, origins, out, 9)[0] == -1  # capacity below the ray count
    before = out.tobytes()
    bad = scan.copy()
    bad["label"][7] = len(origins)
    assert _raw_cast(eng, pose, bad, origins, out, 10) == (-1, 12345)  # a label beyond the origins: nothing written
    assert out.tobytes() == before
    assert _raw_cast(eng, pose, None, origins, out, 10)[0] == -1  # no prepared scan
    assert _raw_cast(eng, pose, scan[:0], origins, None, 0) == (0, 0)  # an empty scan
    got = eng.beam_cast(pose, scan, origins)
    assert len(got) == 10
    eng.close()


def test_beam_cast_parity_program():
    """The node's marker loop on the reference beam model vs castBeams, and a node without its CPU map index vs one with
    it (oracle/_ref/beam_cast_parity_test)."""
    exe = bc.lib_path("parity")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/beam_cast_parity_test not built (no reference checkout at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=1200)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "BEAM CAST PARITY OK" in r.stdout
