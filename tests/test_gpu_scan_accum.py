"""Cloud accumulation on the device (include/mcl3dl_b200.h: mcl3dl_scan_accumulate, mcl3dl_scan_prepare_accumulated).
  1. after each accumulate, the accumulation read back equals tests/accum_restate.py's restatement of accumCloud bit for
     bit, label k on cloud k;
  2. prepare_accumulated without downsampling: the raw cloud it hands the pipeline (scan_get(0)) equals the restated
     second transform, dense and not dense, with NaN and infinite points;
  3. with the node's leaves (0.1, 0.1, 0.05) and default clips, every stage scan_get(0..4) is byte-identical to
     mcl3dl_scan_prepare on the cloud the node would have built (restated accumCloud + measure()'s transform): one cloud,
     three with different layouts and frames, ten, and a ~1.3 M-point accumulation;
  4. a resident cycle on the accumulated scans equals the one on scan_prepare(host cloud);
  5. the state rules: clear, prepare does not consume, prepare on nothing, and every INVALID_ARG of accumulate leaves
     the accumulation as it was;
  6. TOO_LARGE at an accumulated total of 2^30 points, reached honestly: one 2 GB buffer of 2^29 four-byte points
     (x, y, z all at offset 0) accumulated up to 2^30 - 1 points (24 GB of device memory at the peak of the growth copy),
     then refused by one point more with the accumulation unchanged;
  7. oracle/_ref/accum_parity_test (oracle/accum.mk, built where the reference checkout exists): the reference's own
     CloudAccumulationLogic driving the node's restated host path and the C++ adapter's accumulateCloud /
     clearAccumulated / prepareAccumulated, prepared stages and cloud counts equal at every process()."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import accum_restate as A
from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu

NODE_LEAF = (0.1, 0.1, 0.05)
F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def E():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


def _cloud(rng, width, height, point_step, offsets, pad, tf, dense=True, specials=0.0, scale=1.5, bound=None):
    xyz = A.random_xyz(rng, width * height, scale=scale, specials=specials)
    if bound is not None:  # keep the special non-finite values, drop the huge finite ones (they would make PCL's
        xyz[np.isfinite(xyz) & (np.abs(xyz) > bound)] = F(0.75)  # lattice overflow and leave the cloud unfiltered)
    data, row_step = A.pack_cloud(xyz, width, height, point_step, offsets, pad, rng=rng)
    return dict(xyz=xyz, data=data, width=width, height=height, point_step=point_step, row_step=row_step,
                offsets=offsets, dense=dense, tf=tf)


def _push(e, c):
    return e.scan_accumulate(c["data"], c["width"], c["height"], c["point_step"], c["row_step"], c["offsets"], c["dense"],
                             *c["tf"])


def _tf(rng, unit=True, t_scale=0.3):
    return (tuple(float(v) for v in rng.standard_normal(3) * t_scale), A.random_quat(rng, unit=unit))


LAYOUTS = [(16, (0, 4, 8)), (32, (16, 0, 8)), (48, (44, 2, 23)), (12, (8, 0, 4))]


def _clouds(seed, k, width, height=1, specials=0.0, dense=True, unit=True, bound=None):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(k):
        ps, off = LAYOUTS[i % len(LAYOUTS)]
        out.append(_cloud(rng, width, height, ps, off, 4 * (i % 3), _tf(rng, unit), dense=dense if i % 2 else True,
                          specials=specials, bound=bound))
    return out, _tf(rng, unit)


def _restated_accum(clouds):
    acc = []
    for k, c in enumerate(clouds):
        R, t = A.xform(*c["tf"])
        acc.append(A.to_points(A.apply(R, t, c["xyz"]), k))
    return np.concatenate(acc)


def test_accumulated_cloud_equals_restatement(E):
    clouds, _ = _clouds(1, 5, 97, 3, specials=0.05, unit=False)
    e = E.Engine((0,))
    for k, c in enumerate(clouds):
        assert _push(e, c) == k + 1
        got = e.scan_accumulated_get()
        want = _restated_accum(clouds[:k + 1])
        assert A.canon(got) == A.canon(want), k
        assert np.array_equal(got["label"], np.repeat(np.arange(k + 1), [len(c["xyz"]) for c in clouds[:k + 1]]))
    e.close()


@pytest.mark.parametrize("dense", [True, False])
def test_second_transform_without_downsampling(E, dense):
    clouds, base = _clouds(2 + dense, 3, 211, 2, specials=0.08, dense=dense, unit=False)
    e = E.Engine((0,))
    for c in clouds:
        _push(e, c)
    acc = e.scan_accumulated_get()
    sp = E.ScanParams(downsample=(0, 0, 0), lik_num_points=0, beam_num_points=0)
    info = e.scan_prepare_accumulated(sp, *base)
    assert info["n_raw"] == info["n_downsampled"] == len(acc)
    R, t = A.xform(*base)
    xyz = np.stack([acc["x"], acc["y"], acc["z"]], axis=1)
    want = A.to_points(A.second(R, t, xyz, dense), acc["label"])
    got = e.scan_get(0)
    assert A.canon(got) == A.canon(want)
    bad = ~np.all(np.isfinite(xyz), axis=1)
    assert bad.any()
    if not dense:  # the not-dense rule passes such a point bit for bit
        assert got[bad].tobytes() == acc[bad].tobytes()
    assert e.scan_accumulated_get().tobytes() == acc.tobytes()  # not consumed
    e.close()


CASES = {"one": (11, 1, 4000), "three": (12, 3, 3000), "ten": (13, 10, 2000), "big": (14, 10, 130_000)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_every_stage_equals_scan_prepare_of_the_node_cloud(E, case):
    seed, k, width = CASES[case]
    clouds, base = _clouds(seed, k, width, specials=0.01 if case == "three" else 0.0, dense=case != "three", bound=50.0)
    e = E.Engine((0,))
    for c in clouds:
        _push(e, c)
    node = A.node_cloud([(c["xyz"], c["dense"], c["tf"]) for c in clouds], base)
    sp = E.ScanParams(downsample=NODE_LEAF, seed=77)
    a = e.scan_prepare_accumulated(sp, *base)
    got = [e.scan_get(w) for w in range(5)]
    b = e.scan_prepare(node, sp)
    want = [e.scan_get(w) for w in range(5)]
    assert a == b and a["n_raw"] == len(node)
    assert a["n_downsampled"] < a["n_raw"] and a["n_lik"] > 0 and a["n_beam"] > 0
    for w in range(5):
        assert got[w].tobytes() == want[w].tobytes(), w
    e.close()


def test_resident_cycle_equals_the_host_cloud_path(E):
    s = synth.scene(60_000, 500, 64, 8, seed=171)
    e = E.Engine((0,))
    e.set_map(s["map"], E.LikParams(dist_weight=(1, 1, 5)), E.beam_params_from_reference(num_points_default=8))
    rng = np.random.default_rng(5)
    # three sensor clouds of the scene's scans with jitter, in frames close to base_link
    base_pts = np.concatenate([s["lik"], s["beam"]])
    clouds = []
    for i in range(3):
        raw = np.tile(base_pts, 15)
        xyz = np.stack([raw[f] + rng.normal(0, 0.03, len(raw)) for f in ("x", "y", "z")], axis=1).astype(np.float32)
        ps, off = LAYOUTS[i]
        data, row_step = A.pack_cloud(xyz, len(xyz), 1, ps, off, 0, rng=rng)
        tf = (tuple(rng.normal(0, 0.05, 3)), tuple(np.r_[rng.normal(0, 0.01, 3), 1.0]))
        clouds.append(dict(xyz=xyz, data=data, width=len(xyz), height=1, point_step=ps, row_step=row_step, offsets=off,
                           dense=True, tf=tf))
    base = ((0.01, -0.02, 0.0), (0.0, 0.0, 0.005, 1.0))
    origins = rng.normal(0, 0.1, (3, 3)).astype(np.float32)
    st = np.zeros(500, dtype=synth.STATE)
    st["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], axis=1)
    st["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], axis=1)
    prior = np.full(500, 1.0 / 500, np.float32)
    sp = E.ScanParams(downsample=NODE_LEAF, lik_num_points=96, beam_num_points=6, seed=9)
    for c in clouds:
        _push(e, c)
    info_a = e.scan_prepare_accumulated(sp, *base)
    e.particles_set(st, prior)
    a = e.particles_measure_update_prepared(origins, 0.0)
    _, post_a = e.particles_get()
    node = A.node_cloud([(c["xyz"], True, c["tf"]) for c in clouds], base)
    info_b = e.scan_prepare(node, sp)
    e.particles_set(st, prior)
    b = e.particles_measure_update_prepared(origins, 0.0)
    _, post_b = e.particles_get()
    assert info_a == info_b and info_a["n_beam"] == 6
    assert a == b and post_a.tobytes() == post_b.tobytes() and a["kept"] == 1
    e.close()


def test_state_rules(E):
    clouds, base = _clouds(21, 3, 300, 2)
    e = E.Engine((0,))
    sp = E.ScanParams(downsample=NODE_LEAF, seed=3)
    # prepare with nothing accumulated: INVALID_ARG, nothing changes
    with pytest.raises(E.EngineError) as ex:
        e.scan_prepare_accumulated(sp, *base)
    assert ex.value.code == -1
    with pytest.raises(E.EngineError):
        e.scan_get(0)  # still no prepared scan
    _push(e, clouds[0])
    _push(e, clouds[1])
    acc = e.scan_accumulated_get()
    info = e.scan_prepare_accumulated(sp, *base)
    stages = [e.scan_get(w).tobytes() for w in range(5)]
    # not consumed: the same call again gives the same scans
    assert e.scan_accumulated_get().tobytes() == acc.tobytes()
    assert e.scan_prepare_accumulated(sp, *base) == info
    assert [e.scan_get(w).tobytes() for w in range(5)] == stages
    # every INVALID_ARG of accumulate leaves the accumulation as it was
    c = clouds[2]
    bad = [dict(width=0), dict(height=0), dict(offsets=(0, 4, c["point_step"] - 3)), dict(row_step=c["width"] * c["point_step"] - 1)]
    for kw in bad:
        v = dict(c, **kw)
        with pytest.raises(E.EngineError) as ex:
            _push(e, v)
        assert ex.value.code == -1, kw
        assert e.scan_accumulated_get().tobytes() == acc.tobytes(), kw
    # the next good cloud still gets the next label
    assert _push(e, c) == 3
    assert e.scan_accumulated_get()["label"][-1] == 2
    # clear empties it; the prepared scans stay; prepare on nothing is INVALID_ARG and they still read back
    e.scan_accumulate_clear()
    assert len(e.scan_accumulated_get()) == 0
    assert [e.scan_get(w).tobytes() for w in range(5)] == stages
    with pytest.raises(E.EngineError) as ex:
        e.scan_prepare_accumulated(sp, *base)
    assert ex.value.code == -1
    assert [e.scan_get(w).tobytes() for w in range(5)] == stages
    # after a clear, labels start again from 0
    assert _push(e, clouds[1]) == 1
    assert set(e.scan_accumulated_get()["label"]) == {0}
    e.close()


def _count(e):
    n = C.c_size_t(0)
    e._check(e.L.mcl3dl_scan_accumulated_get(e.h, None, 0, C.byref(n)))  # the count only: no 16 GB read-back
    return n.value


def test_too_large_at_two_to_the_thirty_points(E):
    half = 1 << 29
    buf = np.zeros(half, np.float32)  # 2 GB: point_step 4, x = y = z = the one float at offset 0
    e = E.Engine((0,))
    assert e.scan_accumulate(buf, half, 1, 4, 4 * half, (0, 0, 0)) == 1
    with pytest.raises(E.EngineError) as ex:  # 2^29 + 2^29 reaches the limit
        e.scan_accumulate(buf, half, 1, 4, 4 * half, (0, 0, 0))
    assert ex.value.code == -5 and _count(e) == half
    assert e.scan_accumulate(buf, half - 1, 1, 4, 4 * (half - 1), (0, 0, 0)) == 2  # 2^30 - 1 points: accepted
    assert _count(e) == 2 * half - 1
    with pytest.raises(E.EngineError) as ex:
        e.scan_accumulate(buf[:1], 1, 1, 4, 4, (0, 0, 0))
    assert ex.value.code == -5 and _count(e) == 2 * half - 1
    e.scan_accumulate_clear()
    assert _count(e) == 0
    e.close()


def test_adapter_parity_program():
    """The cloud accumulation through the C++ adapter against the node's host path under the reference's own
    CloudAccumulationLogic; built by build() where the reference checkout exists."""
    exe = os.path.join(ROOT, "oracle", "_ref", "accum_parity_test")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/accum_parity_test not built (no reference checkout at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "accum parity ok" in r.stdout
