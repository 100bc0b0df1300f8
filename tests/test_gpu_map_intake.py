"""The map intake on an H100 (mcl3dl_map_load / mcl3dl_map_update_* / mcl3dl_map_get): the node's map callbacks
(src/mcl_3dl.cpp:127-153, 1150-1192, 1350-1378) with the map's conversion and VoxelGrid on the device.
  1. map_get equals tests/map_intake_restate.py (conversion + VoxelGrid + intensity centroid) byte for byte on every
     VoxelGrid case of tests/test_gpu_scan_exact.py, unfiltered and all-non-finite ones included.
  2. After map_load every model's records equal those of a fresh engine that ran set_map on the restated cloud.
  3. load / set / commit / set / set / commit / clear / commit equals set_map of the concatenation, and each commit's
     info equals map_append's of the same points.
  4. State and error rules; 5. two devices; 6. the device read over the host tests' layouts (organised, padded,
     unaligned, absent fields); 7. oracle/_ref/map_intake_parity_test where build() made it."""
import os
import subprocess
import ctypes as C

import numpy as np
import pytest

import map_intake_restate as M
from mcl_3dl_b200 import engine, synth
from test_gpu_map_append import box_patch, map_state, params, records, world  # noqa: F401  (world: a fixture)
from test_gpu_scan_exact import VOXEL_CASES, case_ref

pytestmark = pytest.mark.gpu
F = np.float32
XYZIL = dict(point_step=32, offsets=(0, 4, 8), io=16, lo=20)  # PointXYZIL's own layout


def pack(pts, inten, rng=None, **layout):
    lay = dict(XYZIL, **layout)
    w = len(pts)
    data, rs = M.pack_map(pts, inten, w, 1, lay["point_step"], lay["offsets"], lay["io"], lay["lo"], rng=rng)
    return dict(data=data, width=w, height=1, point_step=lay["point_step"], row_step=rs, offsets=lay["offsets"],
                intensity_offset=None if lay["io"] < 0 else lay["io"], label_offset=None if lay["lo"] < 0 else lay["lo"])


def restated(cloud, leaf):
    lay = cloud
    io = -1 if lay["intensity_offset"] is None else lay["intensity_offset"]
    lo = -1 if lay["label_offset"] is None else lay["label_offset"]
    pts, inten = M.convert(lay["data"], lay["width"], lay["height"], lay["point_step"], lay["row_step"], lay["offsets"], io, lo)
    return M.intake_ref(pts, inten, leaf)


def load(e, cloud, leaf, lik=None, beam=None, stamp=None):
    return e.map_load(cloud["data"], cloud["width"], cloud["height"], cloud["point_step"], cloud["row_step"], cloud["offsets"],
                      leaf, lik, beam, cloud["intensity_offset"], cloud["label_offset"], stamp=stamp)


def update_set(e, cloud, leaf):
    return e.map_update_set(cloud["data"], cloud["width"], cloud["height"], cloud["point_step"], cloud["row_step"],
                            cloud["offsets"], leaf, cloud["intensity_offset"], cloud["label_offset"])


def coarse_beam():
    # a coarse DDA grid stages every case, 1.5e9 m extents included, without a large lattice
    return engine.beam_params_from_reference(dda_grid_size=50.0)


@pytest.mark.parametrize("name", VOXEL_CASES)
def test_map_get_equals_restatement(name):
    raw, leaf, _ = case_ref(name)
    rng = np.random.default_rng(len(raw) + 3)
    inten = rng.uniform(0, 255, len(raw)).astype(F)
    cloud = pack(raw, inten)
    want_p, want_i, want_ds = restated(cloud, leaf)
    e = engine.Engine((0,))
    beam = coarse_beam()
    if len(want_p) == 0:  # all_nonfinite: INVALID_ARG, the previous map kept
        prev = synth.make_points(np.array([[1.0, 2.0, 3.0], [4.0, 5.0, 6.0]], F), [1, 2])
        e.set_map(prev, None, beam)
        with pytest.raises(engine.EngineError) as ei:
            load(e, cloud, leaf, None, beam)
        assert ei.value.code == -1
        got_p, got_i = e.map_get()
        assert got_p.tobytes() == prev.tobytes() and got_i.tobytes() == np.zeros(2, F).tobytes()
        e.close()
        return
    info = load(e, cloud, leaf, None, beam)
    assert (info["n_input"], info["n_staged"], info["downsampled"]) == (len(raw), len(want_p), int(want_ds))
    got_p, got_i = e.map_get()
    assert got_p.tobytes() == want_p.tobytes()
    assert got_i.tobytes() == want_i.tobytes()
    fresh = engine.Engine((0,))
    fresh.set_map(want_p, None, beam)
    assert map_state(e)[0] == map_state(fresh)[0]
    e.close()
    fresh.close()


def dense_map(s, copies=3, seed=11):
    """The scene's map as a denser raw cloud: jittered copies with intensities and labels."""
    rng = np.random.default_rng(seed)
    m = s["map"]
    xyz = np.stack([m["x"], m["y"], m["z"]], 1)
    raw = np.concatenate([xyz + rng.normal(0.0, 0.01, xyz.shape) for _ in range(copies)]).astype(F)
    pts = synth.make_points(raw, rng.integers(0, 3, len(raw)))
    return pts, rng.uniform(0, 100, len(raw)).astype(F)


@pytest.mark.parametrize("caster", ["dda", "kd"])
def test_records_after_load_equal_set_map_of_the_restated_cloud(world, caster):  # noqa: F811
    s, _ = world
    lik, beam = params(caster)
    pts, inten = dense_map(s)
    cloud = pack(pts, inten)
    leaf = (0.1, 0.1, 0.1)
    want_p, want_i, _ = restated(cloud, leaf)
    assert len(want_p) < len(pts)  # the VoxelGrid reduces it
    e = engine.Engine((0,))
    load(e, cloud, leaf, lik, beam)
    want = engine.Engine((0,))
    want.set_map(want_p, lik, beam)
    assert e.map_get()[1].tobytes() == want_i.tobytes()
    assert map_state(e) == map_state(want)
    assert records(e, s, 700) == records(want, s, 700)
    n = len(s["particles"])
    states = np.zeros(n, dtype=synth.STATE)
    states["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], 1)
    states["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], 1)
    prob = np.full(n, 1.0 / n, np.float32)
    pose = s["particles"][:1]
    pts_q = np.concatenate([s["lik"], s["beam"]])
    out = []
    for x in (e, want):
        x.particles_set(states, prob)
        summ = x.particles_measure_update(s["lik"], s["beam"], s["origins"])
        res = [repr(sorted(summ.items()))] + [a.tobytes() for a in x.particles_get()]
        res += [a.tobytes() for a in x.match_output(pose, pts_q, 0.1, 0.5, 20.0, 0.2)]
        res.append(x.beam_cast(s["particles"][3], s["beam"], s["origins"]).tobytes())
        gl = x.global_localization(None, grid=0.5)
        gl.pop("build_ms")  # a device time
        res.append(repr(sorted(gl.items())))
        res += [a.tobytes() for a in x.particles_get()]
        out.append(res)
    assert out[0] == out[1]
    e.close()
    want.close()


def patches(s):
    L, H = s["info"]["L"], s["info"]["H"]
    rng = np.random.default_rng(4)
    out = []
    for k, (cx, cy, z0) in enumerate([(0.3 * L, 0.6 * L, 0.5), (0.7 * L, 0.3 * L, 0.5), (0.5 * L, 0.5 * L, 0.4),
                                      (L + 1.0, 0.5 * L, 0.5 * H)]):  # the last one grows the box
        p = box_patch(cx, cy, 1.2, h=0.05, z0=z0, label=k, seed=k)
        out.append(pack(p, rng.uniform(0, 50, len(p)).astype(F), rng=rng))
    return out


def test_update_sequence_equals_set_map_of_the_concatenation(world):  # noqa: F811
    s, _ = world
    lik, beam = params("dda")
    pts, inten = dense_map(s, copies=2)
    base = pack(pts, inten)
    map_leaf, upd_leaf = (0.1, 0.1, 0.1), (0.2, 0.2, 0.2)
    p = patches(s)
    e = engine.Engine((0,))
    load(e, base, map_leaf, lik, beam)
    ref = engine.Engine((0,))  # the same points through set_map / map_append
    staged_p, staged_i, _ = restated(base, map_leaf)
    ref.set_map(staged_p, lik, beam)

    def commit(patch):
        nonlocal staged_p, staged_i
        info = e.map_update_commit()
        if patch is None:
            assert info["n_appended"] == 0 and info["n_after"] == len(staged_p)
            return
        pp, pi, _ = restated(patch, upd_leaf)
        want = ref.map_append(pp)
        for k in ("n_before", "n_appended", "n_after", "incremental", "cells_reselected"):
            assert info[k] == want[k], k
        staged_p, staged_i = np.concatenate([staged_p, pp]), np.concatenate([staged_i, pi])

    update_set(e, p[0], upd_leaf)
    commit(p[0])
    update_set(e, p[1], upd_leaf)
    update_set(e, p[2], upd_leaf)  # replaces p[1]
    commit(p[2])
    update_set(e, p[3], upd_leaf)
    e.map_update_clear()  # cbPosition
    commit(None)
    update_set(e, p[3], upd_leaf)  # grows the box: the full rebuild
    info = e.map_update_commit()
    pp, pi, _ = restated(p[3], upd_leaf)
    assert info["incremental"] == 0 and info["n_appended"] == len(pp)
    staged_p, staged_i = np.concatenate([staged_p, pp]), np.concatenate([staged_i, pi])
    got_p, got_i = e.map_get()
    assert got_p.tobytes() == staged_p.tobytes() and got_i.tobytes() == staged_i.tobytes()
    want = engine.Engine((0,))
    want.set_map(staged_p, lik, beam)
    assert map_state(e) == map_state(want)
    assert records(e, s, 700) == records(want, s, 700)
    # a reload while a patch is pending drops it
    update_set(e, p[0], upd_leaf)
    load(e, base, map_leaf, lik, beam)
    assert e.map_update_commit()["n_appended"] == 0
    assert e.map_get()[0].tobytes() == restated(base, map_leaf)[0].tobytes()
    for x in (e, ref, want):
        x.close()


def test_state_and_error_rules(world):  # noqa: F811
    s, _ = world
    lik, beam = params("dda")
    Lb = engine.load_library()
    pts, inten = dense_map(s, copies=1)
    base = pack(pts, inten)
    leaf = (0.1, 0.1, 0.1)
    p = patches(s)[0]
    e = engine.Engine((0,))
    # before any map: update_set is allowed, commit is NO_MAP and keeps the patch, map_get is NO_MAP
    n_patch = update_set(e, p, leaf)["n_staged"]
    with pytest.raises(engine.EngineError) as ei:
        e.map_update_commit()
    assert ei.value.code == -2
    with pytest.raises(engine.EngineError) as ei:
        e.map_get()
    assert ei.value.code == -2
    e.set_map(s["map"], lik, beam)
    assert e.map_update_commit()["n_appended"] == n_patch  # the patch was kept
    assert e.map_update_commit()["n_appended"] == 0  # and consumed
    # set_map / map_append intensities read as 0, the committed patch's are its VoxelGrid's
    got_i = e.map_get()[1]
    assert not got_i[:len(s["map"])].view(np.uint32).any() and got_i[len(s["map"]):].all()
    e.map_append(s["map"][:100])
    assert not e.map_get()[1][-100:].view(np.uint32).any()
    # invalid views change nothing
    before = [a.tobytes() for a in e.map_get()]
    d = base["data"]
    ptr = d.ctypes.data_as(C.c_void_p)
    lf = np.asarray(leaf, F)
    lfp = lf.ctypes.data_as(C.c_void_p)

    def mc(width=base["width"], height=1, ps=32, rs=base["row_step"], off=(0, 4, 8), io=16, lo=20, data=ptr):
        v = engine.CloudView(data, width, height, ps, rs, (C.c_uint32 * 3)(*off), 1)
        return engine.MapCloud(v, io, lo)

    info = engine.MapIntakeInfo()
    bad = [mc(width=0), mc(rs=31), mc(off=(0, 4, 29)), mc(io=29), mc(lo=-2), mc(lo=32), mc(data=None)]
    for m in bad:
        assert Lb.mcl3dl_map_load(e.h, C.byref(m), lfp, 5, C.byref(lik), C.byref(beam), C.byref(info)) == -1
        assert Lb.mcl3dl_map_update_set(e.h, C.byref(m), lfp, C.byref(info)) == -1
    good = mc()
    assert Lb.mcl3dl_map_load(e.h, C.byref(good), lfp, 5, None, None, C.byref(info)) == -1  # no params
    assert Lb.mcl3dl_map_load(e.h, C.byref(good), None, 5, C.byref(lik), None, C.byref(info)) == -1  # no leaf
    # TOO_LARGE before data is read: 2^30 points of a 4-byte step over a 1 KB array
    big = engine.MapCloud(engine.CloudView(ptr, 1 << 15, 1 << 15, 12, 12 << 15, (C.c_uint32 * 3)(0, 4, 8), 1), -1, -1)
    assert Lb.mcl3dl_map_load(e.h, C.byref(big), lfp, 5, C.byref(lik), C.byref(beam), C.byref(info)) == -5
    assert Lb.mcl3dl_map_update_set(e.h, C.byref(big), lfp, C.byref(info)) == -5
    assert [a.tobytes() for a in e.map_get()] == before
    assert e.map_update_commit()["n_appended"] == 0  # no patch appeared
    # an all-non-finite patch is a valid empty patch: its commit sets the stamp only
    nan = synth.make_points(np.full((10, 3), np.nan, F))
    assert update_set(e, pack(nan, np.zeros(10, F)), leaf)["n_staged"] == 0
    info = e.map_update_commit()
    assert info["n_appended"] == 0 and info["incremental"] == 1
    assert [a.tobytes() for a in e.map_get()] == before
    # the resident set and the prepared scans are untouched by a load and a commit
    n = len(s["particles"])
    states = np.zeros(n, dtype=synth.STATE)
    states["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], 1)
    states["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], 1)
    prob = np.full(n, 1.0 / n, np.float32)
    sp = engine.ScanParams(downsample=(0.0, 0.0, 0.0), lik_num_points=64, beam_num_points=4)
    e.particles_set(states, prob)
    e.scan_prepare(np.concatenate([s["lik"], s["beam"]]), sp)
    resident = [a.tobytes() for a in e.particles_get()]
    scans = [e.scan_get(k).tobytes() for k in range(5)]
    load(e, base, leaf, lik, beam)
    update_set(e, p, leaf)
    e.map_update_commit()
    assert [a.tobytes() for a in e.particles_get()] == resident
    assert [e.scan_get(k).tobytes() for k in range(5)] == scans
    e.close()


def test_two_devices(world):  # noqa: F811
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s, _ = world
    lik, beam = params("dda")
    pts, inten = dense_map(s, copies=2)
    base = pack(pts, inten)
    p = patches(s)[1]
    leaf = (0.1, 0.1, 0.1)
    two, one = engine.Engine((0, 1)), engine.Engine((0,))
    for x in (two, one):
        load(x, base, leaf, lik, beam)
        update_set(x, p, (0.2, 0.2, 0.2))
        x.map_update_commit()
    assert [a.tobytes() for a in two.map_get()] == [a.tobytes() for a in one.map_get()]
    assert records(two, s, 700) == records(one, s, 700)
    two.close()
    one.close()


@pytest.mark.parametrize("layout", [l for l in __import__("test_map_intake_on_host").LAYOUTS],
                         ids=lambda l: "ps%d_io%d_lo%d_h%d" % (l[0], l[2], l[3], l[5]))
def test_device_read_equals_conversion(layout):
    """Unfiltered (leaf 0): map_get equals the restated conversion, finite points in order, on every layout."""
    ps, off, io, lo, pad, h = layout
    rng = np.random.default_rng(ps + 3 * h)
    w = 311
    pts = synth.make_points(rng.uniform(-5, 5, (w * h, 3)).astype(F), rng.integers(0, 2 ** 32, w * h, dtype=np.uint64))
    inten = rng.uniform(0, 100, w * h).astype(F)
    pts["x"][::17] = np.nan
    data, rs = M.pack_map(pts, inten, w, h, ps, off, io, lo, row_pad=pad, rng=rng)
    want_p, want_i, _ = M.intake_ref(*M.convert(data, w, h, ps, rs, off, io, lo), (0.0, 0.0, 0.0))
    e = engine.Engine((0,))
    info = e.map_load(data, w, h, ps, rs, off, (0.0, 0.0, 0.0), None, coarse_beam(), None if io < 0 else io,
                      None if lo < 0 else lo)
    assert info["downsampled"] == 0 and info["n_staged"] == len(want_p)
    got_p, got_i = e.map_get()
    assert got_p.tobytes() == want_p.tobytes() and got_i.tobytes() == want_i.tobytes()
    e.close()


def test_adapter_parity_program():
    """The node's map callbacks on the restated host path and through the C++ adapter's intake methods; built by
    build() where the reference checkout exists."""
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "map_intake_parity_test")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/map_intake_parity_test not built (no reference checkout at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "map intake parity ok" in r.stdout
