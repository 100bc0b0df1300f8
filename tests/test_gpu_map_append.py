"""mcl3dl_map_append on an H100: the node's map update (cbMapUpdateTimer, src/mcl_3dl.cpp:1350-1378) appends a
downsampled patch to the staged cloud.  After set_map(A) and any number of appends, every call gives records
byte-identical to a fresh engine that ran set_map on the concatenation, and nothing but the map changes."""
import ctypes as C

import numpy as np
import pytest

from mcl_3dl_b200 import engine, synth

pytestmark = pytest.mark.gpu


def box_patch(cx, cy, size, h=0.3, z0=0.0, label=0, seed=0):
    """The faces of an axis-aligned box obstacle at h spacing (a VoxelGrid-ed patch at update_downsample)."""
    rng = np.random.default_rng(seed)
    u = np.arange(0.0, size + 1e-6, h)
    a, b = np.meshgrid(u, u, indexing="ij")
    a, b = a.ravel(), b.ravel()
    x0, y0 = cx - size / 2, cy - size / 2
    faces = [np.stack([x0 + a, y0 + 0 * a, z0 + b], 1), np.stack([x0 + a, y0 + size + 0 * a, z0 + b], 1),
             np.stack([x0 + 0 * a, y0 + a, z0 + b], 1), np.stack([x0 + size + 0 * a, y0 + a, z0 + b], 1),
             np.stack([x0 + a, y0 + b, z0 + size + 0 * a], 1)]
    xyz = np.concatenate(faces) + rng.normal(0.0, 0.01, (5 * len(a), 3))
    return synth.make_points(xyz.astype(np.float32), np.full(len(xyz), label, np.uint32))


def duplicate_cluster(x, y, z, n=64):
    """n copies of one point: more candidates than a voxel's list holds, so the NN field has overflow cells."""
    return synth.make_points(np.tile(np.array([[x, y, z]], np.float32), (n, 1)))


@pytest.fixture(scope="module")
def world():
    s = synth.scene(100_000, 700, 96, 8, seed=23)
    L = s["info"]["L"]
    inside = [box_patch(0.3 * L, 0.6 * L, 1.5, z0=0.5, seed=1), duplicate_cluster(0.45 * L, 0.45 * L, 1.0),
              box_patch(0.7 * L, 0.3 * L, 0.9, h=0.1, z0=0.5, seed=2)]
    return s, inside


def params(caster, filter_label_max=0xFFFFFFFF):
    lik = engine.LikParams(dist_weight=(1, 1, 5))
    beam = engine.beam_params_from_reference(num_points_default=8, dda_grid_size=0.2, filter_label_max=filter_label_max,
                                             use_raycast_using_dda=caster == "dda")
    return lik, beam


def records(e, s, n_particles):
    p = s["particles"][:n_particles]
    out = [e.measure(p, s["lik"], s["beam"], s["origins"]).tobytes(),
           e.measure(p, s["lik"], None, None).tobytes(),
           e.beam_status(p, s["beam"], s["origins"]).tobytes()]
    prior = np.linspace(0.5, 1.5, len(p), dtype=np.float32)
    post, summ, rec = e.measure_update(p, s["lik"], s["beam"], s["origins"], prior, want_records=True)
    return out + [post.tobytes(), repr(sorted(summ.items())), rec.tobytes()]


def map_state(e):
    """Lattices and the NN field's live counts.  (Its bytes are the allocation: after appends they include dead lists.)"""
    mi = e.map_info()
    f = e.nn_field_info()
    return ([mi.n_points, tuple(mi.nn_dims), mi.nn_cell, tuple(mi.nn_origin), tuple(mi.dda_dims), tuple(mi.dda_min),
             tuple(mi.dda_max)], {k: f[k] for k in ("candidates", "overflow_cells", "wide_cells", "voxel_edge")})


def directory_cells(e):
    """Directory cells of a freshly built NN field: its bytes are 8 per cell + 16 per candidate + 16 per wide-table entry
    (min(cells, 2^18) of them)."""
    f = e.nn_field_info()
    rest = f["bytes"] - 16 * f["candidates"]
    return (rest // 3 if rest <= 3 << 21 else rest - (1 << 22)) // 8


def fresh(points, lik, beam):
    e = engine.Engine((0,))
    e.set_map(points, lik, beam)
    return e


@pytest.mark.parametrize("caster", ["dda", "kd"])
@pytest.mark.parametrize("n_particles", [100, 700])  # below / above 256: lik_kernel_nf and lik_kernel_nf_pm
def test_consecutive_appends_equal_fresh_set_map(world, caster, n_particles):
    s, patches = world
    lik, beam = params(caster)
    e = engine.Engine((0,))
    e.set_map(s["map"], lik, beam)
    n_cells = directory_cells(e)
    staged = s["map"]
    for k, p in enumerate(patches):
        info = e.map_append(p)
        assert (info["n_before"], info["n_appended"], info["n_after"]) == (len(staged), len(p), len(staged) + len(p))
        # inside the box: the incremental path, re-selecting a small part of the directory
        assert info["incremental"] == 1 and 0 < info["cells_reselected"] < n_cells // 20 and info["build_ms"] > 0
        staged = np.concatenate([staged, p])
        if k == 1:  # an empty update in between changes the stamp only
            assert e.map_append(staged[:0]) == {"n_before": len(staged), "n_appended": 0, "n_after": len(staged),
                                                "incremental": 1, "cells_reselected": 0, "build_ms": 0.0}
        want = fresh(staged, lik, beam)
        assert map_state(e) == map_state(want)
        assert records(e, s, n_particles) == records(want, s, n_particles)
        want.close()
    assert e.nn_field_info()["overflow_cells"] > 0  # the duplicate cluster
    e.close()


def test_box_growing_append(world):
    """A patch outside the staged map's bounding box moves every lattice: the full device rebuild."""
    s, _ = world
    lik, beam = params("dda")
    L, H = s["info"]["L"], s["info"]["H"]
    grow = box_patch(L + 1.0, 0.5 * L, 1.2, z0=0.5 * H, seed=4)
    e = engine.Engine((0,))
    e.set_map(s["map"], lik, beam)
    info = e.map_append(grow)
    assert info["incremental"] == 0
    both = np.concatenate([s["map"], grow])
    want = fresh(both, lik, beam)
    assert map_state(e) == map_state(want)
    assert e.map_info().dda_max[0] > s["map"]["x"].max()
    assert records(e, s, 300) == records(want, s, 300)
    e.close()
    want.close()


@pytest.mark.parametrize("caster", ["dda", "kd"])
def test_patch_labels_above_filter_label_max(world, caster):
    s, _ = world
    lik, beam = params(caster, filter_label_max=1)
    L = s["info"]["L"]
    p = box_patch(0.55 * L, 0.35 * L, 1.2, label=3, seed=5)
    e = engine.Engine((0,))
    e.set_map(s["map"], lik, beam)
    e.map_append(p)
    want = fresh(np.concatenate([s["map"], p]), lik, beam)
    assert records(e, s, 300) == records(want, s, 300)
    e.close()
    want.close()


def test_match_output_after_append(world):
    s, patches = world
    lik = engine.LikParams(dist_weight=(1, 1, 5))
    e = engine.Engine((0,))
    e.set_map(s["map"], lik, None)
    for p in patches:
        e.map_append(p)
    want = fresh(np.concatenate([s["map"]] + patches), lik, None)
    pose = s["particles"][:1]
    pts = np.concatenate([s["lik"], s["beam"]])
    for a, b in zip(e.match_output(pose, pts, 0.1, 0.5, 20.0, 0.2), want.match_output(pose, pts, 0.1, 0.5, 20.0, 0.2)):
        assert a.tobytes() == b.tobytes()
    e.close()
    want.close()


def test_resident_particles_and_prepared_scans_untouched(world):
    s, patches = world
    lik, beam = params("dda")
    n = len(s["particles"])
    states = np.zeros(n, dtype=synth.STATE)
    states["pos"] = np.stack([s["particles"]["px"], s["particles"]["py"], s["particles"]["pz"]], 1)
    states["rot"] = np.stack([s["particles"][k] for k in ("qx", "qy", "qz", "qw")], 1)
    prob = np.full(n, 1.0 / n, np.float32)
    raw = np.concatenate([s["lik"], s["beam"]])
    sp = engine.ScanParams(downsample=(0.0, 0.0, 0.0), lik_num_points=64, beam_num_points=4)

    def prepared(e):
        return repr(sorted(e.particles_measure_update_prepared(s["origins"]).items())), [a.tobytes() for a in e.particles_get()]

    e = engine.Engine((0,))
    e.set_map(s["map"], lik, beam)
    e.particles_set(states, prob)
    e.scan_prepare(raw, sp)
    before = [a.tobytes() for a in e.particles_get()]
    e.map_append(patches[0])
    assert [a.tobytes() for a in e.particles_get()] == before
    want = fresh(np.concatenate([s["map"], patches[0]]), lik, beam)
    want.particles_set(states, prob)
    want.scan_prepare(raw, sp)
    assert prepared(e) == prepared(want)
    e.close()
    want.close()


def test_field_mode_volume_restaged(world):
    s, patches = world
    lik = engine.LikParams(dist_weight=(1, 1, 5))
    e = engine.Engine((0,))
    e.set_map(s["map"], lik, None)
    e.field_mode(True)
    e.map_append(patches[0])
    want = fresh(np.concatenate([s["map"], patches[0]]), lik, None)
    want.field_mode(True)
    assert e.measure(s["particles"], s["lik"]).tobytes() == want.measure(s["particles"], s["lik"]).tobytes()
    assert e.field_nodes()[0].tobytes() == want.field_nodes()[0].tobytes()
    e.close()
    want.close()


def test_error_codes(world):
    s, patches = world
    L = engine.load_library()
    e = engine.Engine((0,))
    info = engine.MapAppendInfo()
    p = patches[0]
    ptr = p.ctypes.data_as(C.c_void_p)
    assert L.mcl3dl_map_append(None, ptr, len(p), 1, C.byref(info)) == -1
    assert L.mcl3dl_map_append(e.h, ptr, len(p), 1, C.byref(info)) == -2  # before set_map
    e.set_map(s["map"], engine.LikParams(), None)
    assert L.mcl3dl_map_append(e.h, None, 5, 1, C.byref(info)) == -1
    # the sizes are checked before pts is read: a count far beyond the array is refused, not read
    assert L.mcl3dl_map_append(e.h, ptr, (1 << 31) - len(s["map"]), 1, C.byref(info)) == -5
    assert L.mcl3dl_map_append(e.h, ptr, 1 << 40, 1, C.byref(info)) == -5
    # the map is still staged and unchanged
    assert e.map_info().n_points == len(s["map"])
    assert L.mcl3dl_map_append(e.h, ptr, len(p), 7, None) == 0
    assert e.map_info().n_points == len(s["map"]) + len(p)
    e.close()


def test_two_devices(world):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    s, patches = world
    lik, beam = params("dda")
    e = engine.Engine((0, 1))
    e.set_map(s["map"], lik, beam)
    for p in patches:
        e.map_append(p)
    want = fresh(np.concatenate([s["map"]] + patches), lik, beam)
    assert records(e, s, 700) == records(want, s, 700)
    e.close()
    want.close()
