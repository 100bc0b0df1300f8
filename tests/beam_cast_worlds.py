"""Worlds and host builds for the ray markers (mcl3dl_beam_cast): one pose, every ray of a scan, the deciding cast step's
position.

Shared by tests/test_beam_cast_on_host.py (the per-thread device functions compiled for the host, against the CPU
checkers of oracle/beam_cast_api.h) and tests/test_gpu_beam_cast.py (the kernel against the same checkers).  The worlds
are those of tests/beam_edge_worlds.py, plus:

- room_<seed>:  randomized rooms: off-lattice walls and pillars, labels 0..2 under filter_label_max 1 (a filtered pillar
                in front of an unfiltered wall), non-unit quaternions, two sensor origins, ends inside and beyond the walls
- steps:        a particle 7 cm from the x = +1 wall (the first cast step decides) and ends swept up to the wall (the last
                cast step decides: the hit tolerance carries the walk one cell / step beyond the end)

Every pose of a world is cast on its own, as the node casts from its pose estimate.
"""
import ctypes as C
import os
import subprocess

import numpy as np

import beam_edge_worlds as W
from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "beam_cast_hostsim.cpp")
BEAM_RAY = np.dtype([("begin", "<f4", 3), ("end", "<f4", 3), ("pos", "<f4", 3), ("status", "<u4")])
SEEDS = (1, 2, 3, 4)


def room(seed):
    rng = np.random.default_rng(seed)
    n = (int(rng.integers(8, 14)), int(rng.integers(8, 14)), int(rng.integers(5, 8)))
    walls = W._room(*n)
    pil = np.unique(np.array([(i, j, k) for i, j in rng.integers(-5, 6, (3, 2)) for k in range(-n[2] + 1, n[2])]), axis=0)
    pil = pil[~(pil[:, None, :] == walls[None, :, :]).all(axis=2).any(axis=1)]
    ijk = np.vstack([walls, pil]).astype(np.float64)
    xyz = (ijk * W.G + rng.normal(0, 0.01, ijk.shape)).astype(np.float32)
    # walls labelled 0 or 1 (== filter_label_max), pillars 2: filtered, the rays pass them
    lab = np.concatenate([rng.choice(np.array([0, 1], np.uint32), len(walls)), np.full(len(pil), 2, np.uint32)])
    q = rng.normal(0, 1, (4, 4))
    q = q / np.linalg.norm(q, axis=1, keepdims=True) * rng.uniform(0.7, 1.4, (4, 1))
    pos = rng.uniform(-0.5, 0.5, (4, 3)) * np.array([1, 1, 0.5])
    d = rng.normal(0, 1, (96, 3))
    scan = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.3, 2.5, (96, 1))
    origins = ((0.0, 0.0, 0.3), (0.2, -0.1, 0.25))
    return W._world("room_%d" % seed, synth.make_points(xyz, lab), W._poses(pos, q), W._scan(scan, np.arange(96) % 2),
                    origins=origins, filter_label_max=1, dist_weight=(1.0, 1.0, 5.0) if seed % 2 else (1.0, 1.0, 1.0))


def steps():
    d = np.arange(0, 61) * 0.01
    scan = np.vstack([np.stack([0.4 + d, np.zeros_like(d), np.zeros_like(d)], axis=1),
                      [(0.5, 0.0, 0.0), (0.5, 0.02, -0.01), (0.3, 0.1, 0.05)]])
    return W._world("steps", W._pts(W._room()), W._poses([(0.0, 0.0, 0.0), (0.05, 0.05, 0.05), (0.93, 0.01, 0.02)],
                                                         [W.Q_ID] * 3), scan)


def worlds():
    ws = W.worlds() + [room(s) for s in SEEDS] + [steps()]
    for w in ws:
        w["scan"] = W._scan_of(w)
    return ws


def cases():
    """(world name, caster) for every caster a world is valid for."""
    return [(w["name"], c) for w in worlds() for c in w["casters"]]


def world(name):
    return next(w for w in worlds() if w["name"] == name)


def decided_step(rays, w, caster):
    """The index of the cast step that decided each non-LONG ray (1 = the first step) and the ray's last step index,
    restated in float32 from the casters' set-up (raycast_using_dda.h:66-104, raycast_using_kdtree.h:57-64)."""
    b = rays["begin"].astype(np.float32)
    e = rays["end"].astype(np.float32)
    p = rays["pos"].astype(np.float32)
    f = np.float32
    d = e - b
    nrm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    tol = f(w["beam"].get("hit_range", 0.3))
    if caster == "kd":
        g = f(min(w["beam"]["map_grid"]))
        k = np.rint(np.sqrt(((p - b) ** 2).sum(axis=1)) / g)
        last = np.floor((nrm + tol) / g) - 1
        return k, last
    g = np.float64(w["beam"]["dda_grid_size"])
    mp = np.stack([w["map"]["x"], w["map"]["y"], w["map"]["z"]], axis=1)
    mn = mp.min(axis=0)
    idx = lambda v: np.trunc((v - mn).astype(np.float64) / g)  # noqa: E731  (float difference, double division)
    ee = e + (d / nrm[:, None]) * tol
    k = np.abs(np.rint((p.astype(np.float64) - mn) / g - 0.5) - idx(b)).sum(axis=1)
    last = np.abs(idx(ee) - idx(b)).sum(axis=1) - 1
    return k, last


# ------------------------------------------------------------------ the per-thread device functions, compiled for the host
def load_hostsim(out_dir):
    """Compile tests/hostsim/beam_cast_hostsim.cpp into out_dir; returns run(w, pose_index, beam, lik) -> BEAM_RAY[n].
    The NN field is staged as tests/beam_edge_worlds.load_hostsim stages it."""
    so = os.path.join(str(out_dir), "libhostsim_beam_cast.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, HOSTSIM_SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_beam_cast.argtypes = [vp, sz, vp, vp, vp, vp, sz, vp, sz, vp, C.c_int, C.c_int, C.c_int]

    def run(w, i, beam, lik):
        map_pts = np.ascontiguousarray(w["map"], dtype=synth.POINT)
        pose = np.ascontiguousarray(w["poses"][i:i + 1], dtype=synth.POSE)
        scan = np.ascontiguousarray(w["scan"], dtype=synth.POINT)
        origins = np.ascontiguousarray(w["origins"], dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(scan), dtype=BEAM_RAY)
        p = lambda a: a.ctypes.data_as(vp) if a.size else None  # noqa: E731
        rc = L.hostsim_beam_cast(p(map_pts), len(map_pts), C.byref(lik), C.byref(beam), p(pose), p(scan), len(scan),
                                 p(origins), len(origins), p(out), 2, 1, 1)
        assert rc == 0
        return out
    return run
