"""Small beam-model worlds that drive one rule of the ray casters or of the score to its boundary.

Shared by tests/test_beam_edges_on_host.py (the per-ray device functions compiled for the host, against the reference
build) and tests/test_gpu_beam_edges.py (both beam kernels against the same reference).  Each world is a map, particles,
a beam scan, sensor origins and the beam parameters; `casters` names the casters it is valid for.

- lattice:     map points on multiples of the 0.1 m DDA grid, particles on cell corners, faces, edges and centres, rays
               along all 26 lattice directions with ends on cell faces, on the wall and one hit_tolerance beyond it
               (dda_setup's dix/diy/diz == 0 axes, the strict-'<' axis ladder of dda_advance meeting ties)
- map_box:     ray origins outside the map box and exactly on min_* / max_*; ends far outside the DDA grid
- labels:      map labels equal to filter_label_max and one above it; DDA cells whose first point in map order is
               filtered while a later one is not
- hit_range_*: a hit_range sweep across a wall (ends from 0.5 m before to 0.6 m behind it)
- cone_*:      grazing rays onto a floor at ang_total_ref small, default and >= pi/2
- kd_sin_one:  (KD caster) a vertical metric weight of 5: the second search two steps back finds nothing, sin_angle = 1
- pose:        non-unit quaternions of scale 0.5 ... 2 (ray_origin takes the raw rotation, the end point the normalised
               one) and three sensor origins, the last one used
- score_*:     enough short (or long) rays that beam_likelihood^k falls below beam_likelihood_min and underflows to 0,
               in both short-only modes; N = 0; P = 1

Left out because the reference is undefined there (DESIGN section 7 and section 3(a)): zero-length rays, non-finite end
points, KD rays longer than 65 536 steps, and exactly tied nearest neighbours under the KD caster - so no map has
duplicate points.
"""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np

from mcl_3dl_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOSTSIM_SRC = os.path.join(ROOT, "tests", "hostsim", "hostsim.cpp")

G = 0.1  # DDA grid and map grid of the lattice worlds
DIRS = np.array([d for d in itertools.product((-1, 0, 1), repeat=3) if any(d)], dtype=np.float64)
CASTERS = ("dda", "kd")


def _pts(ijk, label=0):
    """Lattice points: integer coordinates in units of G (computed in double, then rounded to float once)."""
    ijk = np.asarray(ijk, dtype=np.float64).reshape(-1, 3)
    return synth.make_points((ijk * G).astype(np.float32), np.broadcast_to(np.asarray(label, np.uint32), (len(ijk),)))


def _room(nx=10, ny=10, nz=6):
    """The hollow box |i| = nx or |j| = ny or |k| = nz (walls at +-1.0, +-1.0, +-0.6 m), each lattice point once,
    and two pillars inside."""
    ijk = np.array([(i, j, k) for i in range(-nx, nx + 1) for j in range(-ny, ny + 1) for k in range(-nz, nz + 1)
                    if abs(i) == nx or abs(j) == ny or abs(k) == nz])
    pillars = np.array([(3, 3, k) for k in range(-nz + 1, nz)] + [(-4, 2, k) for k in range(-2, 3)])
    return np.vstack([ijk, pillars])


def _poses(pos, quat):
    return synth.make_poses(np.asarray(pos, np.float32).reshape(-1, 3), np.asarray(quat, np.float32).reshape(-1, 4))


def _scan(xyz, label=0):
    return synth.make_points(np.asarray(xyz, np.float32).reshape(-1, 3), np.broadcast_to(np.asarray(label, np.uint32),
                                                                                          (len(np.asarray(xyz).reshape(-1, 3)),)))


def _world(name, map_pts, poses, scan, origins=((0.0, 0.0, 0.0),), casters=CASTERS, dist_weight=(1.0, 1.0, 1.0), **beam):
    beam.setdefault("map_grid", (G, G, G))
    beam.setdefault("dda_grid_size", G)
    beam.setdefault("num_points_default", max(len(scan), 1))
    xyz = np.stack([map_pts["x"], map_pts["y"], map_pts["z"]], axis=1)
    assert len(np.unique(xyz, axis=0)) == len(xyz), name  # no duplicate map points (KD ties are excluded)
    return {"name": name, "map": map_pts, "poses": poses, "scan": scan,
            "origins": np.asarray(origins, np.float32).reshape(-1, 3), "casters": casters,
            "dist_weight": tuple(float(w) for w in dist_weight), "beam": beam}


Q_ID, Q_YAW180, Q_ROLL180 = (0, 0, 0, 1), (0, 0, 1, 0), (1, 0, 0, 0)


def lattice():
    # corners, faces, edges and centres of DDA cells; rotations that map the lattice onto itself exactly
    pos = [(0, 0, 0), (0.05, 0, 0), (0, 0.05, 0), (0, 0, 0.05), (0.05, 0.05, 0), (0.05, 0.05, 0.05), (-0.2, 0.1, -0.3),
           (-0.15, 0.45, 0.25), (0.5, -0.5, 0.1), (0.3, 0.3, 0.35)]
    quat = [Q_ID, Q_ID, Q_ID, Q_ID, Q_YAW180, Q_ID, Q_ROLL180, Q_ID, Q_YAW180, (0, 0, 0, 2)]
    # ends on cell faces, one short of / on / one hit_tolerance (0.3 m) beyond the walls of a particle at the centre
    steps = (3, 7, 9, 10, 13, 14, 25)
    scan = np.vstack([DIRS * k * G for k in steps])
    return _world("lattice", _pts(_room()), _poses(pos, quat), scan)


def map_box():
    # begin outside the box, exactly on min_x / max_x / max_z / the min corner, and just inside
    pos = [(1.05, 0, 0), (-1.0, 0, 0), (1.0, 0.3, 0.1), (0.2, 0.1, 0.6), (-1.0, -1.0, -0.6), (0.99, -0.99, 0.59),
           (0, 0, -0.65), (0.1, 1.2, 0.0)]
    quat = [Q_ID] * len(pos)
    scan = np.vstack([DIRS * 0.5, DIRS * 4.0, DIRS * 50.0])  # inside, beyond the grid, far beyond it
    return _world("map_box", _pts(_room()), _poses(pos, quat), scan)


def labels():
    # DDA grid 0.2: every DDA cell of the x = +1 wall holds 8 lattice points.  In map order the label-2 points (one
    # above filter_label_max) come first, the label-1 points (== filter_label_max) of the same cells after them; the
    # y = +1 wall is filtered entirely, the x = -1 wall carries label 1.
    room = _room()
    lab = np.zeros(len(room), np.uint32)
    xw = room[:, 0] == 10
    lab[xw & ((room[:, 1] + room[:, 2]) % 2 == 0)] = 2
    lab[xw & ((room[:, 1] + room[:, 2]) % 2 != 0)] = 1
    lab[(room[:, 1] == 10) & ~xw] = 2
    lab[(room[:, 0] == -10) & (room[:, 1] != 10)] = 1
    order = np.argsort(-lab.astype(np.int64), kind="stable")  # label 2 first, then 1, then 0
    mp = _pts(room[order], lab[order])
    rng = np.random.default_rng(11)
    pos = np.round(rng.uniform(-5, 5, (8, 3)) * np.array([1, 1, 0.6])) * G
    d = rng.normal(0, 1, (64, 3))
    scan = np.vstack([d / np.linalg.norm(d, axis=1, keepdims=True) * 1.8, DIRS * 1.5])
    return _world("labels", mp, _poses(pos, [Q_ID] * 8), scan, filter_label_max=1, dda_grid_size=0.2)


def hit_range(hr):
    # ends from 0.5 m before the x = +1 wall to 0.6 m behind it, in 1 cm steps, from particles on and off the lattice
    pos = [(0, 0, 0), (0.05, 0.05, 0.0), (0.33, -0.21, 0.17)]
    d = np.arange(-50, 61) * 0.01
    scan = np.vstack([np.stack([1.0 + d - p[0], np.full_like(d, off), np.full_like(d, -off)], axis=1)
                      for p, off in zip(pos, (0.0, 0.003, 0.0))])
    return _world("hit_range_%g" % hr, _pts(_room()), _poses(pos, [Q_ID] * 3), scan, hit_range=hr)


def cone(ang):
    # grazing rays onto the floor (z = -0.6) from 2 to 60 degrees below the horizon, ending 0.25 m below it
    el = np.radians(np.concatenate([np.linspace(2, 20, 19), np.linspace(25, 60, 8)]))
    az = np.radians([0, 33, 90, 200])
    h = 0.6 + 0.25
    scan = np.array([(h / np.tan(e) * np.cos(a), h / np.tan(e) * np.sin(a), -h) for e in el for a in az])
    scan = scan[np.linalg.norm(scan[:, :2], axis=1) < 3.0]
    pos = [(0, 0, 0), (0.05, -0.05, 0.2)]
    return _world("cone_%g" % ang, _pts(_room(15, 15, 6)), _poses(pos, [Q_ID] * 2), scan, ang_total_ref=ang)


def kd_sin_one():
    # oblique rays onto the floor with a metric weight of 5 on z: two marching steps back lies farther above the floor in
    # the searched metric than the second search's radius (0.27), so that search finds nothing and sin_angle stays 1,
    # above sin(ang_total_ref) = 0.9975; with unit weights the same rays are total reflections
    el = np.radians([30, 40, 50, 60])
    az = np.radians([0, 90, 200])
    h = 0.6 + 0.1
    scan = np.array([(h / np.tan(e) * np.cos(a), h / np.tan(e) * np.sin(a), -h) for e in el for a in az])
    pos = [(0, 0, 0), (0.05, 0.05, 0.0), (-0.3, 0.4, 0.0)]
    return _world("kd_sin_one", _pts(_room()), _poses(pos, [Q_ID] * 3), scan, casters=("kd",), dist_weight=(1, 1, 5),
                  ang_total_ref=1.5)


def pose():
    # non-unit quaternions of scale 0.5 ... 2, three origins (labels cycle over all three)
    rng = np.random.default_rng(5)
    P, N = 24, 48
    q = rng.normal(0, 1, (P, 4))
    q = q / np.linalg.norm(q, axis=1, keepdims=True) * rng.uniform(0.5, 2.0, (P, 1))
    q[0] = (0, 0, 0, 2.0)
    q[1] = (0, 0, 0.5, 0.0)
    pos = rng.uniform(-0.4, 0.4, (P, 3))
    d = rng.normal(0, 1, (N, 3))
    scan = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.4, 2.0, (N, 1))
    origins = ((0.1, 0.0, 0.2), (-0.05, 0.1, 0.0), (0.0, -0.2, 0.15))
    return _world("pose", _pts(_room()), _poses(pos, q), _scan(scan, np.arange(N) % 3), origins=origins)


def score(short_only, min_like, n_default):
    # all rays of a particle at the centre pass the walls (SHORT); of one near the x = +1 wall half stop short (LONG)
    rng = np.random.default_rng(7)
    d = rng.normal(0, 1, (90, 3))
    scan = d / np.linalg.norm(d, axis=1, keepdims=True) * np.where(np.arange(90) % 2, 1.9, 0.25)[:, None]
    pos = [(0, 0, 0), (0.7, 0.1, 0.0), (-0.3, -0.3, 0.2)]
    return _world("score_%s_%g_%d" % ("short" if short_only else "all", min_like, n_default), _pts(_room()),
                  _poses(pos, [Q_ID] * 3), scan, add_penalty_short_only_mode=short_only, beam_likelihood_min=min_like,
                  num_points_default=n_default)


def empty_scan():
    return _world("empty_scan", _pts(_room()), _poses([(0, 0, 0), (0.1, 0.2, 0.3), (0.5, 0, 0), (0, 0, 0.05), (1, 1, 1)],
                                                      [Q_ID] * 5), np.zeros((0, 3)))


def one_particle():
    return _world("one_particle", _pts(_room()), _poses([(0.05, 0.05, 0.05)], [(0, 0, 0.3, 0.9)]), DIRS * 1.3)


def _scan_of(w):
    s = w["scan"]
    return s if s.dtype == synth.POINT else _scan(s)


def worlds():
    ws = [lattice(), map_box(), labels(), hit_range(0.3), hit_range(0.08), cone(0.02), cone(np.pi / 6), cone(np.pi / 2),
          cone(2.0), kd_sin_one(), pose(), score(True, 0.2, 20), score(True, 1e-30, 3), score(False, 1e-42, 2),
          score(False, 0.2, 1), empty_scan(), one_particle()]
    for w in ws:
        w["scan"] = _scan_of(w)
    return ws


def cases():
    """(world name, caster) for every caster a world is valid for."""
    return [(w["name"], c) for w in worlds() for c in w["casters"]]


def world(name):
    return next(w for w in worlds() if w["name"] == name)


def beam_kwargs(w, caster):
    return dict(w["beam"], use_raycast_using_dda=caster == "dda")


# ------------------------------------------------------------------ the per-ray device functions, compiled for the host
def load_hostsim(out_dir):
    """Compile tests/hostsim/hostsim.cpp (the product's device functions through a small intrinsic shim) into out_dir and
    return a runner: run(w, caster, beam_params, lik_params, near=(k_lik, k_kd)) -> (records, status, beam work counters
    [cells stepped, cells occupied, points tested]).  The NN field is staged for the likelihood radius and the KD
    caster's marching radius, as the engine stages it with MCL3DL_NNF_KD_R2=0 (by default the engine's field also
    covers the KD caster's second search, which changes that caster's count of points tested, not its records)."""
    so = os.path.join(str(out_dir), "libhostsim_beam.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, HOSTSIM_SRC],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.hostsim_measure_nf.argtypes = [vp, sz, vp, vp, C.c_float, vp, sz, vp, sz, vp, sz, vp, sz, vp, vp, C.c_int, C.c_int, vp,
                                     C.c_int]

    def run(map_pts, poses, scan, origins, beam, lik, near):
        map_pts = np.ascontiguousarray(map_pts, dtype=synth.POINT)
        poses = np.ascontiguousarray(poses, dtype=synth.POSE)
        scan = np.ascontiguousarray(scan, dtype=synth.POINT)
        origins = np.ascontiguousarray(origins, dtype=np.float32).reshape(-1, 3)
        out = np.zeros(len(poses), dtype=synth.RESULT)
        st = np.zeros((len(poses), max(len(scan), 1)), dtype=np.uint8)
        wk = np.zeros(9, dtype=np.uint64)
        p = lambda a: a.ctypes.data_as(vp) if a.size else None  # noqa: E731
        rc = L.hostsim_measure_nf(p(map_pts), len(map_pts), C.byref(lik), C.byref(beam), 1.0, p(poses), len(poses), None, 0,
                                  p(scan), len(scan), p(origins), len(origins), p(out), p(st), int(near[0]), int(near[1]),
                                  p(wk), 1)
        assert rc == 0
        return out, st[:, :len(scan)], tuple(int(v) for v in wk[2:5])
    return run
