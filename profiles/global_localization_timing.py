#!/usr/bin/env python
"""Time of the node's global localisation (src/mcl_3dl.cpp:1039-1099) and of its shrink step (resizeParticle, pf.h:399-436)
on an H100, against the CPU path on the same machine.

  device:  mcl3dl_global_localization over the staged map (pts=NULL; its own device time build_ms, and the host clock to
           return), and mcl3dl_particles_resize of the seeded set to 0.75 of its size (host clock; the call synchronises);
  CPU:     one host thread: the VoxelGrid of tests/hostsim/scan_hostsim.cpp (the device's restatement; PCL is absent) and
           the reference's own service body and resizeParticle (oracle/_ref/libmcl3dl_gl_ref.so, shim KdTreeFLANN).

    python profiles/global_localization_timing.py [--reps 5] [--maps c2,c4] [--no-cpu]

Maps: bench.py's synthetic warehouse at 1 M points (c2) and 10 M points (c4), grid 0.3, div_yaw 12, dist_weight (1, 1, 5).
Prints one JSON line per map with medians, min and max over --reps, and the GPU's name and power limit.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from mcl_3dl_b200 import engine, synth  # noqa: E402
from oracle import gl_checker as gc  # noqa: E402
from scan_prepare_timing import gpu_info  # noqa: E402

MAPS = {"c2": 1_000_000, "c4": 10_000_000}
W = (1.0, 1.0, 5.0)
GRID, DIV_YAW, IMU = 0.3, 12, (0.0, 0.0, 0.0, 1.0)


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def hostsim_voxel(tmp):
    so = os.path.join(tmp, "libglhs.so")
    src = os.path.join(ROOT, "tests", "hostsim", "gl_hostsim.cpp")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src], check=True)
    L = C.CDLL(so)
    L.hostsim_scan_voxel_grid.restype = C.c_long
    L.hostsim_scan_voxel_grid.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]

    def voxel(pts):
        out = np.zeros(len(pts), synth.POINT)
        leaf = np.full(3, np.float32(GRID), np.float32)
        m = L.hostsim_scan_voxel_grid(pts.ctypes.data_as(C.c_void_p), len(pts), leaf.ctypes.data_as(C.c_void_p),
                                      out.ctypes.data_as(C.c_void_p))
        return pts.copy() if m < 0 else out[:m]
    return voxel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--maps", default="c2,c4")
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    gpu = gpu_info()
    ref = gc.GlChecker("reference") if (not a.no_cpu and gc.available("reference")) else None
    with tempfile.TemporaryDirectory() as tmp:
        voxel = hostsim_voxel(tmp) if ref else None
        for name in a.maps.split(","):
            mp, _ = synth.warehouse_map(MAPS[name], seed=1)
            eng = engine.Engine((0,))
            eng.set_map(mp, engine.LikParams(dist_weight=W))
            seed_dev, seed_wall, resize_wall, info = [], [], [], None
            for _ in range(a.reps):
                t0 = time.perf_counter()
                info = eng.global_localization(None, GRID, DIV_YAW, IMU, W)
                seed_wall.append((time.perf_counter() - t0) * 1e3)
                seed_dev.append(info["build_ms"])
                num = int(info["n_particles"] * 0.75)
                t0 = time.perf_counter()
                eng.particles_resize(num)
                resize_wall.append((time.perf_counter() - t0) * 1e3)
            states, probs = None, None
            rec = {"map": name, "n_map": len(mp), "n_downsampled": info["n_downsampled"], "n_seeds": info["n_seeds"],
                   "n_particles": info["n_particles"], "resize_to": int(info["n_particles"] * 0.75), "gpu": gpu,
                   "device_seed_ms": stats(seed_dev), "device_seed_wall_ms": stats(seed_wall),
                   "device_resize_wall_ms": stats(resize_wall)}
            if ref:
                eng.global_localization(None, GRID, DIV_YAW, IMU, W)
                states, probs = eng.particles_get()
                t0 = time.perf_counter()
                ds = voxel(mp)
                t1 = time.perf_counter()
                cs, cp = ref.gl_seed(ds, GRID, DIV_YAW, IMU, W)
                t2 = time.perf_counter()
                ref.resize(states, probs, int(len(states) * 0.75))
                t3 = time.perf_counter()
                rec.update({"cpu_voxel_ms": (t1 - t0) * 1e3, "cpu_seed_ms": (t2 - t1) * 1e3, "cpu_resize_ms": (t3 - t2) * 1e3,
                            "cpu_equals_device": bool(cs.tobytes() == states.tobytes() and cp.tobytes() == probs.tobytes())})
            print(json.dumps(rec), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
