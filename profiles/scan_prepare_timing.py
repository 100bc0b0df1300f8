#!/usr/bin/env python
"""Wall time of one mcl3dl_scan_prepare on an accumulated ~1.3 M-point cloud at the node's leaves (0.1, 0.1, 0.05) and
the models' default clips: host clock around the call, which ends in a device synchronise (the counts are read back),
so it includes the 21 MB upload of the raw cloud.

    python profiles/scan_prepare_timing.py [--lib A.so [--lib B.so ...]] [--reps 30] [--warmup 5]

With several libraries the calls alternate between them, one engine each, on the same cloud.  Prints one JSON line
per library (median / min / max ms, counts) plus the GPU's name and power limit, and checks that every library
produced the same downsampled cloud.  The cloud's largest voxel holds a few dozen points, so a per-voxel cost that
grows with the voxel's size does not dominate.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mcl_3dl_b200 import engine, synth  # noqa: E402

LEAF = (0.1, 0.1, 0.05)


def accumulated_cloud(n=1_300_000, seed=4):
    """Floor, three walls and clutter within 25 m of the sensor, labels 0..3 (a few accumulated scans)."""
    rng = np.random.default_rng(seed)
    m = n // 8
    parts = [rng.uniform([-25, -25, -0.02], [25, 25, 0.02], (m * 3, 3)),
             rng.uniform([-25, 20, 0], [25, 20.05, 3], (m, 3)), rng.uniform([-25, -20.05, 0], [25, -20, 3], (m, 3)),
             rng.uniform([18, -20, 0], [18.05, 20, 3], (m, 3)), rng.uniform([-20, -18, 0], [16, 18, 2], (n - 6 * m, 3))]
    xyz = np.concatenate(parts)[rng.permutation(n)]
    return synth.make_points(xyz, rng.integers(0, 4, n))


def largest_voxel(raw):
    xyz = np.stack([raw["x"], raw["y"], raw["z"]], 1).astype(np.float32)
    inv = (np.float32(1) / np.asarray(LEAF, np.float32)).astype(np.float32)
    ijk = np.floor(xyz * inv).astype(np.int64)
    ijk -= ijk.min(0)
    span = ijk.max(0) + 1
    key = ijk[:, 0] + ijk[:, 1] * span[0] + ijk[:, 2] * span[0] * span[1]
    return int(np.unique(key, return_counts=True)[1].max())


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the timing itself needs no nvidia-smi
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=None, help="engine library (default: the in-tree build)")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    libs = a.lib or [None]
    raw = accumulated_cloud()
    sp = engine.ScanParams(downsample=LEAF, lik_num_points=96, beam_num_points=3, seed=1)
    engs = [engine.Engine((0,), lib_path=p) for p in libs]
    times = [[] for _ in libs]
    infos = [None] * len(libs)
    for rep in range(a.warmup + a.reps):
        for k, e in enumerate(engs):
            t0 = time.perf_counter()
            infos[k] = e.scan_prepare(raw, sp)
            dt = time.perf_counter() - t0
            if rep >= a.warmup:
                times[k].append(dt * 1e3)
    ds = [e.scan_get(0).tobytes() for e in engs]
    gpu = gpu_info()
    for k, p in enumerate(libs):
        t = np.array(times[k])
        print(json.dumps({"lib": p or "in-tree", "gpu": gpu, "n_raw": len(raw), "largest_voxel": largest_voxel(raw),
                          "info": infos[k], "reps": a.reps, "median_ms": round(float(np.median(t)), 3),
                          "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3),
                          "same_downsampled_cloud_as_first": ds[k] == ds[0]}))
    for e in engs:
        e.close()


if __name__ == "__main__":
    main()
