#!/usr/bin/env python
"""Wall time of one mcl3dl_scan_sample_with_normal (the node's PointCloudSamplerWithNormal on both clipped clouds) after
a mcl3dl_scan_prepare of the ~1.3 M-point accumulated cloud of scan_prepare_timing.py at the node's leaves
(0.1, 0.1, 0.05) and the models' default clips, with the node's sampler defaults (96 / 3 points, r = 0.4, ratios 2 / 5,
max_weight 5): host clock around the call, which ends in a device synchronise.

    python profiles/normal_sampler_timing.py [--reps 30] [--warmup 5]

Prints one JSON line: median / min / max ms, the clipped sizes, the finite normals, rounds and draws, and the GPU's name
and power limit.  No CPU figure is compared: PCL's NormalEstimation is not available here to time.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from mcl_3dl_b200 import engine  # noqa: E402
from scan_prepare_timing import LEAF, accumulated_cloud, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    raw = accumulated_cloud()
    eng = engine.Engine((0,))
    prep = eng.scan_prepare(raw, engine.ScanParams(downsample=LEAF, lik_num_points=96, beam_num_points=3, seed=1))
    cov = np.diag([0.6, 0.05, 0.02, 0.01, 0.01, 0.01])  # an elongated position covariance: ratio sqrt(12), max_weight 2.95
    rot = (0.0, 0.0, 0.38268343, 0.92387953)
    times, info = [], None
    for i in range(a.warmup + a.reps):
        t0 = time.perf_counter()
        info = eng.scan_sample_with_normal(rot, cov, None, 96, 3, seed=i)
        t1 = time.perf_counter()
        if i >= a.warmup:
            times.append((t1 - t0) * 1e3)
    eng.close()
    t = np.array(times)
    print(json.dumps({"call": "scan_sample_with_normal", "median_ms": round(float(np.median(t)), 3),
                      "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3), "reps": a.reps,
                      "n_raw": prep["n_raw"], "n_downsampled": prep["n_downsampled"],
                      "clipped": [prep["n_lik_clipped"], prep["n_beam_clipped"]], "n_normal": info["n_normal"],
                      "rounds": info["rounds"], "draws": info["draws"], "max_weight": info["max_weight"],
                      "gpu": gpu_info()}))


if __name__ == "__main__":
    main()
