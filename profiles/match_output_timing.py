#!/usr/bin/env python
"""Wall time of one mcl3dl_match_output (the node's matched / unmatched output, src/mcl_3dl.cpp:761-805) on an H100,
beside the node's own loop on one host thread (the reference's State6DOF::transform + ChunkedKdtree::radiusSearch,
oracle/_ref/libmcl3dl_match_ref.so, built by build() where a reference checkout exists; skipped without it).

    python profiles/match_output_timing.py [--reps 30] [--warmup 5] [--ref-reps 3]

Host clock around the synchronous call (it ends in a device synchronise), median of --reps calls after --warmup, at the
node's defaults (match 0.1, unmatch 0.5, map_chunk 20, max_search_radius 0.2, dist_weight (1, 1, 5)) on the synthetic
c2 map (1 M points) for:
  scan20k:          a 20 000-point scan around a pose in the map (host cloud);
  accum_host:       the downsampled accumulated cloud of scan_prepare_timing.py (704 503 voxels) as a host cloud;
  accum_prepared:   the same cloud where mcl3dl_scan_prepare left it on the device (pts = NULL).
Prints one JSON line per case with the GPU's name and power limit; the device and reference classes are compared.
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
from mcl_3dl_b200 import engine, synth  # noqa: E402
from scan_prepare_timing import LEAF, accumulated_cloud, gpu_info  # noqa: E402

W = (1.0, 1.0, 5.0)


def c2_scene(seed=0):
    s = synth.scene(1_000_000, 1, 20_000, 0, seed=seed)
    pos = s["truth_pos"]
    q = synth.quat_from_rpy(np.array([s["truth_rpy"]]))[0]
    return s["map"], synth.make_poses(pos, q), s["lik"]


def timed(f, reps, warmup):
    t = []
    for i in range(warmup + reps):
        t0 = time.perf_counter()
        r = f()
        dt = (time.perf_counter() - t0) * 1e3
        if i >= warmup:
            t.append(dt)
    t = np.array(t)
    return r, {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
               "max_ms": round(float(t.max()), 3), "reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-reps", type=int, default=3)
    a = ap.parse_args()
    gpu = gpu_info()
    mp, pose, scan = c2_scene()
    eng = engine.Engine((0,))
    eng.set_map(mp, engine.LikParams(dist_weight=W), None)
    eng.scan_prepare(accumulated_cloud(), engine.ScanParams(downsample=LEAF))
    accum = eng.scan_get(0)
    ref = None
    from oracle import cpu_checker as cc, match_checker as mc
    if mc.available("reference"):
        ref = mc.MatchChecker("reference").create(mp, cc.lik_params(dist_weight=W), 20.0, 0.2)
    cases = [("scan20k", scan), ("accum_host", accum), ("accum_prepared", None)]
    for name, pts in cases:
        before = eng.kernel_launches()
        (m, u), t = timed(lambda: eng.match_output(pose, pts, 0.1, 0.5, 20.0, 0.2), a.reps, a.warmup)
        row = {"case": name, "gpu": gpu, "n": len(scan) if name == "scan20k" else len(accum), "n_matched": len(m),
               "n_unmatched": len(u), "device_call": t,
               "launches_per_call": (eng.kernel_launches() - before) // (a.reps + a.warmup)}
        if ref is not None and name != "accum_prepared":
            cls, tr = timed(lambda: ref.match_output(pose, pts, 0.1, 0.5), a.ref_reps, 0)
            row["reference_one_thread"] = tr
            row["reference_counts"] = [int(np.count_nonzero(cls == 1)), int(np.count_nonzero(cls == 2))]
            row["counts_equal"] = row["reference_counts"] == [len(m), len(u)]
        print(json.dumps(row), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
