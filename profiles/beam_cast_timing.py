#!/usr/bin/env python
"""What the node's rviz ray markers (src/mcl_3dl.cpp:464-628) cost on an H100 with mcl3dl_beam_cast, beside what the node
pays on the CPU for them today:
  (a) the device call from the pose estimate, at 3 rays (the default beam/num_points) and at 256 rays, both casters,
      with a host scan and with the scan mcl3dl_scan_prepare left on the device: host clock around the synchronous call,
      median of --reps after --warmup calls;
  (b) the reference marker loop (getBeamStatus per ray, oracle/_ref/libmcl3dl_beam_cast_ref.so) on one host thread over
      the same rays, median of --reps;
  (c) what a map change costs the node's CPU while it fills its index: ChunkedKdtree::setInputCloud at map_chunk 20 and
      max_search_radius 0.4 (the beam model's search range, 4 x map_grid) — the oracle's stand-in kd-tree
      (oracle/shim/pcl/kdtree/kdtree_flann.h), not FLANN — and, for the DDA caster, its first updatePointCloud (the first
      getBeamStatus after the map changed minus a later one).  Medians of --index-reps.
Maps: bench.py's c2 map (synthetic warehouse, 1 M points) for everything, c4's (10 M points) for (c) as well; likelihood
grid at dist_weight (1, 1, 5), DDA grid 0.2 m.  The records of (a) are checked against (b) byte for byte.  Prints one JSON
line per measurement with the GPU's name and power limit.

    python profiles/beam_cast_timing.py [--reps 30] [--warmup 5] [--index-reps 3] [--maps c2,c4]
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
from oracle import beam_cast_checker as bc  # noqa: E402
from oracle import cpu_checker as cc  # noqa: E402
from scan_prepare_timing import gpu_info  # noqa: E402

MAPS = {"c2": 1_000_000, "c4": 10_000_000}
W = (1.0, 1.0, 5.0)
CASTERS = {"kd": False, "dda": True}


def stats(t):
    t = np.array(t)
    return {"median_ms": round(float(np.median(t)), 4), "min_ms": round(float(t.min()), 4),
            "max_ms": round(float(t.max()), 4), "reps": len(t)}


def timed(fn, reps, warmup=0):
    for _ in range(warmup):
        fn()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--index-reps", type=int, default=3)
    ap.add_argument("--maps", default="c2,c4")
    a = ap.parse_args()
    gpu = gpu_info()
    ref_ok = bc.available("reference")
    for name in a.maps.split(","):
        base, info = synth.warehouse_map(MAPS[name], seed=1001)
        rng = np.random.default_rng(7)
        truth = synth.free_space_position(info, rng)
        quat = synth.quat_from_rpy((0.0, 0.0, 0.4))[0]
        raw = synth.make_scan(base, truth, quat, 20_000, 0.5, 10.0, n_origins=2, seed=5)
        origins = synth.sensor_origins(2)
        # the pose estimate, a little off the truth (a unit quaternion, as the node normalises it)
        pose = synth.make_poses(np.asarray(truth, np.float32).reshape(1, 3) + np.float32(0.02), quat.astype(np.float32).reshape(1, 4))
        # (c) the node's index build per map change, on the oracle's stand-in kd-tree
        if ref_ok:
            ref = bc.BeamCastChecker("reference")
            for caster, dda in CASTERS.items():
                lik, beam = cc.lik_params(dist_weight=W), cc.beam_raw(use_raycast_using_dda=dda, dda_grid_size=0.2)
                t_index, t_first = [], []
                for _ in range(a.index_reps):
                    t0 = time.perf_counter()
                    m = ref.create(base, lik, beam, 20.0, 0.4)
                    t_index.append((time.perf_counter() - t0) * 1e3)
                    if dda:
                        t0 = time.perf_counter()
                        m.beam_cast(pose, raw[:1], origins)
                        first = (time.perf_counter() - t0) * 1e3
                        later = np.median(timed(lambda: m.beam_cast(pose, raw[:1], origins), 5))
                        t_first.append(first - later)
                    m.close()
                out = {"map": name, "n_map": len(base), "caster": caster, "what": "cpu_per_map_change",
                       "setInputCloud_standin_kdtree": stats(t_index)}
                if dda:
                    out["dda_first_updatePointCloud"] = stats(t_first)
                print(json.dumps(out), flush=True)
        if name != "c2":
            continue
        # (a) and (b)
        for caster, dda in CASTERS.items():
            eng = engine.Engine((0,))
            eng.set_map(base, engine.LikParams(dist_weight=W), engine.beam_params_from_reference(
                num_points_default=3, dda_grid_size=0.2, use_raycast_using_dda=dda))
            m = bc.BeamCastChecker("reference").create(base, cc.lik_params(dist_weight=W), cc.beam_raw(
                num_points_default=3, dda_grid_size=0.2, use_raycast_using_dda=dda), 20.0, 0.4) if ref_ok else None
            for n in (3, 256):
                eng.scan_prepare(raw, engine.ScanParams(lik_num_points=0, beam_num_points=n, beam_clip=(0.5, 10.0, -2.0, 2.0)))
                scan = eng.scan_get(4)
                assert len(scan) == n
                got = eng.beam_cast(pose, scan, origins)
                assert got.tobytes() == eng.beam_cast(pose, None, origins).tobytes()
                t_host = timed(lambda: eng.beam_cast(pose, scan, origins), a.reps, a.warmup)
                t_prep = timed(lambda: eng.beam_cast(pose, None, origins), a.reps, a.warmup)
                out = {"map": name, "n_map": len(base), "caster": caster, "rays": n, "gpu": gpu,
                       "device_host_scan": stats(t_host), "device_prepared_scan": stats(t_prep),
                       "statuses": {int(k): int(v) for k, v in zip(*np.unique(got["status"], return_counts=True))}}
                if m is not None:
                    m.beam_cast(pose, scan, origins)  # (the DDA caster's first call builds its grid)
                    want = m.beam_cast(pose, scan, origins)
                    assert got.tobytes() == want.tobytes()
                    out["reference_marker_loop_1_thread"] = stats(timed(lambda: m.beam_cast(pose, scan, origins), a.reps))
                print(json.dumps(out), flush=True)
            if m is not None:
                m.close()
            eng.close()


if __name__ == "__main__":
    main()
