#!/usr/bin/env python
"""Wall time of the node's map update (cbMapUpdateTimer, src/mcl_3dl.cpp:1350-1378: map += VoxelGrid(patch)) on an H100,
two ways, alternating in one session:
  (a) restage: what the adapter paid before mcl3dl_map_append - the merged cloud packed on the host (here: the
      concatenation of the packed arrays) and mcl3dl_set_map of all of it;
  (b) append:  mcl3dl_map_append of the patch alone.
Host clock to return (both calls end in a device synchronise); (b) also reports its own device time (build_ms) and the
NN-field directory cells it re-selected, (a) the device build time set_map reports (map_info().build_ms).

    python profiles/map_append_timing.py [--reps 5] [--maps c2,c4]

Maps: bench.py's c2 map (synthetic warehouse, 1 M points) and its largest, c4's (10 M points), likelihood grid at
dist_weight (1, 1, 5) and the DDA beam grid (0.2 m), as bench stages them.  Patches: new box obstacles at 0.3 m
(update_downsample) inside the map's box, about 1 k, 10 k and 100 k points, and a 10 k patch with one box outside it
(grows the box).  Before every timed call the engine holds the base map (set_map, not timed).  Prints one JSON line per
(map, patch) with medians, min and max over --reps, and the GPU's name and power limit.
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
from scan_prepare_timing import gpu_info  # noqa: E402

MAPS = {"c2": 1_000_000, "c4": 10_000_000}
W = (1.0, 1.0, 5.0)


def boxes(info, n_target, seed, outside=False, h=0.3, size=1.5):
    """Box obstacles (four walls and a lid at h spacing) at random places on the floor, cut to n_target points."""
    rng = np.random.default_rng(seed)
    L, H = info["L"], info["H"]
    u = np.arange(0.0, size + 1e-6, h, dtype=np.float64)
    a, b = [g.ravel() for g in np.meshgrid(u, u, indexing="ij")]
    z = np.zeros_like(a)
    one = np.concatenate([np.stack([a, z, b], 1), np.stack([a, z + size, b], 1), np.stack([z, a, b], 1),
                          np.stack([z + size, a, b], 1), np.stack([a, b, z + size], 1)])
    parts, n = [], 0
    while n < n_target:
        x0, y0 = rng.uniform(0.1 * L, 0.9 * L - size, 2)
        z0 = rng.uniform(0.05, H - size - 0.05)
        if outside and not parts:
            x0 = L + 1.0  # one box beyond the map's +x wall
        p = one + (x0, y0, z0) + rng.normal(0.0, 0.01, one.shape)
        parts.append(p)
        n += len(p)
    xyz = np.concatenate(parts)[:n_target].astype(np.float32)
    return synth.make_points(xyz)


def stats(t):
    t = np.array(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3),
            "max_ms": round(float(t.max()), 3), "reps": len(t)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--maps", default="c2,c4")
    a = ap.parse_args()
    gpu = gpu_info()
    lik = engine.LikParams(dist_weight=W)
    beam = engine.beam_params_from_reference(num_points_default=8, dda_grid_size=0.2)
    for name in a.maps.split(","):
        base, info = synth.warehouse_map(MAPS[name], seed=1001)
        patches = [("1k", boxes(info, 1_000, 1)), ("10k", boxes(info, 10_000, 2)), ("100k", boxes(info, 100_000, 3)),
                   ("10k_grows_box", boxes(info, 10_000, 4, outside=True))]
        eng = engine.Engine((0,))
        eng.set_map(base, lik, beam)  # warm-up: module load, first allocations
        for pname, patch in patches:
            ta, tb, dev_a, dev_b, cells, incr = [], [], [], [], [], []
            for _ in range(a.reps):
                eng.set_map(base, lik, beam)
                t0 = time.perf_counter()
                merged = np.concatenate([base, patch])
                eng.set_map(merged, lik, beam)
                ta.append((time.perf_counter() - t0) * 1e3)
                dev_a.append(eng.map_info().build_ms)
                want = eng.measure(synth.tracking_particles(64, (info["L"] / 2, info["L"] / 2, 0.6), (0, 0, 0)),
                                   base[:256])
                eng.set_map(base, lik, beam)
                t0 = time.perf_counter()
                r = eng.map_append(patch)
                tb.append((time.perf_counter() - t0) * 1e3)
                dev_b.append(r["build_ms"])
                cells.append(r["cells_reselected"])
                incr.append(r["incremental"])
                got = eng.measure(synth.tracking_particles(64, (info["L"] / 2, info["L"] / 2, 0.6), (0, 0, 0)),
                                  base[:256])
                assert got.tobytes() == want.tobytes()
            print(json.dumps({"map": name, "n_map": len(base), "patch": pname, "n_patch": len(patch), "gpu": gpu,
                              "restage_host": stats(ta), "restage_build_ms": stats(dev_a),
                              "append_host": stats(tb), "append_build_ms": stats(dev_b),
                              "cells_reselected": int(np.median(cells)), "incremental": sorted(set(incr))}), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
