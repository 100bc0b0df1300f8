#!/usr/bin/env python
"""Time of the resident set's landmark update and of reading the published particle poses on an H100, against what a
node does without them.

  landmark: mcl3dl_particles_landmark_update (it synchronises) against a host round trip: mcl3dl_particles_get, the
            reference's own code on one host thread through the checker library oracle/_ref/libmcl3dl_pf_landmark_ref.so
            (cbLandmark's lambda inside pf_->measure), then mcl3dl_particles_set.  The checker builds a
            pf::ParticleFilter of n particles per call and converts every state both ways, which a node keeping its own
            pf_ does not; so this is the round trip through the checker library, an estimate of a node's round trip, not
            a bound on it;
  poses:    mcl3dl_particles_get_poses (32 B per particle) against mcl3dl_particles_get (72 B per particle), the
            download publishParticles needed before.
Device calls are timed with the host clock around the call and with CUDA events recorded on the current stream just
before and after it.

    python profiles/pf_landmark_timing.py [--reps 7] [--sizes 65536,1048576]

The two paths alternate within each repetition.  Prints one JSON line per (event, size) with medians, min and max over
--reps, and the GPU's name and power limit.
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
from oracle import pf_landmark_checker as lc  # noqa: E402
from pf_events_timing import particle_set, stats  # noqa: E402
from scan_prepare_timing import gpu_info  # noqa: E402

MEASURED = np.zeros(1, synth.POSE)
MEASURED["px"], MEASURED["py"], MEASURED["qz"], MEASURED["qw"] = 1.0, -2.0, 0.1, 0.995
COV = np.diag([4.0, 4.0, 1.0, 0.1, 0.1, 0.3]).reshape(36)   # wide enough that the weights do not all underflow


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="65536,1048576")
    a = ap.parse_args()
    gpu = gpu_info()
    ref = lc.PfLandmarkChecker("reference")
    nd_a, si = engine.landmark_nd(COV)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    device = {"landmark": lambda e: e.particles_landmark_update(MEASURED, nd_a, si),
              "poses": lambda e: e.particles_get_poses()}

    def host(event, e):
        st, pr = e.particles_get()
        if event == "landmark":
            e.particles_set(st, ref.landmark(st, pr, MEASURED, nd_a, si)[0])

    for n in [int(s) for s in a.sizes.split(",")]:
        st, pr = particle_set(n)
        eng = engine.Engine((0,))
        for event in ("landmark", "poses"):
            eng.particles_set(st, pr)
            device[event](eng)   # warm-up of both paths
            host(event, eng)
            dev_ev, dev_wall, host_wall = [], [], []
            for _ in range(a.reps):
                eng.particles_set(st, pr)
                torch.cuda.synchronize()
                ev0.record()
                t0 = time.perf_counter()
                device[event](eng)
                t1 = time.perf_counter()
                ev1.record()
                ev1.synchronize()
                dev_wall.append((t1 - t0) * 1e3)
                dev_ev.append(ev0.elapsed_time(ev1))
                eng.particles_set(st, pr)
                t0 = time.perf_counter()
                host(event, eng)
                host_wall.append((time.perf_counter() - t0) * 1e3)
            rec = {"event": event, "n_particles": n, "gpu": gpu, "device_wall_ms": stats(dev_wall),
                   "device_event_ms": stats(dev_ev),
                   ("host_round_trip_ms" if event == "landmark" else "particles_get_ms"): stats(host_wall),
                   "speedup_median": float(np.median(host_wall) / np.median(dev_wall))}
            print(json.dumps(rec), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
