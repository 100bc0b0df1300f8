#!/usr/bin/env python
"""Time of the resident set's odometry-noise redraw, expansion noise and IMU gravity update on an H100, against a host
round trip through the reference's code for each of them.

  device:  mcl3dl_particles_redraw_odom_noise / _noise / _imu_update (the calls synchronise): the host clock around the
           call, and CUDA events recorded on the current stream just before and after it (they bracket the call's work
           and its launch overhead);
  host:    mcl3dl_particles_get, the reference's own code on one host thread through the checker library
           oracle/_ref/libmcl3dl_pf_events_ref.so (the node's redraw lambda through pf_->predict,
           addNoiseUsingNoiseGenerator, ImuMeasurementModelGravity inside pf_->measure), then mcl3dl_particles_set.  The
           normal draws come from numpy.  The checker builds a pf::ParticleFilter of n particles per call and converts
           every state both ways, which a node keeping its own pf_ does not; so this is the round trip through the checker
           library, an estimate of a node's round trip, not a bound on it.

    python profiles/pf_events_timing.py [--reps 7] [--sizes 65536,1048576]

The device and host paths alternate within each repetition.  Prints one JSON line per (event, size) with medians, min and
max over --reps, and the GPU's name and power limit.
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
from oracle import pf_events_checker as pc  # noqa: E402
from scan_prepare_timing import gpu_info  # noqa: E402

SIG_ODOM = (0.01, 0.01, 0.01, 0.01)
SIG_POS, SIG_RPY = (0.2, 0.2, 0.05), (0.02, 0.02, 0.1)
ACC, ACC_VAR = (0.05, -0.02, 0.99), 0.3


def stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def particle_set(n, seed=0):
    rng = np.random.default_rng(seed)
    st = np.zeros(n, synth.STATE)
    st["pos"] = rng.uniform(-20, 20, (n, 3))
    q = rng.normal(0, 0.05, (n, 4))
    q[:, 3] = 1
    st["rot"] = q / np.linalg.norm(q, axis=1, keepdims=True)
    return st, np.full(n, 1.0 / n, np.float32)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="65536,1048576")
    a = ap.parse_args()
    gpu = gpu_info()
    ref = pc.PfEventsChecker("reference")
    rng = np.random.default_rng(1)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    device = {"redraw": lambda e: e.particles_redraw_odom_noise(*SIG_ODOM, seed=5),
              "noise": lambda e: e.particles_noise(SIG_POS, SIG_RPY, seed=5),
              "imu": lambda e: e.particles_imu_update(ACC, ACC_VAR)}

    def host(event, e, n):
        st, pr = e.particles_get()
        if event == "redraw":
            st = ref.redraw(st, rng.standard_normal((n, 4), np.float32), *SIG_ODOM)
        elif event == "noise":
            org = (rng.standard_normal((n, 6), np.float32) * np.array(SIG_POS + SIG_RPY, np.float32)).astype(np.float32)
            st = ref.noise(st, org)
        else:
            pr = ref.imu(st, pr, ACC, ACC_VAR)[0]
        e.particles_set(st, pr)

    for n in [int(s) for s in a.sizes.split(",")]:
        st, pr = particle_set(n)
        eng = engine.Engine((0,))
        for event in ("redraw", "noise", "imu"):
            eng.particles_set(st, pr)
            device[event](eng)   # warm-up of both paths
            host(event, eng, n)
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
                host(event, eng, n)
                host_wall.append((time.perf_counter() - t0) * 1e3)
            rec = {"event": event, "n_particles": n, "gpu": gpu, "device_wall_ms": stats(dev_wall),
                   "device_event_ms": stats(dev_ev), "host_round_trip_ms": stats(host_wall),
                   "speedup_median": float(np.median(host_wall) / np.median(dev_wall))}
            print(json.dumps(rec), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
