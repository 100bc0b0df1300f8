#!/usr/bin/env python
"""Time of the resident set's initial seed on an H100 against the host path a node takes without it.

  device: mcl3dl_particles_init (it synchronises), for the configured start's DiagonalNoiseGenerator and for cbPosition's
          MultivariateNoiseGenerator;
  host:   six standard normals per particle from numpy's generator (standing in for std::normal_distribution), the
          reference's own initUsingNoiseGenerator on one host thread through the checker library
          oracle/_ref/libmcl3dl_pf_init_ref.so, then mcl3dl_particles_set.  The checker builds a pf::ParticleFilter of n
          particles per call and converts every state, which a node keeping its own pf_ does not; so this is the round
          trip through the checker library, an estimate of a node's host path, not a bound on it.
Device calls are timed with the host clock around the call and with CUDA events recorded on the current stream just
before and after it.  The kernel writes 68 B of state and 4 B of probability per particle.

    python profiles/pf_init_timing.py [--reps 7] [--sizes 4096,65536,1048576]

The two paths alternate within each repetition.  Prints one JSON line per (generator, size) with medians, min and max
over --reps, and the GPU's name and power limit.
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
from oracle import pf_init_checker as pic  # noqa: E402
from pf_events_timing import stats  # noqa: E402
from scan_prepare_timing import gpu_info  # noqa: E402

POSE = np.array([1.0, -2.0, 0.1, 0.0, 0.0, 0.0998, 0.995], np.float32)
SIGMA = np.array([0.5, 0.5, 0.0, 0.0, 0.0, 0.2], np.float32)
COV = np.diag([0.25, 0.25, 0.0, 0.0, 0.0, 0.0685]).reshape(36)   # RViz's 2-D pose estimate


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="4096,65536,1048576")
    a = ap.parse_args()
    gpu = gpu_info()
    ref = pic.PfInitChecker("reference")
    mean6 = ref.mean(POSE)
    T = ref.transform(COV)
    gens = {"diagonal": (dict(sigma=SIGMA), dict(sigma=SIGMA)), "multivariate": (dict(norm_transform=T), dict(norm_transform=T))}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rng = np.random.default_rng(1)
    for n in [int(s) for s in a.sizes.split(",")]:
        eng = engine.Engine((0,))
        for name, (dev_kw, ref_kw) in gens.items():
            def host():
                z = rng.standard_normal((n, 6), dtype=np.float32)
                eng.particles_set(*ref.init(POSE, z, **ref_kw))

            eng.particles_init(n, mean6, 1, **dev_kw)   # warm-up of both paths
            host()
            dev_ev, dev_wall, host_wall = [], [], []
            for r in range(a.reps):
                torch.cuda.synchronize()
                ev0.record()
                t0 = time.perf_counter()
                eng.particles_init(n, mean6, r, **dev_kw)
                t1 = time.perf_counter()
                ev1.record()
                ev1.synchronize()
                dev_wall.append((t1 - t0) * 1e3)
                dev_ev.append(ev0.elapsed_time(ev1))
                t0 = time.perf_counter()
                host()
                host_wall.append((time.perf_counter() - t0) * 1e3)
            rec = {"generator": name, "n_particles": n, "gpu": gpu, "device_wall_ms": stats(dev_wall),
                   "device_event_ms": stats(dev_ev), "host_path_ms": stats(host_wall),
                   "speedup_median": float(np.median(host_wall) / np.median(dev_wall)),
                   "bytes_written": 72 * n}
            print(json.dumps(rec), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
