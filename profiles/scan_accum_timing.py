#!/usr/bin/env python
"""Cloud accumulation on the device against the node's host path (include/mcl3dl_b200.h: mcl3dl_scan_accumulate).

    python profiles/scan_accum_timing.py [--reps 30] [--warmup 5]

Host clock around each call; every call ends in a device synchronise.  Prints JSON lines, each with the GPU's name and
power limit:
  accumulate:  one mcl3dl_scan_accumulate of a 130 k-point cloud at point_step 16 / 32 / 48 (the raw bytes go up, the
               first transform and the labels run on the device);
  prepare:     mcl3dl_scan_prepare_accumulated on a 10-cloud, 1.3 M-point accumulation against mcl3dl_scan_prepare on the
               cloud the node would have built from the same clouds (its 21 MB upload included), alternating, at the
               node's leaves (0.1, 0.1, 0.05); the five stages of both are checked equal in the same run;
  host:        profiles/accum_host_standin.cpp (g++ -O2, this machine's CPU), a STAND-IN for the host work the node no
               longer does (tf2 / PCL are not installed: their loops are restated; see that file).
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from mcl_3dl_b200 import engine  # noqa: E402
import accum_restate as A  # noqa: E402
from scan_prepare_timing import accumulated_cloud, gpu_info  # noqa: E402

LEAF = (0.1, 0.1, 0.05)
N_CLOUD = 130_000
OFFSETS = {16: (0, 4, 8), 32: (0, 4, 8), 48: (16, 20, 24)}


def cpu_info():
    """What /proc/cpuinfo says of the first CPU (some virtual machines report the model name as "unknown", so the
    vendor, family, model and stepping numbers are kept too) and the number of CPUs this process may use."""
    keys = ("model name", "vendor_id", "cpu family", "model", "stepping", "cpu MHz")
    info = {}
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if not line.strip():
                    break
                k, _, v = line.partition(":")
                if k.strip() in keys:
                    info[k.strip()] = v.strip()
    except OSError as e:
        info["error"] = str(e)
    info["cpus"] = len(os.sched_getaffinity(0))
    return info


def stats(t):
    t = np.asarray(t)
    return {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(t.min()), 3), "max_ms": round(float(t.max()), 3),
            "p10_ms": round(float(np.percentile(t, 10)), 3), "p90_ms": round(float(np.percentile(t, 90)), 3)}


def sensor_clouds(k=10):
    """The 1.3 M-point scene of scan_prepare_timing split into k clouds at point_step 32, each in its own sensor frame
    (the inverse of its sensor -> odom transform applied in double first, so the accumulation is the scene again)."""
    pts = accumulated_cloud(N_CLOUD * k)
    xyz = np.stack([pts["x"], pts["y"], pts["z"]], 1).astype(np.float64)
    rng = np.random.default_rng(3)
    out = []
    for i in range(k):
        part = xyz[i * N_CLOUD:(i + 1) * N_CLOUD]
        yaw = rng.uniform(-0.2, 0.2)
        q = (0.0, 0.0, np.sin(yaw / 2), np.cos(yaw / 2))
        t = tuple(rng.normal(0, 0.1, 3))
        c, s = np.cos(yaw), np.sin(yaw)
        local = (part - np.asarray(t)) @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
        data, row_step = A.pack_cloud(local.astype(np.float32), N_CLOUD, 1, 32, OFFSETS[32], 0, rng=rng)
        out.append(dict(xyz=local.astype(np.float32), data=data, row_step=row_step, tf=(t, q)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    gpu = gpu_info()
    e = engine.Engine((0,))
    rng = np.random.default_rng(1)
    tf = ((0.3, -0.2, 0.1), (0.01, 0.02, 0.3, 0.95))
    # 1. one accumulate per 130 k-point cloud
    for ps in (16, 32, 48):
        data, row_step = A.pack_cloud(A.random_xyz(rng, N_CLOUD), N_CLOUD, 1, ps, OFFSETS[ps], 0, rng=rng)
        t = []
        for rep in range(a.warmup + a.reps):
            e.scan_accumulate_clear()
            t0 = time.perf_counter()
            e.scan_accumulate(data, N_CLOUD, 1, ps, row_step, OFFSETS[ps], True, *tf)
            dt = (time.perf_counter() - t0) * 1e3
            if rep >= a.warmup:
                t.append(dt)
        print(json.dumps(dict({"what": "scan_accumulate", "gpu": gpu, "points": N_CLOUD, "point_step": ps,
                               "bytes": len(data), "reps": a.reps}, **stats(t))))
    # 2. prepare on the accumulation vs scan_prepare on the node's host cloud, alternating
    clouds = sensor_clouds()
    base = ((0.05, -0.1, 0.0), (0.0, 0.0, 0.0998, 0.995))
    e.scan_accumulate_clear()
    for c in clouds:
        e.scan_accumulate(c["data"], N_CLOUD, 1, 32, c["row_step"], OFFSETS[32], True, *c["tf"])
    node = A.node_cloud([(c["xyz"], True, c["tf"]) for c in clouds], base)
    sp = engine.ScanParams(downsample=LEAF, lik_num_points=96, beam_num_points=3, seed=1)
    ta, tb, same = [], [], True
    for rep in range(a.warmup + a.reps):
        t0 = time.perf_counter()
        ia = e.scan_prepare_accumulated(sp, *base)
        t1 = time.perf_counter()
        if rep == a.warmup:
            sa = [e.scan_get(w).tobytes() for w in range(5)]
        t2 = time.perf_counter()
        ib = e.scan_prepare(node, sp)
        t3 = time.perf_counter()
        if rep == a.warmup:
            same = ia == ib and sa == [e.scan_get(w).tobytes() for w in range(5)]
        if rep >= a.warmup:
            ta.append((t1 - t0) * 1e3)
            tb.append((t3 - t2) * 1e3)
    print(json.dumps(dict({"what": "scan_prepare_accumulated", "gpu": gpu, "clouds": len(clouds), "n_raw": ia["n_raw"],
                           "info": ia, "reps": a.reps, "stages_equal_to_scan_prepare": bool(same)}, **stats(ta))))
    print(json.dumps(dict({"what": "scan_prepare(host cloud)", "gpu": gpu, "n_raw": ib["n_raw"], "reps": a.reps}, **stats(tb))))
    e.close()
    # 3. the host stand-in
    d = tempfile.mkdtemp()
    try:
        exe = os.path.join(d, "standin")
        r = subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "profiles", "accum_host_standin.cpp")],
                           capture_output=True, text=True)
        if r.returncode != 0:
            print(json.dumps({"what": "host stand-in", "error": r.stderr[-500:]}))
        else:
            out = subprocess.run([exe, "10", str(N_CLOUD), "32", str(a.reps)], capture_output=True, text=True).stdout.split()
            cpu = cpu_info()
            print(json.dumps({"what": "host stand-in (restated tf2/PCL loops, g++ -O2; not PCL itself)", "cpu": cpu,
                              "clouds": 10, "points": 10 * N_CLOUD, "point_step": 32, "reps": a.reps,
                              "median_ms": float(out[0]), "min_ms": float(out[1]), "max_ms": float(out[2])}))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
