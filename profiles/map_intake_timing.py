#!/usr/bin/env python
"""The map intake on the device against the node's host path (include/mcl3dl_b200.h: mcl3dl_map_load).

    python profiles/map_intake_timing.py [--reps 3] [--maps c2,c4]

Host clock around each call; every call ends in a device synchronise.  Prints JSON lines, each with the GPU's name and
power limit.  Input: bench.py's c2 (1 M) and c4 (10 M) maps, each point twice with a 2 cm jitter so that the map's
VoxelGrid really reduces it, as PointCloud2 bytes at point_step 32 (x y z . intensity label ..).
  load:   (a) host path: the VoxelGrid of tests/hostsim/scan_hostsim.cpp (g++ -O2, one thread of the GPU machine's CPU;
          the device functions compiled for the host, a STAND-IN for pcl::VoxelGrid, which is not installed), the
          packing into mcl3dl_point, and mcl3dl_set_map; (b) mcl3dl_map_load.  Both staged maps are checked equal.
  patch:  10 k and 100 k raw points inside the map: (a) host VoxelGrid + mcl3dl_map_append; (b) mcl3dl_map_update_set +
          mcl3dl_map_update_commit.
  get:    the mcl3dl_map_get readback of the staged map (points and intensities).
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
from mcl_3dl_b200 import engine, synth  # noqa: E402
import bench  # noqa: E402

LEAF = (0.1, 0.1, 0.1)
UPDATE_LEAF = (0.1, 0.1, 0.1)
XYZIL = np.dtype({"names": ["x", "y", "z", "intensity", "label"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u4"],
                  "offsets": [0, 4, 8, 16, 20], "itemsize": 32})


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "unknown (%s)" % e


def host_voxel_lib(tmp):
    so = os.path.join(tmp, "libscanhs.so")
    src = os.path.join(ROOT, "tests", "hostsim", "scan_hostsim.cpp")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so, src], check=True)
    L = C.CDLL(so)
    L.hostsim_scan_voxel_grid.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.hostsim_scan_voxel_grid.restype = C.c_long
    return L


def dense_cloud(m, copies, seed):
    rng = np.random.default_rng(seed)
    n = len(m)
    out = np.zeros(n * copies, XYZIL)
    for k in range(copies):
        sl = slice(k * n, (k + 1) * n)
        for f in ("x", "y", "z"):
            out[f][sl] = m[f] + rng.normal(0.0, 0.02, n).astype(np.float32)
        out["label"][sl] = m["label"]
    out["intensity"] = rng.uniform(0, 100, len(out)).astype(np.float32)
    return out


def host_path(L, cloud, leaf):
    """fromROSMsg + VoxelGrid on one thread + the packing into mcl3dl_point."""
    pts = np.zeros(len(cloud), synth.POINT)
    for f in ("x", "y", "z", "label"):
        pts[f] = cloud[f]
    out = np.zeros(len(pts), synth.POINT)
    m = L.hostsim_scan_voxel_grid(pts.ctypes.data, len(pts), np.asarray(leaf, np.float32).ctypes.data, out.ctypes.data)
    return out[:m] if m >= 0 else pts


def timed(f, reps):
    ts = []
    r = None
    for _ in range(reps):
        t0 = time.perf_counter()
        r = f()
        ts.append((time.perf_counter() - t0) * 1e3)
    return sorted(ts), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--maps", default="c2,c4")
    args = ap.parse_args()
    gpu = gpu_info()
    with tempfile.TemporaryDirectory() as tmp:
        L = host_voxel_lib(tmp)
        for wl in args.maps.split(","):
            s, dda, _, _ = bench.build_scene(wl, 0, 1)
            lik = engine.LikParams(dist_weight=bench.DIST_WEIGHT)
            beam = engine.beam_params_from_reference(dda_grid_size=dda)
            cloud = dense_cloud(s["map"], 2, 7)
            data = cloud.view(np.uint8)
            e = engine.Engine((0,))

            def load():
                return e.map_load(data, len(cloud), 1, 32, 32 * len(cloud), (0, 4, 8), LEAF, lik, beam, 16, 20)

            def host_load():
                e.set_map(host_path(L, cloud, LEAF), lik, beam)

            load()  # warm-up of both paths
            host_load()
            t_dev, info = [], None
            t_host = []
            for _ in range(args.reps):  # alternating
                t, info = timed(load, 1)
                t_dev += t
                t_host += timed(host_load, 1)[0]
            host_map = e.map_get()[0]
            load()
            same = e.map_get()[0].tobytes() == host_map.tobytes()
            print(json.dumps({"gpu": gpu, "map": wl, "leg": "load", "n_raw": len(cloud), "n_staged": info["n_staged"],
                              "map_load_ms": t_dev, "intake_device_ms": info["device_ms"],
                              "build_ms": e.map_info().build_ms, "host_voxelgrid_pack_set_map_ms": sorted(t_host),
                              "staged_maps_equal": same}), flush=True)
            t, _ = timed(e.map_get, args.reps)
            print(json.dumps({"gpu": gpu, "map": wl, "leg": "get", "n": len(host_map), "map_get_ms": t}), flush=True)
            for n_patch in (10_000, 100_000):
                rng = np.random.default_rng(n_patch)
                patch = cloud[rng.integers(0, len(cloud), n_patch)].copy()
                for f in ("x", "y", "z"):
                    patch[f] += rng.normal(0.0, 0.01, n_patch).astype(np.float32)
                pd = patch.view(np.uint8)
                t_dev, t_host, infos = [], [], []
                for _ in range(args.reps):
                    t0 = time.perf_counter()
                    e.map_update_set(pd, n_patch, 1, 32, 32 * n_patch, (0, 4, 8), UPDATE_LEAF, 16, 20)
                    infos.append(e.map_update_commit())
                    t_dev.append((time.perf_counter() - t0) * 1e3)
                    t0 = time.perf_counter()
                    e.map_append(host_path(L, patch, UPDATE_LEAF))
                    t_host.append((time.perf_counter() - t0) * 1e3)
                print(json.dumps({"gpu": gpu, "map": wl, "leg": "patch", "n_raw": n_patch,
                                  "update_set_commit_ms": sorted(t_dev), "host_voxelgrid_map_append_ms": sorted(t_host),
                                  "incremental": [i["incremental"] for i in infos]}), flush=True)
            e.close()


if __name__ == "__main__":
    main()
