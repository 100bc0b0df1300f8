#!/usr/bin/env python
"""The map window on a map whose whole likelihood lattice is refused (include/mcl3dl_b200.h, "Map window").

    python profiles/map_window_timing.py [--copies 4] [--steps 200]

Map: copies of synth.warehouse_map(400 000) 1.5 km apart on a square grid (the whole lattice is far above 2^31 cells),
the KD caster and the likelihood model at the node's defaults (dist_weight 1 1 5, match_dist_min 0.2).  Reports, as JSON
lines with the GPU's name and power limit:
  set_map:       host clock of mcl3dl_set_map of the whole map (windowed staging: the points and boxes only);
  first_window:  stream time of the first window (mcl3dl_map_window_info.rebuild_ms: the selection and the build, event to
                 event, with the build's own count readbacks) and its lattice;
  rebuild:       stream time of the window rebuilds (as rebuild_ms) as the particles jump from copy to copy;
  check:         the per-call cost of the window check: measure_update_prepared on the windowed engine with the window in
                 place, against the same call on an engine that staged only the local copy, alternating (CUDA events
                 are not usable around a synchronising call: host clock, median of --steps);
Every timed call is checked to give the same summary as the local engine.
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

F = np.float32
PITCH = 1500.0


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:  # noqa: BLE001
        return "unknown (%s)" % ex


def emit(gpu, **kv):
    kv["gpu"] = gpu
    print(json.dumps(kv), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--copies", type=int, default=4)
    ap.add_argument("--steps", type=int, default=200)
    a = ap.parse_args()
    gpu = gpu_info()
    engine.load_library()
    mp, info = synth.warehouse_map(400_000, seed=7)
    side = int(np.ceil(np.sqrt(a.copies)))
    offs = [(PITCH * (k % side), PITCH * (k // side)) for k in range(a.copies)]
    parts = []
    for ox, oy in offs:
        c = mp.copy()
        c["x"] = (c["x"].astype(np.float64) + ox).astype(F)
        c["y"] = (c["y"].astype(np.float64) + oy).astype(F)
        parts.append(c)
    big = np.concatenate(parts)
    lik = engine.LikParams(dist_weight=(1, 1, 5))
    beam = engine.beam_params_from_reference(num_points_default=64, dda_grid_size=0.2, use_raycast_using_dda=0)
    e = engine.Engine((0,))
    t0 = time.perf_counter()
    e.set_map(big, lik, beam)
    emit(gpu, what="set_map", n_points=len(big), host_ms=(time.perf_counter() - t0) * 1e3, window=e.map_window_info())
    L = info["L"]
    sp = engine.ScanParams(lik_num_points=384, beam_num_points=64)
    n_p = 4096
    local = engine.Engine((0,))
    rebuilds = []
    for k, (ox, oy) in enumerate(offs):
        pos = np.array([ox + 0.5 * L, oy + 0.5 * L, 0.6])
        q = synth.quat_from_rpy(np.array([[0.0, 0.0, 0.3]]))[0]
        raw = synth.make_scan(parts[k], pos, q, 20_000, 0.5, 10.0, seed=40 + k)
        origins = synth.sensor_origins(1)
        mean6 = np.array([pos[0], pos[1], pos[2], 0.0, 0.0, 0.3], F)
        sig = np.array([0.2, 0.2, 0.05, 0.02, 0.02, 0.1], F)
        local.set_map(parts[k], lik, beam)
        for x in (e, local):
            x.particles_init(n_p, mean6, 1, sigma=sig)
            x.scan_prepare(raw, sp)
        before = e.map_window_info()["rebuilds"]
        s_w = e.particles_measure_update_prepared(origins)
        wi = e.map_window_info()
        if k == 0:
            emit(gpu, what="first_window", stream_ms=wi["rebuild_ms"], dims=wi["dims"], box_min=wi["box_min"],
                 box_max=wi["box_max"], bytes=e.map_info().device_bytes)
        elif wi["rebuilds"] > before:
            rebuilds.append(wi["rebuild_ms"])
        s_l = local.particles_measure_update_prepared(origins)
        assert s_w == s_l, (s_w, s_l)
        if k == 0:
            tw, tl = [], []
            for _ in range(a.steps):
                for x, acc in ((e, tw), (local, tl)):
                    x.particles_init(n_p, mean6, 1, sigma=sig)
                    t = time.perf_counter()
                    x.particles_measure_update_prepared(origins)
                    acc.append((time.perf_counter() - t) * 1e3)
            assert e.map_window_info()["rebuilds"] == wi["rebuilds"]
            emit(gpu, what="check", particles=n_p, n_lik=384, n_beam=64, windowed_ms=float(np.median(tw)),
                 local_ms=float(np.median(tl)), check_ms=float(np.median(tw) - np.median(tl)), steps=a.steps)
    emit(gpu, what="rebuild", stream_ms=rebuilds, rebuilds=e.map_window_info()["rebuilds"])
    e.close()
    local.close()


if __name__ == "__main__":
    main()
