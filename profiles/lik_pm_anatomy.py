"""Where the c2 step of lik_kernel_nf_pm goes, segment by segment.

kernels.cuh's MCL3DL_PM_CUT ends the kernel after one segment of its chain and keeps that segment's results live:
1 returns at entry (the launch-and-drain floor of the same grid and parameter block), 2 after the pose is normalised,
3 after phase A (scan point, transform, directory load), 4 after the owner table, 5 after phase B (the candidate
loads), 6 before the fold; the whole kernel is the default.  Every variant is timed with bench.py's protocol: one CUDA
graph of --steps c2 steps on the 32 rotating stations between one event pair, and the same graph on one station
(L2-warm).  The variants run alternately, --runs rounds; the card, its power limit and the SM clock are read in the
same run.  Libraries are built with build.build(defines=..., out=...) into --lib-dir unless they are already there.

    python profiles/lik_pm_anatomy.py [--runs 3] [--steps 200] [--lib-dir DIR] [--extra NAME=LIB ...] [--out FILE]
    python profiles/lik_pm_anatomy.py --count    # host-side count over the 32 c2 stations (no GPU)
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import bench  # noqa: E402
from mcl_3dl_b200 import build, engine, synth  # noqa: E402

CUTS = [(1, "empty kernel"), (2, "+ pose normalised"), (3, "+ phase A"), (4, "+ owner table"), (5, "+ phase B"),
        (6, "+ owners' terms"), (0, "+ fold = whole kernel")]
UNIT, LOADS = 4, 4  # kNfU points per warp trip, kNfB candidate loads per lane and round


def variant_libs(lib_dir):
    os.makedirs(lib_dir, exist_ok=True)
    want = [(name, os.path.join(lib_dir, "pm_cut%d.so" % cut), cut) for cut, name in CUTS]

    def make(item):
        _, path, cut = item
        if not os.path.exists(path):
            build.build(defines=["MCL3DL_PM_CUT=%d" % cut], out=path)
    with ThreadPoolExecutor(len(want)) as ex:
        list(ex.map(make, want))
    return [(name, path) for name, path, _ in want]


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                       text=True)
    return dict(zip(q.split(","), (c.strip() for c in r.stdout.strip().split(","))))


def time_variants(libs, steps, runs):
    import torch
    dev = torch.device("cuda:0")
    s, _, _, P = bench.build_scene("c2", 0, 1)
    stations = bench.build_stations("c2", 0, 1, s, 32)
    n_lik = len(s["lik"])

    def up(a):
        return torch.from_numpy(bench.as_u8(a)).to(dev)
    dst = [(up(st["particles"]), up(st["lik"])) for st in stations]
    d_b = torch.zeros(16, dtype=torch.uint8, device=dev)
    d_o = torch.from_numpy(np.ascontiguousarray(s["origins"], dtype=np.float32)).to(dev)
    d_out = torch.zeros(P * 24, dtype=torch.uint8, device=dev)

    arms = []
    for name, path in libs:
        eng = engine.Engine((0,), lib_path=path)
        eng.set_map(s["map"], engine.LikParams(dist_weight=bench.DIST_WEIGHT), None)

        def step_on(i, eng=eng):
            sp, sl = dst[i % len(dst)]
            eng.measure_device(sp.data_ptr(), P, sl.data_ptr(), n_lik, d_b.data_ptr(), 0, d_o.data_ptr(),
                               len(s["origins"]), d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)

        def capture(pick, step_on=step_on):
            for i in range(3):
                step_on(pick(i))
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for i in range(steps):
                    step_on(pick(i))
            g.replay()
            torch.cuda.synchronize()
            return g
        arms.append((name, eng, capture(lambda i: i), capture(lambda i: 0)))

    def replay_us(g):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        return 1e3 * a.elapsed_time(b) / steps

    clock = bench.ClockSampler(0)
    clock.start()
    res = {name: {"rotate": [], "same": []} for name, _, _, _ in arms}
    for _ in range(runs):
        for name, _, g_rot, g_same in arms:
            res[name]["rotate"].append(replay_us(g_rot))
            res[name]["same"].append(replay_us(g_same))
    clk = clock.stop()
    for _, eng, _, _ in arms:
        eng.close()
    return res, clk


def table(res, names):
    lines = ["| cut | rotating µs/step: median (runs) | segment µs | L2-warm µs/step: median (runs) | segment µs |",
             "|---|---|---|---|---|"]
    prev = {"rotate": 0.0, "same": 0.0}
    for name in names:
        row = [name]
        for kind in ("rotate", "same"):
            v = res[name][kind]
            med = float(np.median(v))
            row.append("%.2f (%s)" % (med, ", ".join("%.2f" % x for x in v)))
            row.append("%+.2f" % (med - prev[kind]))
            prev[kind] = med
        lines.append("| " + " | ".join(row) + " |")
    return "\n".join(lines)


def counts():
    """Per warp trip of lik_kernel_nf_pm over the 32 c2 stations (32 consecutive particles x UNIT consecutive points):
    W (flattened slots), the longest list per u, the iterations the serial owner fill took (sum over u of the longest
    list), the owner table's marks, words and scan rounds, the phase-B rounds (ceil(W / (32 * LOADS))) and the share of
    evals without candidates."""
    tmp = tempfile.mkdtemp()
    so = os.path.join(tmp, "liblikpmcounts.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", so,
                        os.path.join(ROOT, "profiles", "lik_pm_counts.cpp")], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(r.stderr)
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.lik_pm_counts.argtypes = [vp, sz, vp, vp, sz, vp, sz, vp]
    s, _, _, P = bench.build_scene("c2", 0, 1)
    stations = bench.build_stations("c2", 0, 1, s, 32)
    lik = engine.LikParams(dist_weight=bench.DIST_WEIGHT)
    mp = np.ascontiguousarray(s["map"], dtype=synth.POINT)
    W, longest, fill, rounds, marks, ovf, zero, evals = [], [], [], [], [], 0, 0, 0
    for st in stations:
        poses = np.ascontiguousarray(st["particles"], dtype=synth.POSE)
        pts = np.ascontiguousarray(st["lik"], dtype=synth.POINT)
        n = len(pts)
        cnt = np.zeros((len(poses), n), np.int32)
        rc = L.lik_pm_counts(mp.ctypes.data, len(mp), C.byref(lik), poses.ctypes.data, len(poses), pts.ctypes.data,
                             n, cnt.ctypes.data)
        assert rc == 0
        ovf += int((cnt < 0).sum())
        zero += int((cnt == 0).sum())
        evals += cnt.size
        c = np.maximum(cnt, 0)
        n_pad = -(-n // UNIT) * UNIT
        c = np.pad(c, ((0, 0), (0, n_pad - n)))
        trips = c.reshape(len(poses) // 32, 32, n_pad // UNIT, UNIT)  # warp, lane, trip, u
        w = trips.sum(axis=(1, 3)).ravel()
        mx = trips.max(axis=1)                                        # warp, trip, u
        W.append(w)
        longest.append(mx.reshape(-1, UNIT))
        fill.append(mx.sum(axis=2).ravel())
        rounds.append(-(-w // (32 * LOADS)))
        marks.append((trips > 0).sum(axis=(1, 3)).ravel())
    W, longest, fill, rounds, marks = (np.concatenate(x) for x in (W, longest, fill, rounds, marks))

    def stat(x):
        return {"mean": round(float(x.mean()), 2), "p50": float(np.median(x)), "p90": float(np.quantile(x, 0.9)),
                "max": int(x.max())}
    # the owner table (kernels.cuh: nf_warp_scan) of a trip's one pass: the marks (lists with candidates), the 32-bit
    # words that hold it, and its scan rounds of 32 lanes x 16 bytes
    return {"warp_trips": int(len(W)), "W_slots": stat(W), "longest_list_per_u": stat(longest),
            "owner_fill_iterations": stat(fill), "owner_table_marks": stat(marks),
            "owner_table_words": stat(-(-W // 4)), "owner_scan_rounds": stat(-(-W // 512)),
            "phase_b_rounds": stat(rounds), "trips_over_1024_slots": int((W > 1024).sum()),
            "evals_without_candidates": round(zero / max(evals, 1), 4), "overflow_evals": ovf}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--lib-dir", default=None, help="where the cut variants are built or found (default: a temp dir)")
    ap.add_argument("--extra", action="append", default=[], metavar="NAME=LIB",
                    help="another whole-kernel library timed alternately with the variants")
    ap.add_argument("--count", action="store_true", help="only the host-side count over the 32 c2 stations")
    ap.add_argument("--out", default=None, help="also write the results as JSON")
    args = ap.parse_args()
    if args.count:
        out = {"count": counts()}
        print(json.dumps(out, indent=1))
    else:
        libs = variant_libs(args.lib_dir or tempfile.mkdtemp(prefix="lik_pm_anatomy_"))
        libs += [tuple(e.split("=", 1)) for e in args.extra]
        res, clk = time_variants(libs, args.steps, args.runs)
        out = {"card": card(), "sm_clock": clk, "steps": args.steps, "runs": args.runs, "us_per_step": res}
        print("card: %s, power limit %s, max SM clock %s; SM clock during the runs: %s MHz" % (
            out["card"].get("name"), out["card"].get("power.limit"), out["card"].get("clocks.max.sm"),
            clk.get("sm_mhz")))
        print(table(res, [name for _, name in CUTS]))
        for name, _ in libs[len(CUTS):]:
            print("%s: rotating %s, L2-warm %s" % (name, ["%.2f" % x for x in res[name]["rotate"]],
                                                    ["%.2f" % x for x in res[name]["same"]]))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
