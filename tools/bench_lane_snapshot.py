#!/usr/bin/env python
"""Cost of lane snapshots (aloam_lane_save / aloam_lane_restore).
1. Save and restore against store size: a mapped lane whose cube store is grown to about 0.1, 0.3 and 1 M points (thin-map frames
   of uniform clouds at a 5 cm leaf, so nothing is filtered away), saved to a device tensor and to a pinned host tensor and
   restored from each; median microseconds and GB/s of the snapshot bytes.  Each restored lane is saved again and compared.
2. Time slicing: 32 VLP-16 trajectories over 16 lanes, mapped -- once in two groups of 16 run to their end (no slicing), once
   round-robin in slices of --slice scans with a save and a restore at every swap; useful scans per second of each (median of
   --repeats runs, alternating) and whether every trajectory's map poses are bit-identical between the two.
Every line carries the GPU name and power limit read in the same run.
usage: python tools/bench_lane_snapshot.py [--repeats 5] [--scans 20] [--slice 5]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("a-loam_b200")
synth = importlib.import_module("a-loam_b200.synth")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception:
        return "unknown", "unknown"


def _median_us(fn, reps, torch):
    us = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        us.append(1e6 * (time.perf_counter() - t0))
    return float(np.median(us))


def bench_save_restore(torch, gpu, R):
    rng = np.random.default_rng(7)
    npts = 65536
    ctx = pkg.Aloam(n_scans=16, max_points=npts, max_map_points=400000, line_res=0.05, plane_res=0.05)
    raw = synth.scan("VLP-16", 0, n_az=900)
    d_raw = torch.from_numpy(raw).cuda()
    # lane 0 runs a mapped trajectory (its START frame); aloam_mapper_step then grows lane 0's store with thin frames
    ctx.scan_stream_lanes(np.array([[d_raw.data_ptr()]], np.uint64), np.array([[raw.shape[0]]]), np.array([[pkg.LANE_START]], np.int32), True)
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    for target in (100_000, 300_000, 1_000_000):
        while ctx.mapper_export_size(pkg.EXPORT_MAP) < target:
            surf = np.zeros((npts, 4), np.float32)
            surf[:, :3] = rng.uniform([-120, -120, -20], [120, 120, 20], size=(npts, 3))
            surf[:, 3] = rng.uniform(0, 16, npts)
            ctx.mapper_step(empty, surf, ident, np.zeros(3))
        ref = ctx.lane_save(0)
        n = len(ref)
        bufs = {"device": torch.empty(n, dtype=torch.uint8, device="cuda"), "pinned_host": torch.empty(n, dtype=torch.uint8).pin_memory()}
        res = {}
        for name, buf in bufs.items():
            save = _median_us(lambda: ctx.lane_save(0, buf), R, torch)
            restore = _median_us(lambda: ctx.lane_restore(0, buf), R, torch)
            assert ctx.lane_save(0).tobytes() == ref.tobytes(), name   # the restored lane saves the same bytes
            res[name] = {"save_us": round(save, 1), "restore_us": round(restore, 1), "save_GB_per_s": round(n / save / 1e3, 1),
                         "restore_GB_per_s": round(n / restore / 1e3, 1)}
        print(json.dumps({"bench": "lane_snapshot", "map_points": int(pkg.snapshot_info(ref)["map_points"]), "bytes": n, **res,
                          "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)
    ctx.close()


def _lane_call(ctx, lanes, plan):
    """plan = {lane: [(address, points, op), ...]}: one mapped lanes call; {lane: map poses of its entries}"""
    steps = max(len(e) for e in plan.values())
    ptrs, counts, ops = np.zeros((steps, lanes), np.uint64), np.zeros((steps, lanes), np.int64), np.zeros((steps, lanes), np.int32)
    for lane, entries in plan.items():
        for k, (p, n, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    _, mp = ctx.scan_stream_lanes(ptrs, counts, ops, True)
    return {lane: mp[:len(e), lane] for lane, e in plan.items()}


def _entries(dev, i0, i1):
    return [(d.data_ptr(), d.shape[0], pkg.LANE_START if i == 0 else pkg.LANE_SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def run_unsliced(ctx, dev, lanes, L):
    out = {}
    for g in range(0, len(dev), lanes):
        res = _lane_call(ctx, lanes, {i: _entries(dev[g + i], 0, L) for i in range(min(lanes, len(dev) - g))})
        out.update({g + i: m for i, m in res.items()})
    return out


def run_sliced(ctx, dev, lanes, L, S):
    n = len(dev)
    pos, saved, parts = [0] * n, {}, {t: [] for t in range(n)}
    order, rnd = list(range(n)), 0
    while any(p < L for p in pos):
        live = [t for t in order if pos[t] < L]
        group = live[:lanes]
        for i, t in enumerate(group):
            if t in saved:
                ctx.lane_restore(i, saved.pop(t))
        res = _lane_call(ctx, lanes, {i: _entries(dev[t], pos[t], min(pos[t] + S, L)) for i, t in enumerate(group)})
        for i, t in enumerate(group):
            parts[t].append(res[i])
            pos[t] += len(res[i])
            if pos[t] < L:
                saved[t] = ctx.lane_save(i)
        order = order[len(group):] + group   # round robin
        rnd += 1
    return {t: np.concatenate(p) for t, p in parts.items()}


def bench_slicing(torch, gpu, R, L, S):
    lanes, n = 16, 32
    trajs = [[synth.scan("VLP-16", k, seed=synth.BASE_SEED + 700 + t, n_az=900) for k in range(L)] for t in range(n)]
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    ctx = {m: pkg.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, max_batch=lanes, max_ring_points=4096) for m in ("whole", "sliced")}
    run = {"whole": lambda: run_unsliced(ctx["whole"], dev, lanes, L), "sliced": lambda: run_sliced(ctx["sliced"], dev, lanes, L, S)}
    secs, poses = {"whole": [], "sliced": []}, {}
    for r in range(R + 1):   # run 0 warms up
        for m in (("whole", "sliced") if r % 2 == 0 else ("sliced", "whole")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            poses[m] = run[m]()
            torch.cuda.synchronize()
            if r > 0:
                secs[m].append(time.perf_counter() - t0)
    same = all(np.array_equal(poses["whole"][t], poses["sliced"][t]) for t in range(n))
    useful = n * L
    rate = {m: useful / float(np.median(v)) for m, v in secs.items()}
    for c in ctx.values():
        c.close()
    print(json.dumps({"bench": "time_slicing", "sensor": "VLP-16", "lanes": lanes, "trajectories": n, "scans_each": L, "slice": S,
                      "useful_scans_per_s_unsliced": round(rate["whole"], 1), "useful_scans_per_s_sliced": round(rate["sliced"], 1),
                      "sliced_over_unsliced": round(rate["sliced"] / rate["whole"], 3), "map_poses_identical": bool(same),
                      "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--slice", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_snapshot needs a CUDA device")
    gpu = gpu_info()
    bench_save_restore(torch, gpu, max(a.repeats, 1) * 4)
    bench_slicing(torch, gpu, max(a.repeats, 1), a.scans, a.slice)


if __name__ == "__main__":
    main()
