#!/usr/bin/env python
"""Cost of the mapper's published clouds (aloam_set_registered_sink, aloam_mapper_export).
1. Registered sink: HDL-32 scans through aloam_scan_stream_mapped_batch at mapping_skip_frame 1 and 3, 1 and 16 lanes, on two
   contexts fed the same device-resident scans -- one without a sink, one with a device sink -- alternating call by call.  One JSON
   line per (k, lanes): median ms per step of each, and whether the map poses are bit-identical.
2. Export: a cube store of about 1 M points (thin-map frames of uniform clouds at a 5 cm leaf, so nothing is filtered away), then
   the whole map to a device tensor, a pinned host tensor and a pageable numpy array; median microseconds of each and GB/s.
Every line carries the GPU name and power limit read in the same run.
usage: python tools/bench_mapper_clouds.py [--steps 20] [--warmup 3] [--repeats 3]"""
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


def bench_sink(torch, gpu, k, B, K, W, R):
    n = 1 + W + R * K
    scans = [[synth.scan("HDL-32", j, seed=synth.BASE_SEED + 100 + b) for j in range(n)] for b in range(B)]
    maxn = max(s.shape[0] for tr in scans for s in tr)
    dev = [[torch.from_numpy(scans[b][j]).cuda() for b in range(B)] for j in range(n)]
    ptrs = np.array([[dev[j][b].data_ptr() for b in range(B)] for j in range(n)], np.uint64)
    counts = np.array([[scans[b][j].shape[0] for b in range(B)] for j in range(n)])
    ctx = {s: pkg.Aloam(n_scans=32, max_points=maxn + 1024, max_map_points=400000, max_batch=B, max_ring_points=2304, mapping_skip_frame=k)
           for s in ("off", "on")}
    sink = torch.zeros((K * B * maxn + 16, 4), dtype=torch.float32, device="cuda")
    ctx["on"].set_registered_sink(sink)
    ms = {"off": [], "on": []}
    poses = {"off": [], "on": []}
    spans = [(0, 1 + W)] + [(1 + W + r * K, 1 + W + (r + 1) * K) for r in range(R)]
    for i, (a, b) in enumerate(spans):
        for s in (("off", "on") if i % 2 == 0 else ("on", "off")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, mp = ctx[s].scan_stream_mapped_batch(ptrs[a:b], counts[a:b], True)
            dt = time.perf_counter() - t0
            poses[s].append(mp)
            if i > 0:
                ms[s].append(1e3 * dt / (b - a))
    same = all(np.array_equal(x, y) for x, y in zip(poses["off"], poses["on"]))
    for c in ctx.values():
        c.close()
    print(json.dumps({"bench": "registered_sink", "sensor": "HDL-32", "mapping_skip_frame": k, "lanes": B, "steps": K, "repeats": R,
                      "ms_per_step_no_sink": [round(v, 3) for v in ms["off"]], "ms_per_step_device_sink": [round(v, 3) for v in ms["on"]],
                      "median_no_sink": round(float(np.median(ms["off"])), 3), "median_device_sink": round(float(np.median(ms["on"])), 3),
                      "map_poses_identical": bool(same), "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)


def bench_export(torch, gpu, R):
    rng = np.random.default_rng(7)
    npts = 65536
    ctx = pkg.Aloam(n_scans=16, max_points=npts, max_map_points=400000, line_res=0.05, plane_res=0.05)
    ctx.mapper_reset()
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    while ctx.mapper_export_size(pkg.EXPORT_MAP) < 1_000_000:   # thin frames (no corner points): the pose stays the odometry pose
        surf = np.zeros((npts, 4), np.float32)
        surf[:, :3] = rng.uniform([-120, -120, -20], [120, 120, 20], size=(npts, 3))
        surf[:, 3] = rng.uniform(0, 16, npts)
        ctx.mapper_step(empty, surf, ident, np.zeros(3))
    n = ctx.mapper_export_size(pkg.EXPORT_MAP)
    outs = {"device": torch.empty((n, 4), dtype=torch.float32, device="cuda"),
            "pinned_host": torch.empty((n, 4), dtype=torch.float32).pin_memory(), "pageable_host": None}
    ref = ctx.mapper_export(pkg.EXPORT_MAP)
    res = {}
    for name, out in outs.items():
        us = []
        for _ in range(max(R, 1) * 5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = ctx.mapper_export(pkg.EXPORT_MAP, out=out)
            us.append(1e6 * (time.perf_counter() - t0))
        host = got.cpu().numpy() if hasattr(got, "cpu") else got
        assert np.array_equal(host.view(np.int32), ref.view(np.int32)), name
        med = float(np.median(us))
        res[name] = {"median_us": round(med, 1), "GB_per_s": round(16.0 * n / med / 1e3, 1)}
    ctx.close()
    print(json.dumps({"bench": "mapper_export", "what": "map", "points": int(n), **res, "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    gpu = gpu_info()
    for k in (1, 3):
        for B in (1, 16):
            bench_sink(torch, gpu, k, B, a.steps, a.warmup, 2 * a.repeats)
    bench_export(torch, gpu, a.repeats)


if __name__ == "__main__":
    main()
