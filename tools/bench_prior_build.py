#!/usr/bin/env python
"""Building a prior map from two map-frame clouds (aloam_prior_map_build), and localising against a large built map.
  build     synth.build_map maps of 1 M and 8 M points (HDL-64 features at their true poses, tiled), from device memory and from
            pinned host memory: median and range of --repeats calls after one untimed call (host clock around the synchronous call).
            The 1 M map is built at the HDL-64 leaves (0.4 / 0.8); the 8 M map at 0.8 / 1.0, because at 0.4 one of its corner cubes
            keeps more than 65536 points, which the build refuses.
  localise  1 and 16 lanes armed at the true pose of scan 24 localise HDL-64 scans 24 .. 24 + --steps - 1 (device-resident, not
            part of the map) against the 1 M-point built map: ms per step (host clock around aloam_scan_stream_lanes).
One JSON line with every number, the GPU's name and its power limit, read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_prior_build.py [--repeats 5] [--steps 16]"""
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


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")[:2]]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--steps", type=int, default=16)
    a = ap.parse_args()
    if a.repeats < 1 or not 2 <= a.steps <= 16:
        ap.error("repeats >= 1, steps in 2 .. 16")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_prior_build needs a CUDA device")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    fx = pkg.Aloam(n_scans=64, max_points=200000)

    def feats(raw):
        f = fx.extract_features(raw)
        return f["less_sharp"], f["less_flat"]

    maps = {n: synth.build_map(feats, n) for n in (1_000_000, 8_000_000)}
    fx.close()
    out = {"build_ms": {}, "map_points": {}, "gpu": name, "power_limit": power}
    for n, leaves in ((1_000_000, (0.4, 0.8)), (8_000_000, (0.8, 1.0))):
        ctx = pkg.Aloam(n_scans=64, max_points=200000, line_res=leaves[0], plane_res=leaves[1])
        corner, surf = maps[n]
        for what, conv in (("device", lambda x: torch.from_numpy(x).cuda()), ("pinned", lambda x: torch.from_numpy(x).pin_memory())):
            c, s = conv(corner), conv(surf)
            ctx.prior_map_build(c, s)
            ts = []
            for _ in range(a.repeats):
                t0 = time.perf_counter(); ctx.prior_map_build(c, s); ts.append((time.perf_counter() - t0) * 1e3)
            out["build_ms"]["%dM_%s" % (n // 1_000_000, what)] = {"median": round(float(np.median(ts)), 3), "range": [round(min(ts), 3), round(max(ts), 3)]}
        out["map_points"]["%dM" % (n // 1_000_000)] = ctx.mapper_export_size(pkg.EXPORT_MAP, pkg.PRIOR_MAP)
        ctx.close()
    # localising lanes against the 1 M-point built map
    scans = [synth.scan("HDL-64", k) for k in range(24, 24 + a.steps)]
    dev = [torch.from_numpy(x).cuda() for x in scans]
    maxn = max(x.shape[0] for x in scans) + 1024
    q0, t0 = synth.pose(24)
    out["localise_ms_per_step"] = {}
    for B in (1, 16):
        ctx = pkg.Aloam(n_scans=64, max_points=maxn, max_map_points=600000, max_batch=B)
        ctx.prior_map_build(*maps[1_000_000])
        ptrs = np.array([[d.data_ptr()] * B for d in dev], np.uint64)
        counts = np.array([[x.shape[0]] * B for x in scans], np.int64)
        ops = np.full((a.steps, B), pkg.LANE_SCAN, np.int32)
        ops[0] = pkg.LANE_START
        ts = []
        for r in range(a.repeats + 1):
            ctx.reset_odometry()
            for l in range(B):
                ctx.lane_localise(l, q0, t0)
            t = time.perf_counter()
            ctx.scan_stream_lanes(ptrs, counts, ops, True)
            if r:
                ts.append((time.perf_counter() - t) * 1e3 / a.steps)
        out["localise_ms_per_step"]["B%d" % B] = {"median": round(float(np.median(ts)), 3), "range": [round(min(ts), 3), round(max(ts), 3)]}
        ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
