#!/usr/bin/env python
"""Cost of per-row records (aloam_set_map_rows) on localising lanes, with tools/bench_localise.py's setup: HDL-32 32 x 2200 scans,
device-resident, B lanes replaying one seeded trajectory, cfg.mapping_skip_frame = k, every lane armed with the identity against the
prior map of a mapping lane that ran the same scans.  One process, one context per (B, k); after one untimed pass of each, four arms
alternate --repeats times:
  off      recording off;
  rows     rows only (k_map_rows after every frame);
  s256     rows and scores at 256 scoring points per type (k_inlier_score after every localising frame);
  s1024    rows and scores at 1 024 points per type.
inlier_sq = 0.25.  Per (B, k) and arm one JSON line: median and range of ms per step (host clock around the synchronous call) and
launches per step.  The GPU's name and power limit are read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_map_rows.py [--steps 60] [--repeats 3] [--batches 1,16] [--skips 1,3]"""
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_localise import gpu_info, parse   # noqa: E402

ARMS = (("off", 0, 0), ("rows", 1, 0), ("s256", 1, 256), ("s1024", 1, 1024))


def main():
    a = parse()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_map_rows needs a CUDA device")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    scans = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 900, n_az=a.n_az) for k in range(a.steps)]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    maxn = max(s.shape[0] for s in scans) + 1024
    ident = (np.array([0, 0, 0, 1.0]), np.zeros(3))
    for k in a.skips:
        for B in a.batches:
            ctx = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_batch=B, max_ring_points=2304, mapping_skip_frame=k)
            ptrs = np.array([[d.data_ptr()] * B for d in dev], np.uint64)
            counts = np.array([[s.shape[0]] * B for s in scans], np.int64)
            ops = np.full((a.steps, B), pkg.LANE_SCAN, np.int32)
            ops[0] = pkg.LANE_START
            ctx.scan_stream_lanes(ptrs, counts, ops, True)   # one mapping lane's store becomes the prior map
            ctx.prior_map_load(ctx.lane_save(0))

            def run(on, pts):
                ctx.set_map_rows(on, 0.25, pts)
                ctx.reset_odometry()
                for l in range(B):
                    ctx.lane_localise(l, *ident)
                l0, t0 = ctx.launch_count(), time.perf_counter()
                ctx.scan_stream_lanes(ptrs, counts, ops, True)
                t = (time.perf_counter() - t0) * 1e3 / a.steps
                if on:
                    ctx.map_rows(ops.size)
                return t, (ctx.launch_count() - l0) / a.steps

            for _, on, pts in ARMS:
                run(on, pts)
            ms = {arm: [] for arm, _, _ in ARMS}
            launches = {}
            for _ in range(a.repeats):
                for arm, on, pts in ARMS:
                    t, launches[arm] = run(on, pts)
                    ms[arm].append(t)
            for arm, _, pts in ARMS:
                print(json.dumps({"arm": arm, "B": B, "skip": k, "steps": a.steps, "max_score_points": pts,
                                  "ms_per_step_median": round(float(np.median(ms[arm])), 4),
                                  "ms_per_step_range": [round(min(ms[arm]), 4), round(max(ms[arm]), 4)], "launches_per_step": launches[arm],
                                  "gpu": name, "power_limit": power}), flush=True)
            ctx.close()


if __name__ == "__main__":
    main()
