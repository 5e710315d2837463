#!/usr/bin/env python
"""The cost of recovering localising lanes inside the stream (aloam_set_recovery).  The localising lanes of tools/bench_localise.py:
HDL-32 32 x 2200 scans of seed BASE_SEED + 900, device-resident, B lanes localising against the ~76 k-point prior map of a lane
that mapped the same scans, rows scored at max_score_points 256, inlier_sq 0.25.  Per B and candidate grid, four arms alternate
--repeats times after one untimed pass of each:
  score    rows and scores only (aloam_set_map_rows), recovery off;
  never    recovery on with trigger_frac 0: no row triggers, the four launches per localising frame run and leave at once;
  one      lane 0 armed 45 degrees and 10 m off its true pose (the other lanes at it: beyond the reach of either grid), trigger_frac
           0.5, accept_frac 1: lane 0's rows trigger on every frame and never adopt;
  all      trigger_frac 1, accept_frac 1: every row that misses a point triggers.
Candidate grids: pose_grid(identity, 0, half, step, 72 headings) at (half, step) = (1, 0.5) -> 1 800 and (4, 0.5) -> 20 808
deltas.  One JSON line per (B, grid, arm): median and range of ms per step (host clock around the synchronous call), launches per
step, and the rows that triggered and adopted in the last timed call.  The GPU's name and power limit are read in the same run.
Needs a GPU: without one it fails.
usage: python tools/bench_recovery.py [--steps 60] [--repeats 3] [--batches 1,16]"""
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

ISQ, PTS = 0.25, 256
GRIDS = ((1.0, 0.5), (4.0, 0.5))


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")[:2]]
    return name, power


def mis_armed():
    """the identity turned by 45 degrees about z and moved 10 m sideways"""
    h = np.radians(45.0) / 2
    return np.array([0, 0, np.sin(h), np.cos(h)]), np.array([0.0, 10.0, 0.0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--n-az", type=int, default=2200)
    a = ap.parse_args()
    batches = [int(x) for x in a.batches.split(",")]
    if a.steps < 2 or a.repeats < 1 or min(batches) < 1 or max(batches) > 16:
        ap.error("steps >= 2, repeats >= 1, batches in 1..16")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_recovery needs a CUDA device")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    scans = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 900, n_az=a.n_az) for k in range(a.steps)]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    maxn = max(s.shape[0] for s in scans) + 1024
    ident = (np.array([0, 0, 0, 1.0]), np.zeros(3))
    yaws = np.arange(72) * (2 * np.pi / 72)
    # the prior map: the snapshot of a lane that mapped the scans
    ctx = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_batch=1, max_ring_points=2304)
    ptrs = np.array([[d.data_ptr()] for d in dev], np.uint64)
    counts = np.array([[s.shape[0]] for s in scans], np.int64)
    ops = np.full((a.steps, 1), pkg.LANE_SCAN, np.int32)
    ops[0] = pkg.LANE_START
    ctx.scan_stream_lanes(ptrs, counts, ops, True)
    blob = ctx.lane_save(0)
    ctx.close()
    for B in batches:
        ptrs = np.array([[d.data_ptr()] * B for d in dev], np.uint64)
        counts = np.array([[s.shape[0]] * B for s in scans], np.int64)
        ops = np.full((a.steps, B), pkg.LANE_SCAN, np.int32)
        ops[0] = pkg.LANE_START
        ctx = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_batch=B, max_ring_points=2304)
        ctx.prior_map_load(blob)
        for half, step in GRIDS:
            deltas = pkg.pose_grid(ident[0], ident[1], half, step, yaws)
            arms = {"score": None, "never": (0.0, 1.0), "one": (0.5, 1.0), "all": (1.0, 1.0)}

            def run(arm):
                ctx.set_map_rows(True, ISQ, PTS)
                if arms[arm] is None:
                    ctx.set_recovery(False)
                else:
                    ctx.set_recovery(True, arms[arm][0], arms[arm][1], deltas)
                ctx.reset_odometry()
                for l in range(B):
                    ctx.lane_localise(l, *(mis_armed() if arm == "one" and l == 0 else ident))
                l0, t0 = ctx.launch_count(), time.perf_counter()
                ctx.scan_stream_lanes(ptrs, counts, ops, True)
                return (time.perf_counter() - t0) * 1e3 / a.steps, (ctx.launch_count() - l0) / a.steps

            for arm in arms:
                run(arm)
            ms = {arm: [] for arm in arms}
            launches, trig = {}, {}
            for _ in range(a.repeats):
                for arm in arms:
                    t, launches[arm] = run(arm)
                    ms[arm].append(t)
                    r = ctx.recovery_rows(a.steps * B)
                    trig[arm] = (int(r["triggered"].sum()), int(r["adopted"].sum()))
            for arm in arms:
                print(json.dumps({"arm": arm, "B": B, "n_delta": len(deltas), "steps": a.steps, "ms_per_step_median": round(float(np.median(ms[arm])), 4),
                                  "ms_per_step_range": [round(min(ms[arm]), 4), round(max(ms[arm]), 4)], "launches_per_step": launches[arm],
                                  "rows_triggered": trig[arm][0], "rows_adopted": trig[arm][1], "gpu": name, "power_limit": power}), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
