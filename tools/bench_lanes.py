#!/usr/bin/env python
"""Fleet replay of trajectories of different lengths: continuous refill (aloam_scan_stream_lanes) against lockstep groups
(aloam_scan_stream_mapped_batch).  A seeded mix of HDL-32 32x2200 trajectories with lengths drawn uniformly from [--min-len,
--max-len] scans, B lanes, extraction + odometry + scan-to-map, device-resident scans, one context for both schedules:
  refill    a lane STARTs the next trajectory of the arrival order at the step after its previous one ended, fed to
            aloam_scan_stream_lanes in calls of --chunk steps;
  lockstep  groups of B trajectories in arrival order, each run for the length of its longest trajectory; a finished lane is
            fed repeats of its last scan and those results are discarded; odometry and cube stores reset between groups.
The two alternate --repeats times after one untimed pass of each.  Prints one JSON line per schedule (useful map-refined
scans/s, median and range over the repeats, lane-steps issued) and one summary line (ratio, whether every trajectory's poses
are bit-identical under both schedules, the GPU name and power limit read in the same run).
usage: python tools/bench_lanes.py [--trajectories 32] [--batch 16] [--min-len 20] [--max-len 60] [--repeats 5]"""
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


def refill_plan(lengths, B):
    """ops / trajectory / scan index per (step, lane), -1 where idle"""
    free_at = [0] * B
    placed = []
    for t, n in enumerate(lengths):
        lane = min(range(B), key=lambda b: (free_at[b], b))
        placed.append((t, lane, free_at[lane]))
        free_at[lane] += n
    steps = max(free_at)
    ops = np.zeros((steps, B), np.int32)
    who = np.full((steps, B), -1)
    idx = np.full((steps, B), -1)
    for t, lane, s in placed:
        for i in range(lengths[t]):
            ops[s + i, lane] = pkg.LANE_START if i == 0 else pkg.LANE_SCAN
            who[s + i, lane], idx[s + i, lane] = t, i
    return ops, who, idx


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--trajectories", type=int, default=32)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--min-len", type=int, default=20)
    ap.add_argument("--max-len", type=int, default=60)
    ap.add_argument("--chunk", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    B = a.batch
    lengths = [int(x) for x in np.random.default_rng(a.seed).integers(a.min_len, a.max_len + 1, a.trajectories)]
    scans = [[synth.scan("HDL-32", k, seed=synth.BASE_SEED + 500 + t) for k in range(n)] for t, n in enumerate(lengths)]
    maxn = max(s.shape[0] for tr in scans for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in scans]
    ptr = [[d.data_ptr() for d in tr] for tr in dev]
    cnt = [[s.shape[0] for s in tr] for tr in scans]
    name, power = gpu_info()
    useful = sum(lengths)
    ctx = pkg.Aloam(n_scans=32, max_points=maxn + 1024, max_map_points=600000, max_batch=B, max_ring_points=2304)

    ops, who, idx = refill_plan(lengths, B)
    R_ptrs = np.zeros(who.shape, np.uint64)
    R_counts = np.zeros(who.shape, np.int64)
    for (k, b), t in np.ndenumerate(who):
        if t >= 0:
            R_ptrs[k, b], R_counts[k, b] = ptr[t][idx[k, b]], cnt[t][idx[k, b]]

    def run_refill():
        """seconds, {trajectory: (odom, map) rows}"""
        ctx.reset_odometry()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs = [ctx.scan_stream_lanes(R_ptrs[s:s + a.chunk], R_counts[s:s + a.chunk], ops[s:s + a.chunk], True)
                for s in range(0, ops.shape[0], a.chunk)]
        torch.cuda.synchronize()
        secs = time.perf_counter() - t0
        odom, mapped = np.concatenate([o for o, _ in outs]), np.concatenate([m for _, m in outs])
        res = {}
        for t in range(len(lengths)):
            ks, bs = np.nonzero(who == t)
            res[t] = (odom[ks, bs], mapped[ks, bs])
        return secs, res

    groups = [list(range(g, min(g + B, len(lengths)))) for g in range(0, len(lengths), B)]

    def run_lockstep():
        secs, res = 0.0, {}
        for g in groups:
            ctx.reset_odometry(); ctx.mapper_reset()   # (between groups: not timed)
            steps = max(lengths[t] for t in g)
            p = np.array([[ptr[t][min(k, lengths[t] - 1)] for t in g] for k in range(steps)], np.uint64)
            c = np.array([[cnt[t][min(k, lengths[t] - 1)] for t in g] for k in range(steps)])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            odom, mapped = ctx.scan_stream_mapped_batch(p, c, True)
            torch.cuda.synchronize()
            secs += time.perf_counter() - t0
            for j, t in enumerate(g):
                res[t] = (odom[:lengths[t], j], mapped[:lengths[t], j])
        ctx.reset_odometry()
        return secs, res

    run_refill(); run_lockstep()   # untimed: every shape warmed
    times = {"refill": [], "lockstep": []}
    results = {}
    for _ in range(a.repeats):
        for sched, fn in (("refill", run_refill), ("lockstep", run_lockstep)):
            s, results[sched] = fn()
            times[sched].append(s)
    same = all(np.array_equal(results["refill"][t][i], results["lockstep"][t][i]) for t in range(len(lengths)) for i in (0, 1))
    lane_steps = {"refill": int((ops != pkg.LANE_IDLE).sum()), "lockstep": sum(B * max(lengths[t] for t in g) for g in groups)}
    workload = ("HDL-32 synthetic 32x2200, %d trajectories of %d..%d scans (seed %d, %d scans in all), %d lanes, extraction + odometry + "
                "scan-to-map, device-resident" % (len(lengths), min(lengths), max(lengths), a.seed, useful, B))
    rate = {}
    for sched in ("refill", "lockstep"):
        med = float(np.median(times[sched]))
        rate[sched] = useful / med
        print(json.dumps({"metric": "useful map-refined scans/s", "schedule": sched, "value": rate[sched], "unit": "scans/s",
                          "range": [useful / max(times[sched]), useful / min(times[sched])], "seconds_median": med,
                          "lane_steps_issued": lane_steps[sched], "useful_lane_steps": useful, "repeats": a.repeats,
                          "gpu": name, "power_limit": power, "workload": workload}), flush=True)
    print(json.dumps({"refill_over_lockstep": rate["refill"] / rate["lockstep"], "poses_identical_under_both_schedules": bool(same),
                      "lengths": lengths, "gpu": name, "power_limit": power}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
