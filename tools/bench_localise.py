#!/usr/bin/env python
"""Mapping lanes against localising lanes on the map those mapping lanes produced.  HDL-32 32 x 2200 scans, device-resident,
B lanes replaying one seeded trajectory, cfg.mapping_skip_frame = k.  One process, one context per (B, k); the two arms alternate
--repeats times after one untimed pass of each:
  map       every lane STARTs a mapping trajectory and runs --steps scans (aloam_scan_stream_lanes);
  localise  every lane is armed with the identity (the vehicle starts where the map's did) and runs the same scans against the
            prior map loaded from the snapshot of a mapping lane.
Per (B, k) and arm one JSON line: median and range of ms per step (host clock around the synchronous call), launches per step,
device memory taken by the lanes (cudaMemGetInfo before / after their first call).  Then the load time of the prior map from
device and from pinned memory.  (Per-kernel times of k_map_knn5_prior against K0 + k_map_knn5 are not taken here: the profile
hooks time the first 192 launches of a call on the main stream, and the frames run on the mapper stream.)  The GPU's name and power limit are read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_localise.py [--steps 60] [--repeats 3] [--batches 1,16] [--skips 1,3]"""
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


def parse(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--batches", default="1,16")
    ap.add_argument("--skips", default="1,3")
    ap.add_argument("--n-az", type=int, default=2200)
    a = ap.parse_args(argv)
    a.batches = [int(x) for x in a.batches.split(",")]
    a.skips = [int(x) for x in a.skips.split(",")]
    if a.steps < 2 or a.repeats < 1 or min(a.batches) < 1 or max(a.batches) > 16 or min(a.skips) < 1:
        ap.error("steps >= 2, repeats >= 1, batches in 1..16, skips >= 1")
    return a


def main():
    a = parse()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_localise needs a CUDA device")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    scans = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 900, n_az=a.n_az) for k in range(a.steps)]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    maxn = max(s.shape[0] for s in scans) + 1024
    ident = (np.array([0, 0, 0, 1.0]), np.zeros(3))

    def free():
        torch.cuda.synchronize()
        return torch.cuda.mem_get_info()[0]

    def arrays(B):
        ptrs = np.array([[d.data_ptr()] * B for d in dev], np.uint64)
        counts = np.array([[s.shape[0]] * B for s in scans], np.int64)
        ops = np.full((a.steps, B), pkg.LANE_SCAN, np.int32)
        ops[0] = pkg.LANE_START
        return ptrs, counts, ops

    blob = None
    for k in a.skips:
        for B in a.batches:
            ctx = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_batch=B, max_ring_points=2304, mapping_skip_frame=k)
            ptrs, counts, ops = arrays(B)

            def run(arm):
                ctx.reset_odometry()
                if arm == "localise":
                    for l in range(B):
                        ctx.lane_localise(l, *ident)
                l0, t0 = ctx.launch_count(), time.perf_counter()
                ctx.scan_stream_lanes(ptrs, counts, ops, True)
                return (time.perf_counter() - t0) * 1e3 / a.steps, (ctx.launch_count() - l0) / a.steps

            mem = {}
            f0 = free(); run("map"); mem["map"] = f0 - free()
            blob = ctx.lane_save(0, torch.empty(ctx.lane_save(0).size + 64, dtype=torch.uint8, device="cuda"))
            ctx.prior_map_load(blob)
            f0 = free(); run("localise"); mem["localise"] = f0 - free()   # (the mapping lanes' stores stay: the delta is the locators')
            ms = {"map": [], "localise": []}
            launches = {}
            for _ in range(a.repeats):
                for arm in ("map", "localise"):
                    t, launches[arm] = run(arm)
                    ms[arm].append(t)
            for arm in ("map", "localise"):
                print(json.dumps({"arm": arm, "B": B, "skip": k, "steps": a.steps, "ms_per_step_median": round(float(np.median(ms[arm])), 4),
                                  "ms_per_step_range": [round(min(ms[arm]), 4), round(max(ms[arm]), 4)], "launches_per_step": launches[arm],
                                  "lanes_device_bytes": int(mem[arm]), "map_points": int(pkg.snapshot_info(
                                      blob.cpu().numpy())["map_points"]), "gpu": name, "power_limit": power}))
            ctx.close()
    # load time of the last prior map, from device and from pinned memory
    ctx = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_batch=1, max_ring_points=2304, mapping_skip_frame=a.skips[-1])
    pinned = blob.cpu().pin_memory()
    ctx.prior_map_load(blob)
    load = {}
    for what, b in (("device", blob), ("pinned", pinned)):
        ts = []
        for _ in range(5):
            t0 = time.perf_counter(); ctx.prior_map_load(b); ts.append((time.perf_counter() - t0) * 1e3)
        load[what] = round(float(np.median(ts)), 3)
    print(json.dumps({"prior_map_load_ms": load, "map_points": int(pkg.snapshot_info(pinned.numpy())["map_points"]), "bytes": int(blob.numel()),
                      "gpu": name, "power_limit": power}))
    ctx.close()


if __name__ == "__main__":
    main()
