#!/usr/bin/env python
"""Cost of taking each return's ring from the sensor driver (cfg.ring_source = ALOAM_RING_FIELD) instead of the elevation formula.
  (a) HDL-64 64x2000 scans with float 3 set to the formula's ring, one context per ring source, the two alternated --repeats
      times after one untimed pass each: k_classify time per launch (aloam_profile_*, CUDA events, over one aloam_scan_to_pose
      per scan) and scans/s of aloam_scan_stream (device-resident scans, profiling off).  The two sources must give
      bit-identical poses and features; the tool fails if they do not.
  (b) OS64 (tests: synth.RING_SENSORS, 64 x 1024) field-mode streams at B = 1 and B = 16 lanes, unmapped
      (aloam_scan_stream_batch) and mapped (aloam_scan_stream_mapped_batch): scans/s, median over the repeats.  Lane b runs the
      trajectory from scan b.
Prints one JSON line per measurement and a last line with the GPU name and power limit read in the same run.
usage: python tools/bench_ring_source.py [--scans 40] [--repeats 5]"""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("a-loam_b200")
synth = importlib.import_module("a-loam_b200.synth")
from ring_edge_cases import ring_ids  # noqa: E402  (the formula's ring of a return, numpy)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception:
        return "unknown", "unknown"


def stacked(raws):
    import torch
    n = max(len(r) for r in raws)
    dev = torch.zeros((len(raws), n, 4), dtype=torch.float32)
    for i, r in enumerate(raws):
        dev[i, :len(r)] = torch.from_numpy(r)
    return dev.cuda(), [len(r) for r in raws]


def part_a(args):
    raws = []
    for k in range(args.scans):
        r = synth.scan("HDL-64", k)
        r[:, 3] = ring_ids(r, 64)
        raws.append(r)
    dev, counts = stacked(raws)
    ptrs = [dev[i].data_ptr() for i in range(len(raws))]
    mp = max(counts) + 1024
    ctx = {rs: pkg.Aloam(n_scans=64, max_points=mp, ring_source=rs) for rs in (pkg.RING_ELEVATION, pkg.RING_FIELD)}
    for rs in ctx:   # untimed pass
        ctx[rs].reset_odometry()
        ctx[rs].scan_stream(ptrs, counts, True)
    f = [ctx[rs].extract_features(raws[0]) for rs in ctx]
    same = all(np.array_equal(f[0][n].view(np.uint32), f[1][n].view(np.uint32)) for n in f[0])
    rate = {rs: [] for rs in ctx}
    classify = {rs: [] for rs in ctx}
    poses = {}
    for _ in range(args.repeats):
        for rs, c in ctx.items():
            c.reset_odometry()
            t0 = time.perf_counter()
            p, _ = c.scan_stream(ptrs, counts, True)
            rate[rs].append(len(raws) / (time.perf_counter() - t0))
            if rs in poses:
                same &= np.array_equal(poses[rs], p)
            poses[rs] = p
            c.reset_odometry()
            c.profile_enable(True)
            for r in raws:
                c.scan_to_pose(r)
            prof = c.profile_read()
            c.profile_enable(False)
            ms, n = prof["k_classify"]
            classify[rs].append(1000.0 * ms / n)
    same &= np.array_equal(poses[pkg.RING_ELEVATION], poses[pkg.RING_FIELD])
    for rs, c in ctx.items():
        name = "elevation" if rs == pkg.RING_ELEVATION else "field"
        print(json.dumps({"part": "a", "sensor": "HDL-64", "ring_source": name, "scans": len(raws),
                          "k_classify_us_median": round(float(np.median(classify[rs])), 2),
                          "k_classify_us_range": [round(min(classify[rs]), 2), round(max(classify[rs]), 2)],
                          "scans_per_s_median": round(float(np.median(rate[rs])), 1),
                          "scans_per_s_range": [round(min(rate[rs]), 1), round(max(rate[rs]), 1)]}))
        c.close()
    print(json.dumps({"part": "a", "bit_identical": bool(same)}))
    return same


def part_b(args):
    B = 16
    raws = [synth.scan_rings("OS64", k) for k in range(args.scans + B)]
    dev, counts = stacked(raws)
    mp = max(counts) + 1024
    c = pkg.Aloam(n_scans=64, max_points=mp, ring_source=pkg.RING_FIELD, minimum_range=synth.RING_RANGES[0],
                  line_res=synth.RING_RANGES[1], plane_res=synth.RING_RANGES[2], max_batch=B, max_map_points=400000)
    for b in (1, B):
        ptrs = np.array([[dev[k + j].data_ptr() for j in range(b)] for k in range(args.scans)], np.uint64)
        cnt = np.array([[counts[k + j] for j in range(b)] for k in range(args.scans)], np.int64)
        for mapped in (False, True):
            run = c.scan_stream_mapped_batch if mapped else c.scan_stream_batch
            rates = []
            for rep in range(args.repeats + 1):
                c.reset_odometry()
                if mapped:
                    c.mapper_reset()
                t0 = time.perf_counter()
                run(ptrs, cnt, True)
                dt = time.perf_counter() - t0
                if rep:   # the first pass is untimed
                    rates.append(args.scans * b / dt)
            print(json.dumps({"part": "b", "sensor": "OS64", "batch": b, "mapped": mapped, "scans": args.scans,
                              "scans_per_s_median": round(float(np.median(rates)), 1),
                              "scans_per_s_range": [round(min(rates), 1), round(max(rates), 1)]}))
    c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_ring_source needs a CUDA device")
    same = part_a(args)
    part_b(args)
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": power}))
    if not same:
        raise SystemExit("the two ring sources gave different results")


if __name__ == "__main__":
    main()
