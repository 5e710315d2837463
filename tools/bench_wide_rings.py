#!/usr/bin/env python
"""Cost of 128-beam lidars (contexts of aloam_create_wide) next to 64-beam ones.
  (a) --parent DIR: bench.py's JSON record from this tree and from DIR (a built checkout of the parent commit), run ABBA twice in
      one call (this, parent, parent, this, ...).  Reports each run's headline and e2e scans/s; the difference of the two trees
      is to be read against the spread of each tree's own runs.
  (b) OS128 and OS64 (synth.WIDE_RING_SENSORS / RING_SENSORS) at 1024 and 2048 azimuth steps: scans/s of aloam_scan_stream_batch
      and aloam_scan_stream_mapped_batch (device-resident scans) at B = 1 and B = 16, median over the repeats after one untimed
      pass; then, B = 1, per-kernel times from aloam_profile_read over one aloam_scan_to_pose per scan.
  (c) OS128 at 2048 azimuth steps, max_ring_points 2048 and 4096: B = 1 stream scans/s and k_ring_features time per launch.
Prints one JSON line per measurement and a last line with the GPU name and power limit read in the same run.
usage: python tools/bench_wide_rings.py [--scans 20] [--repeats 3] [--parent DIR] [--steps 100] [--warmup 10]"""
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

KERNELS = ("k_classify", "k_ring_scan", "k_scatter", "k_ring_features", "k_compact", "k_rab_build(3 launches)", "k_odom_assoc", "k_lm_solve")


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception:
        return "unknown", "unknown"


def part_a(args):
    trees = [("this", ROOT), ("parent", os.path.abspath(args.parent))]
    order = [0, 1, 1, 0, 0, 1, 1, 0]   # ABBA twice
    for i in order:
        name, tree = trees[i]
        out = subprocess.run([sys.executable, "bench.py", "--gpus", "1", "--steps", str(args.steps), "--warmup", str(args.warmup)] + args.bench_args.split(),
                             cwd=tree, capture_output=True, text=True)
        rec = None
        for line in out.stdout.splitlines():
            if line.startswith("{"):
                rec = json.loads(line)
        if rec is None:
            print(json.dumps({"part": "a", "tree": name, "error": out.stderr[-2000:]}))
            continue
        print(json.dumps({"part": "a", "tree": name, "value": rec.get("value"), "e2e": rec.get("e2e"),
                          "batch": (rec.get("batch") or {}).get("value") if isinstance(rec.get("batch"), dict) else rec.get("batch")}))


def stacked(raws):
    import torch
    n = max(len(r) for r in raws)
    dev = torch.zeros((len(raws), n, 4), dtype=torch.float32)
    for i, r in enumerate(raws):
        dev[i, :len(r)] = torch.from_numpy(r)
    return dev.cuda(), [len(r) for r in raws]


def context(sensor, mp, batch, max_ring_points=4096):
    ns = len((synth.WIDE_RING_SENSORS.get(sensor) or synth.RING_SENSORS[sensor])[0])
    return pkg.Aloam(n_scans=ns, max_points=mp, ring_source=pkg.RING_FIELD, minimum_range=synth.RING_RANGES[0],
                     line_res=synth.RING_RANGES[1], plane_res=synth.RING_RANGES[2], max_batch=batch, max_map_points=400000,
                     max_ring_points=max_ring_points, wide=ns > 64)


def stream_rates(c, dev, counts, scans, b, mapped, repeats):
    ptrs = np.array([[dev[k + j].data_ptr() for j in range(b)] for k in range(scans)], np.uint64)
    cnt = np.array([[counts[k + j] for j in range(b)] for k in range(scans)], np.int64)
    run = c.scan_stream_mapped_batch if mapped else c.scan_stream_batch
    rates = []
    for rep in range(repeats + 1):
        c.reset_odometry()
        if mapped:
            c.mapper_reset()
        t0 = time.perf_counter()
        run(ptrs, cnt, True)   # returns after the device has finished (the poses are read back)
        dt = time.perf_counter() - t0
        if rep:   # the first pass is untimed
            rates.append(scans * b / dt)
    return rates


def profile(c, raws):
    c.reset_odometry()
    c.profile_enable(True)
    for r in raws:
        c.scan_to_pose(r)
    prof = c.profile_read()
    c.profile_enable(False)
    return {k: round(1000.0 * prof[k][0] / prof[k][1], 2) for k in KERNELS if k in prof and prof[k][1]}


def part_b(args):
    B = 16
    for n_az in (1024, 2048):
        for sensor in ("OS64", "OS128"):
            raws = [synth.scan_rings(sensor, k, n_az=n_az) for k in range(args.scans + B)]
            dev, counts = stacked(raws)
            c = context(sensor, max(counts) + 1024, B)
            for b in (1, B):
                for mapped in (False, True):
                    r = stream_rates(c, dev, counts, args.scans, b, mapped, args.repeats)
                    print(json.dumps({"part": "b", "sensor": sensor, "n_az": n_az, "batch": b, "mapped": mapped, "scans": args.scans,
                                      "scans_per_s_median": round(float(np.median(r)), 1), "scans_per_s_range": [round(min(r), 1), round(max(r), 1)]}))
            print(json.dumps({"part": "b", "sensor": sensor, "n_az": n_az, "kernel_us_per_launch": profile(c, raws[:args.scans])}))
            c.close()
            del dev


def part_c(args):
    raws = [synth.scan_rings("OS128", k, n_az=2048) for k in range(args.scans)]
    dev, counts = stacked(raws)
    for mrp in (2048, 4096):
        c = context("OS128", max(counts) + 1024, 1, mrp)
        r = stream_rates(c, dev, counts, args.scans, 1, False, args.repeats)
        prof = profile(c, raws)
        print(json.dumps({"part": "c", "sensor": "OS128", "n_az": 2048, "max_ring_points": mrp, "scans_per_s_median": round(float(np.median(r)), 1),
                          "scans_per_s_range": [round(min(r), 1), round(max(r), 1)], "k_ring_features_us": prof.get("k_ring_features")}))
        c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built checkout of the parent commit: runs part (a)")
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--parts", default="abc")
    ap.add_argument("--bench-args", default="", help="further bench.py options of part (a), e.g. --no-cpu-baseline")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_wide_rings needs a CUDA device")
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": power}))
    if "a" in args.parts and args.parent:
        part_a(args)
    if "b" in args.parts:
        part_b(args)
    if "c" in args.parts:
        part_c(args)
    name, power = gpu_info()
    print(json.dumps({"gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
