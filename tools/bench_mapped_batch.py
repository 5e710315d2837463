#!/usr/bin/env python
"""Throughput of aloam_scan_stream_mapped_batch: HDL-32 32x2200 scans (the shape of BASELINE configs[4]), B differently seeded
trajectories through extraction, odometry and scan-to-map in one context.  Per B one JSON line: aggregate map-refined scans/s,
ms per step, launches per step, lane 0 == its solo run, host path == device path, and the GPU name and power limit read in
the same run.  At B = 1 the batch call alternates with the solo aloam_scan_stream_mapped in the same process.
--mapping-skip-frame k1,k2,...: one set of lines per k (cfg.mapping_skip_frame): every k-th scan of a trajectory is mapped, the
others get the high-frequency pose, so the rate counts map-pose rows (refined or high-frequency) per second.
--sensor HDL-64: 64x2000 scans instead (one trajectory is --batches 1).
usage: python tools/bench_mapped_batch.py [--batches 1,4,16] [--steps 20] [--warmup 3] [--repeats 3] [--mapping-skip-frame 1]
                                          [--sensor HDL-32]"""
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


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,4,16")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--mapping-skip-frame", default="1")
    ap.add_argument("--sensor", default="HDL-32", choices=["HDL-32", "HDL-64"])
    a = ap.parse_args()
    skips = [int(k) for k in a.mapping_skip_frame.split(",")]
    ns = synth.SENSORS[a.sensor][0]
    max_ring = 2304 if a.sensor == "HDL-32" else 2048
    batches = [int(b) for b in a.batches.split(",")]
    K, W = a.steps, a.warmup
    n = 1 + W + K
    Bmax = max(batches)
    scans = [[synth.scan(a.sensor, k, seed=synth.BASE_SEED + 100 + b) for k in range(n)] for b in range(Bmax)]
    maxn = max(s.shape[0] for tr in scans for s in tr)
    host = torch.zeros((n, Bmax, maxn, 4), dtype=torch.float32).pin_memory()
    counts = np.zeros((n, Bmax), np.int32)
    for b in range(Bmax):
        for k in range(n):
            s = scans[b][k]; host[k, b, :s.shape[0]] = torch.from_numpy(s); counts[k, b] = s.shape[0]
    dev = host.to("cuda")
    name, power = gpu_info()

    def make(B, skip):
        return pkg.Aloam(n_scans=ns, max_points=maxn + 1024, max_map_points=600000, max_batch=B, max_ring_points=max_ring,
                         mapping_skip_frame=skip)

    def run(ctx, B, base, solo=False):
        """(seconds of the K timed scans, odometry poses, map poses, launches) after a fresh start and W + 1 untimed scans"""
        ctx.reset_odometry(); ctx.mapper_reset()
        ptrs = np.array([[base[k, b].data_ptr() for b in range(B)] for k in range(n)], np.uint64)
        dr = base is dev
        call = (lambda p, c: tuple(x[:, None] for x in ctx.scan_stream_mapped(p[:, 0], c[:, 0], dr))) if solo else \
            (lambda p, c: ctx.scan_stream_mapped_batch(p, c, dr))
        o0, m0 = call(ptrs[:1 + W], counts[:1 + W, :B])
        torch.cuda.synchronize()
        l0 = ctx.launch_count()
        t0 = time.perf_counter()
        o1, m1 = call(ptrs[1 + W:], counts[1 + W:, :B])
        torch.cuda.synchronize()
        secs = time.perf_counter() - t0
        return secs, np.concatenate([o0, o1]), np.concatenate([m0, m1]), ctx.launch_count() - l0

    for skip in skips:
        solo_ctx = make(1, skip)
        ctxs = {B: make(B, skip) for B in batches}
        for B, ctx in ctxs.items():   # every shape warmed (lanes created, buffers touched) before anything is timed
            run(ctx, B, dev)
        run(solo_ctx, 1, dev, solo=True)
        times = {B: [] for B in batches}
        solo_times = []
        res = {}
        for _ in range(a.repeats):
            for B, ctx in ctxs.items():
                secs, odom, mapped, launches = run(ctx, B, dev)
                times[B].append(secs)
                res[B] = (odom, mapped, launches)
                if B == 1:   # the solo call, alternating with the batch of one
                    s, so, sm, _ = run(solo_ctx, 1, dev, solo=True)
                    solo_times.append(s)
        _, solo_odom, solo_mapped, _ = run(solo_ctx, 1, dev, solo=True)
        for B, ctx in ctxs.items():
            odom, mapped, launches = res[B]
            _, odom_h, mapped_h, _ = run(ctx, B, host)
            med = float(np.median(times[B]))
            rec = {"metric": "map-refined scans/s" if skip == 1 else "map-pose scans/s", "batch": B, "mapping_skip_frame": skip, "value": B * K / med, "unit": "scans/s", "steps": K, "warmup": W,
                   "ms_per_step": 1e3 * med / K, "ms_per_step_range": [1e3 * min(times[B]) / K, 1e3 * max(times[B]) / K],
                   "launches_per_step": launches / K,
                   "lane0_equals_solo": bool(np.array_equal(odom[:, 0], solo_odom[:, 0]) and np.array_equal(mapped[:, 0], solo_mapped[:, 0])),
                   "host_equals_device_path": bool(np.array_equal(odom, odom_h) and np.array_equal(mapped, mapped_h)),
                   "gpu": name, "power_limit": power,
                   "workload": "%s synthetic %dx%d, %d differently seeded trajectories, aloam_scan_stream_mapped_batch "
                               "(extraction + odometry + scan-to-map of %s), median of %d repeats"
                               % (a.sensor, ns, synth.SENSORS[a.sensor][1], B, "every scan" if skip == 1 else "one scan in %d" % skip, a.repeats)}
            if B == 1:
                sm = float(np.median(solo_times))
                rec["solo_scan_stream_mapped"] = {"value": K / sm, "ms_per_step": 1e3 * sm / K,
                                                  "ms_per_step_range": [1e3 * min(solo_times) / K, 1e3 * max(solo_times) / K]}
            print(json.dumps(rec), flush=True)
        for ctx in list(ctxs.values()) + [solo_ctx]:
            ctx.close()


if __name__ == "__main__":
    main()
