#!/usr/bin/env python
"""Mapping lanes that start on a copy of the prior map (aloam_lane_map_on_prior) against lanes that start on an empty store.
Two prior maps:
  hdl32   the store of an HDL-32 lane that mapped --steps scans of one seeded trajectory (bench_localise.py's map, about 76 k points),
          loaded from its snapshot;
  built   synth.build_map's 1 M-point HDL-64 map built at the HDL-64 leaves (bench_prior_build.py's map, about 0.8 M points).
Per map, with one untimed pass of each arm first and the arms alternating --repeats times:
  start   a call of one step that STARTs one lane, seeded or fresh: the extra time of a seeded START (host clock around the
          synchronous call, which ends in a device synchronise), and its launches;
  steps   B = 1 and 16 lanes replaying the map's trajectory from its first scan, seeded at that scan's pose or fresh, --steps scans: ms per
          step.  A seeded lane gathers and indexes full windows from its first frame, so it costs more per step than a young map.
A map that does not fit a lane's store (a cube above the slab capacity) is reported as refused.  One JSON line per map with every
number, the GPU's name and its power limit, read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_map_on_prior.py [--steps 40] [--repeats 3]"""
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


def stats(ts):
    return {"median": round(float(np.median(ts)), 3), "range": [round(min(ts), 3), round(max(ts), 3)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if a.steps < 2 or a.repeats < 1:
        ap.error("steps >= 2, repeats >= 1")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_map_on_prior needs a CUDA device")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    ident = (np.array([0, 0, 0, 1.0]), np.zeros(3))

    # the two maps, each with the scans its lanes replay and the context settings they run with
    worlds = {}
    scans = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 900, n_az=2200) for k in range(a.steps)]
    cfg = dict(n_scans=32, max_points=max(s.shape[0] for s in scans) + 1024, max_map_points=600000, max_ring_points=2304)
    ctx = pkg.Aloam(max_batch=1, **cfg)
    dev = [torch.from_numpy(s).cuda() for s in scans]
    ptrs = np.array([[d.data_ptr()] for d in dev], np.uint64)
    counts = np.array([[s.shape[0]] for s in scans], np.int64)
    ops = np.full((a.steps, 1), pkg.LANE_SCAN, np.int32)
    ops[0] = pkg.LANE_START
    ctx.scan_stream_lanes(ptrs, counts, ops, True)
    blob = ctx.lane_save(0)
    ctx.close()
    worlds["hdl32"] = (dev, cfg, lambda c: c.prior_map_load(blob), ident)
    fx = pkg.Aloam(n_scans=64, max_points=200000)

    def feats(raw):
        f = fx.extract_features(raw)
        return f["less_sharp"], f["less_flat"]

    corner, surf = synth.build_map(feats, 1_000_000)
    fx.close()
    scans64 = [synth.scan("HDL-64", k) for k in range(a.steps)]
    dev64 = [torch.from_numpy(x).cuda() for x in scans64]
    cfg64 = dict(n_scans=64, max_points=max(x.shape[0] for x in scans64) + 1024, max_map_points=600000)
    worlds["built"] = (dev64, cfg64, lambda c: c.prior_map_build(corner, surf), synth.pose(0))   # the map frame is the world frame

    for key, (dev, cfg, install, init) in worlds.items():
        out = {"map": key, "gpu": name, "power_limit": power}
        for B in (1, 16):
            ctx = pkg.Aloam(max_batch=B, **cfg)
            install(ctx)
            out["map_points"] = int(ctx.mapper_export_size(pkg.EXPORT_MAP, pkg.PRIOR_MAP))
            try:
                ctx.lane_map_on_prior(0, *init)
            except pkg.AloamError as e:
                out["refused"] = e.code
                ctx.close()
                break
            n = len(dev)
            ptrs = np.array([[d.data_ptr()] * B for d in dev], np.uint64)
            counts = np.array([[d.shape[0]] * B for d in dev], np.int64)
            ops = np.full((n, B), pkg.LANE_SCAN, np.int32)
            ops[0] = pkg.LANE_START

            def run(arm, steps):
                ctx.reset_odometry()
                if arm == "seeded":
                    for l in range(B):
                        ctx.lane_map_on_prior(l, *init)
                l0, t0 = ctx.launch_count(), time.perf_counter()
                ctx.scan_stream_lanes(ptrs[:steps], counts[:steps], ops[:steps], True)
                return (time.perf_counter() - t0) * 1e3 / steps, ctx.launch_count() - l0

            arms = ("fresh", "seeded")
            if B == 1:   # the START step alone
                for arm in arms:
                    run(arm, 1)
                ts, launches = {x: [] for x in arms}, {}
                for _ in range(a.repeats):
                    for arm in arms:
                        t, launches[arm] = run(arm, 1)
                        ts[arm].append(t)
                out["start_ms"] = {arm: stats(ts[arm]) for arm in arms}
                out["start_extra_ms"] = round(float(np.median(ts["seeded"]) - np.median(ts["fresh"])), 3)
                out["start_launches"] = launches
            for arm in arms:
                run(arm, n)
            ts = {x: [] for x in arms}
            for _ in range(a.repeats):
                for arm in arms:
                    ts[arm].append(run(arm, n)[0])
            out["ms_per_step_B%d" % B] = {arm: stats(ts[arm]) for arm in arms}
            ctx.close()
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
