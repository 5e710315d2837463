#!/usr/bin/env python
"""Cost of cube growth (aloam_set_cube_growth).
  (a) no regression with growth off: bench.py's mapped_stream record (HDL-64 scans through aloam_scan_stream_mapped, growth
      never set) run from this tree and from a parent tree (--parent-tree, a checkout with its library built), in ABBA order
      within one call: ms_per_step of every run and the run-to-run spread.
  (b) growth off against on on that trajectory (nothing grows), at 1 and 16 lanes (aloam_scan_stream_mapped_batch).
  (c) growth on where it happens: the VLP-16 trajectory at the default 0.2 / 0.4 m leaves and the OS64 field-mode trajectory, at 1
      and 16 lanes, off against on.
  (d) device memory per mapping lane (cudaMemGetInfo before and after a context maps one lane), off against on.
Per-step time = wall time of one stream call over all scans (device-resident), synchronised, divided by the scans; median of
--repeats calls after one untimed call.  Prints one JSON line per measurement and a last line with the GPU name and power limit.
usage: python tools/bench_cube_growth.py [--parent-tree DIR] [--scans 48] [--repeats 5] [--bench-steps 20]"""
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
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return name, power
    except Exception:
        return "unknown", "unknown"


def scene(synth, name, n):
    """(raw scans, Aloam keyword arguments) of a named trajectory"""
    if name == "os64":
        raws = [synth.scan_rings("OS64", k) for k in range(n)]
        return raws, dict(n_scans=len(synth.RING_SENSORS["OS64"][0]), ring_source=1, minimum_range=0.3, line_res=0.2, plane_res=0.4)
    raws = [synth.scan("VLP-16", k, seed=synth.BASE_SEED + 50, n_az=900) for k in range(n)]
    leaves = dict(line_res=0.5, plane_res=1.0) if name == "vlp16_coarse" else dict(line_res=0.2, plane_res=0.4)
    return raws, dict(n_scans=16, **leaves)


def run(name, lanes, growth, n, repeats):
    """ms per step of the mapped stream: one process"""
    import torch
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    raws, kw = scene(synth, name, n)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    free0 = torch.cuda.mem_get_info()[0]
    c = pkg.Aloam(max_points=max(len(r) for r in raws) + 1024, max_map_points=400000, max_batch=lanes, **kw)
    c.set_cube_growth(growth)
    ptrs = np.array([[d.data_ptr()] * lanes for d in dev], np.uint64)
    counts = np.array([[len(r)] * lanes for r in raws])
    times = []
    for r in range(repeats + 1):
        c.mapper_reset()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if lanes == 1:
            c.scan_stream_mapped(ptrs[:, 0], counts[:, 0], True)
        else:
            c.scan_stream_mapped_batch(ptrs, counts, True)
        torch.cuda.synchronize()
        if r:
            times.append(1e3 * (time.perf_counter() - t0) / n)
    mem = free0 - torch.cuda.mem_get_info()[0]
    c.close()
    return {"ms_per_step": float(np.median(times)), "each": times, "device_bytes": int(mem)}


def child(args):
    print(json.dumps(run(args.scene, args.lanes, args.growth, args.scans, args.repeats)))


def spawn(name, lanes, growth, n, repeats):
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--scene", name, "--lanes", str(lanes), "--growth", str(growth),
           "--scans", str(n), "--repeats", str(repeats)]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout.strip().splitlines()
    return json.loads(out[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-tree", default="", help="a checkout of the parent commit with its library built")
    ap.add_argument("--bench-steps", type=int, default=20)
    ap.add_argument("--scans", type=int, default=48)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--child", action="store_true")
    ap.add_argument("--scene", default="vlp16_coarse")
    ap.add_argument("--lanes", type=int, default=1)
    ap.add_argument("--growth", type=int, default=0)
    args = ap.parse_args()
    if args.child:
        return child(args)
    name, power = gpu_info()
    n, rp = args.scans, args.repeats
    if args.parent_tree:   # (a) bench.py's mapped_stream, ABBA
        order = ["this", "parent", "parent", "this"]
        res = {"this": [], "parent": []}
        for which in order:
            tree = ROOT if which == "this" else os.path.abspath(args.parent_tree)
            cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(args.bench_steps), "--warmup", "5",
                   "--no-cpu-baseline", "--no-batch", "--no-mapping"]
            out = subprocess.run(cmd, cwd=tree, capture_output=True, text=True, check=True).stdout
            rec = [json.loads(l) for l in out.splitlines() if l.startswith("{")][-1]
            res[which].append(rec["mapped_stream"]["ms_per_step"])
        allv = res["this"] + res["parent"]
        print(json.dumps({"measure": "abba_bench_mapped_stream", "order": order, "this_ms_per_step": res["this"],
                          "parent_ms_per_step": res["parent"], "spread_ms": max(allv) - min(allv),
                          "this_minus_parent_ms": float(np.mean(res["this"]) - np.mean(res["parent"]))}))
    for scn in ("vlp16_coarse", "vlp16_default", "os64"):   # (b), (c), (d)
        for lanes in (1, 16):
            r = {g: spawn(scn, lanes, g, n if scn != "os64" else min(n, 20), rp) for g in (0, 1)}
            print(json.dumps({"measure": "growth_off_vs_on", "scene": scn, "lanes": lanes, "off_ms_per_step": r[0]["ms_per_step"],
                              "on_ms_per_step": r[1]["ms_per_step"], "off_each": r[0]["each"], "on_each": r[1]["each"],
                              "device_bytes_off": r[0]["device_bytes"], "device_bytes_on": r[1]["device_bytes"]}))
    print(json.dumps({"gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
