"""Loop verification (aloam_set_loops, aloam_loop_verify): the per-step cost of verification inside the mapped stream, and the time
of one verification on request.
  stream   aloam_scan_stream_lanes over a 20-scan HDL-32 32 x 2200 return trip (scans 0 .. 10 of seed BASE_SEED + 900, then scans
           9 .. 0 of another seed), every lane STARTing at scan 0, at 1 and 16 lanes.  Place recording on in every mode (keyframe_gap
           0, exclude_recent 4); loops off, on but never triggering (max_distance 0), and on with every candidate verified
           (max_distance 2); window 10, cloud_points 1000, outer_iters 4.  The modes alternate --repeats times in one process:
           median call time / 20 steps.
  verify   aloam_loop_verify of the last keyframe of a 40 + 39-scan return trip against its candidate, window 10 / 25 x outer_iters
           4 / 8 (cloud_points 1000): median of --repeats synchronous calls.
Host clock around synchronous calls.  The GPU's name and power limit are read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_loops.py [--repeats 5] [--out FILE]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")[:2]]
    return name, power


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter(); fn(); ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_loops needs a GPU")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power}
    seed = synth.BASE_SEED + 900
    trip = [synth.scan("HDL-32", k, seed=seed) for k in range(11)] + [synth.scan("HDL-32", k, seed=seed + 1) for k in range(9, -1, -1)]
    M = max(s.shape[0] for s in trip) + 1024
    dev = [torch.from_numpy(s).cuda() for s in trip]
    loop = dict(window=10, cloud_points=1000, outer_iters=4)
    stream = {}
    for lanes in (1, 16):
        c = pkg.Aloam(n_scans=32, max_points=M, max_batch=lanes, max_map_points=400000, max_ring_points=4096)
        c.set_place(True, keyframe_gap=0.0, exclude_recent=4, max_keyframes=64)
        ptrs = np.array([[d.data_ptr()] * lanes for d in dev], np.uint64); counts = np.array([[d.shape[0]] * lanes for d in dev], np.int64)
        ops = np.full((len(dev), lanes), 1, np.int32); ops[0] = 2
        modes = {"off": None, "never": 0.0, "on": 2.0}
        ts = {m: [] for m in modes}
        verified = 0
        for r in range(a.repeats + 1):
            for m, dist in modes.items():
                if dist is None:
                    c.set_place(True, keyframe_gap=0.0, exclude_recent=4, max_keyframes=64)
                else:
                    c.set_loops(True, max_distance=dist, **loop)
                torch.cuda.synchronize()
                t0 = time.perf_counter(); c.scan_stream_lanes(ptrs, counts, ops, True); dt = (time.perf_counter() - t0) * 1e3
                if r:
                    ts[m].append(dt / len(dev))
                if m == "on":
                    verified = sum(row["verified"] for row in c.loop_rows(len(dev) * lanes))
        stream["lanes%d" % lanes] = {m: float(np.median(v)) for m, v in ts.items()}
        stream["lanes%d" % lanes]["verified_rows"] = int(verified)
        c.close()
    res["stream_ms_per_step"] = stream
    # one verification on request: the last keyframe of a 40 + 39-scan return trip against its candidate
    out = [synth.scan("HDL-32", k, seed=seed) for k in range(40)]
    back = [synth.scan("HDL-32", k, seed=seed + 1) for k in range(38, -1, -1)]
    scans = out + back
    dev = [torch.from_numpy(s).cuda() for s in scans]
    M = max(s.shape[0] for s in scans) + 1024
    ver = {}
    for window in (10, 25):
        for outer in (4, 8):
            c = pkg.Aloam(n_scans=32, max_points=M, max_batch=1, max_map_points=400000, max_ring_points=4096)
            c.set_place(True, keyframe_gap=0.0, exclude_recent=10, max_keyframes=200)
            c.set_loops(True, max_distance=0.0, window=window, cloud_points=1000, outer_iters=outer)
            ops = np.full((len(scans), 1), 1, np.int32); ops[0] = 2
            c.scan_stream_lanes(np.array([[d.data_ptr()] for d in dev], np.uint64), np.array([[d.shape[0]] for d in dev], np.int64), ops, True)
            pr = c.place_rows(len(scans))
            q, cand, s = int(pr["keyframe"][-1]), int(pr["loop"][-1]), int(pr["shift"][-1])
            row = c.loop_verify(0, q, cand, s)
            ver["w%d_it%d" % (window, outer)] = {"ms": timed(lambda: c.loop_verify(0, q, cand, s), a.repeats), "n_sub": list(row["n_sub"]),
                                                  "score": row["score"], "n_score": row["n_score"]}
            c.close()
    res["verify"] = ver
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
