"""Place recognition (Scan Context, aloam_place_*): describe time per scan, brute-force query time against M keyframes, the cost of
keyframe recording inside the mapped stream, and relocalisation through place hypotheses against the grid search.
  describe   aloam_place_describe of HDL-32 32 x 2200 scan 30 (its less-sharp / less-flat clouds), median of --repeats calls;
  query      M = 10^3, 10^4, 10^5 random keyframe records, n_query 1 and 16, k = 10: median of --repeats synchronous calls;
  record     aloam_scan_stream_mapped_batch over 20 HDL-32 32 x 2200 scans at 1 and 16 lanes, recording on (keyframe_gap 0, every
             mapped row a keyframe) against off, alternated --repeats times in one process: median call time of each;
  reloc      the ~76 k-point map of tools/bench_relocalise.py (HDL-32 scans 0 .. 59, seed BASE_SEED + 900, keyframes every 2 m):
             scan 31 relocalised through place_query (k = 3) + place_hypotheses (+-2 m, 1 m, +-10 deg in 5 deg) + prior_relocalise,
             against prior_relocalise over the 21 x 21 m x 72-heading grid (0.5 m) around its map pose.
Host clock around synchronous calls.  The GPU's name and power limit are read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_place.py [--repeats 5] [--out FILE]"""
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
        raise SystemExit("bench_place needs a GPU")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    name, power = gpu_info()
    res = {"gpu": name, "power_limit": power}
    seed = synth.BASE_SEED + 900
    scans = [synth.scan("HDL-32", k, seed=seed) for k in range(60)]
    M = max(s.shape[0] for s in scans) + 1024
    ctx = pkg.Aloam(n_scans=32, max_points=M, max_batch=16, max_map_points=400000, max_ring_points=4096)
    f = ctx.extract_features(scans[30])
    res["describe_ms"] = timed(lambda: ctx.place_describe(f["less_sharp"], f["less_flat"]), a.repeats)
    rng = np.random.default_rng(0)
    q = {}
    for m in (1000, 10000, 100000):
        rec = np.zeros(m, pkg.PLACE_RECORD_DTYPE)
        rec["pose"][:, 3] = 1.0; rec["max_range"] = 80.0; rec["z_offset"] = 2.0
        rec["desc"] = rng.uniform(0, 6, (m, 1200)).astype(np.float32)
        ctx.place_db_load(rec)
        for nq in (1, 16):
            d = rec["desc"][:nq].copy()
            q["M%d_q%d" % (m, nq)] = timed(lambda: ctx.place_query(d, 10), a.repeats)
    res["query_ms"] = q
    ctx.place_db_clear()
    dev = [torch.from_numpy(s).cuda() for s in scans[:20]]
    rec_ms = {}
    for lanes in (1, 16):
        c = pkg.Aloam(n_scans=32, max_points=M, max_batch=lanes, max_map_points=400000, max_ring_points=4096)
        ptrs = np.array([[d.data_ptr()] * lanes for d in dev], np.uint64); counts = np.array([[d.shape[0]] * lanes for d in dev], np.int64)
        ts = {True: [], False: []}
        for r in range(a.repeats + 1):
            for on in (False, True):
                c.set_place(on, keyframe_gap=0.0, max_keyframes=64)
                c.reset_odometry()
                torch.cuda.synchronize()
                t0 = time.perf_counter(); c.scan_stream_mapped_batch(ptrs, counts, True); dt = (time.perf_counter() - t0) * 1e3
                if r:
                    ts[on].append(dt)
        rec_ms["lanes%d" % lanes] = {"off": float(np.median(ts[False])), "on": float(np.median(ts[True]))}
        c.close()
    res["record_20_scans_ms"] = rec_ms
    # relocalisation: map scans 0..59 with keyframes every 2 m, relocalise scan 31 (not a keyframe unless the gate says so)
    c = pkg.Aloam(n_scans=32, max_points=M, max_batch=1, max_map_points=400000, max_ring_points=4096)
    c.set_place(True, keyframe_gap=2.0, max_keyframes=64)
    dev = [torch.from_numpy(s).cuda() for s in scans]
    ops = np.full((60, 1), 1, np.int32); ops[0] = 2
    _, mp = c.scan_stream_lanes(np.array([[d.data_ptr()] for d in dev], np.uint64), np.array([[d.shape[0]] for d in dev], np.int64), ops, True)
    rows = c.place_rows(60)
    recs = c.place_keyframes(0)
    blob = c.lane_save(0)
    c.close()
    L = pkg.Aloam(n_scans=32, max_points=M, max_batch=1, max_map_points=400000, max_ring_points=4096)
    L.prior_map_load(blob)
    L.place_db_load(recs)
    k = next(j for j in range(31, 60) if rows["keyframe"][j] < 0)
    fk = L.extract_features(scans[k])

    def place_path():
        m = L.place_query(L.place_describe(fk["less_sharp"], fk["less_flat"]), 3)
        h = pkg.place_hypotheses({"keyframe": m["keyframe"][0], "shift": m["shift"][0]}, recs, 2.0, 1.0, np.deg2rad(10), np.deg2rad(5))
        out, _ = L.prior_relocalise(h, fk["less_sharp"], fk["less_flat"], refine=1, scores=False)
        return out[0]["pose"], h.shape[0]

    p, nh = place_path()
    grid = pkg.pose_grid(mp[k, 0, :4], mp[k, 0, 4:], 10.5, 0.5, np.arange(72) * (2 * np.pi / 72))
    res["reloc"] = {"keyframes": int(len(recs)), "scan": int(k), "place_hypotheses": int(nh),
                    "place_err_m": float(np.linalg.norm(p[4:] - mp[k, 0, 4:])),
                    "place_ms": timed(place_path, a.repeats), "grid_hypotheses": int(grid.shape[0]),
                    "grid_ms": timed(lambda: L.prior_relocalise(grid, fk["less_sharp"], fk["less_flat"], refine=1, scores=False), a.repeats)}
    L.close(); ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
