"""Relocalisation against a prior map (aloam_prior_relocalise): time per call and hypotheses scored per second.
Two maps, one process:
  loc76k  the ~76 k-point map of tools/bench_localise.py: the snapshot of a lane that mapped HDL-32 32 x 2200 scans 0 .. 59 of
          seed BASE_SEED + 900; the scan relocalised is scan 30 of that trajectory, hypotheses around its map pose;
  built1M the 1 M-point map of tools/bench_prior_build.py (synth.build_map of HDL-64 features, leaves 0.4 / 0.8), built with
          aloam_prior_map_build; the scan is HDL-64 scan 24 at its true pose.
Per map, n_hyp in --hyps and max_score_points in --points, refine = 1: the median and range of --repeats calls (host clock around
the synchronous call, after one untimed call), hypotheses per second, and from one profiled call the time of the k_reloc_score
launches (CUDA events around them: the coarse launch and the one over the refined poses) and the probe model: 27 probes per
scoring point and hypothesis, and the fraction of (point, hypothesis) pairs that are inliers -- the ones that leave the candidate
walk early.  Then the call at n_hyp = K = 1 and K = 16 (the scoring is negligible there: the time is the upload, the stack filter
and the refining frames), and the oracle's scoring rate on one host core on the same scan and hypotheses.  The GPU's name and power
limit are read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_relocalise.py [--hyps 1000,10000,100000,1000000] [--points 256,1024] [--repeats 5]"""
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


def hypotheses(pkg, pose7, n):
    """n hypotheses around pose7: 0.5 m lattice, 72 headings, as wide as n needs, first n rows"""
    half = 0.5
    while (2 * int(half / 0.5) + 1) ** 2 * 72 < n:
        half += 0.5
    return pkg.pose_grid(pose7[:4], pose7[4:], half, 0.5, np.arange(72) * (2 * np.pi / 72))[:n]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hyps", default="1000,10000,100000,1000000")
    ap.add_argument("--points", default="256,1024")
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    hyps_n = [int(x) for x in a.hyps.split(",")]
    points = [int(x) for x in a.points.split(",")]
    if a.repeats < 1 or min(hyps_n) < 16 or min(points) < 1:
        ap.error("repeats >= 1, hyps >= 16, points >= 1")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_relocalise needs a CUDA device")
    pkg = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    import reloc_cases as RC
    name, power = gpu_info()

    # ---- the two maps, each in its own context, with the scan to relocalise and its pose
    worlds = {}
    scans = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 900, n_az=2200) for k in range(60)]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    maxn = max(s.shape[0] for s in scans) + 1024
    m = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_ring_points=2304)
    ptrs = np.array([[d.data_ptr()] for d in dev], np.uint64)
    counts = np.array([[s.shape[0]] for s in scans], np.int64)
    ops = np.full((60, 1), pkg.LANE_SCAN, np.int32)
    ops[0] = pkg.LANE_START
    _, mp = m.scan_stream_lanes(ptrs, counts, ops, True)
    blob = m.lane_save(0)
    m.close()
    c = pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_ring_points=2304)
    c.prior_map_load(blob)
    f = c.extract_features(scans[30])
    worlds["loc76k"] = (c, f, mp[30, 0], (0.2, 0.4))
    fx = pkg.Aloam(n_scans=64, max_points=200000)

    def feats(raw):
        g = fx.extract_features(raw)
        return g["less_sharp"], g["less_flat"]

    corner, surf = synth.build_map(feats, 1_000_000)
    f64 = fx.extract_features(synth.scan("HDL-64", 24))
    fx.close()
    c = pkg.Aloam(n_scans=64, max_points=200000, line_res=0.4, plane_res=0.8)
    c.prior_map_build(corner, surf)
    q, t = synth.pose(24)
    worlds["built1M"] = (c, f64, np.concatenate([q, t]), (0.4, 0.8))

    for wname, (ctx, f, pose7, leaves) in worlds.items():
        n_map = ctx.mapper_export_size(pkg.EXPORT_MAP, pkg.PRIOR_MAP)
        for npts in points:
            for n in hyps_n:
                H = hypotheses(pkg, pose7, n)
                run = lambda: ctx.prior_relocalise(H, f["less_sharp"], f["less_flat"], inlier_sq=0.25, max_score_points=npts, refine=1)
                run()
                ts = []
                for _ in range(a.repeats):
                    t0 = time.perf_counter(); res, sc = run(); ts.append((time.perf_counter() - t0) * 1e3)
                ctx.profile_enable(True)
                ctx.profile_read()
                run()
                prof = ctx.profile_read()
                ctx.profile_enable(False)
                m_pts = sum(min(len(s), npts) for s in RC.scoring_points(f["less_sharp"], f["less_flat"], npts, *leaves))
                med = float(np.median(ts))
                print(json.dumps({"map": wname, "map_points": n_map, "n_hyp": n, "max_score_points": npts, "scoring_points": m_pts,
                                  "call_ms_median": round(med, 3), "call_ms_range": [round(min(ts), 3), round(max(ts), 3)],
                                  "hyp_per_s": round(n / med * 1e3), "k_reloc_score_ms": round(prof.get("k_reloc_score", (0, 0))[0], 4),
                                  "k_reloc_score_launches": prof.get("k_reloc_score", (0, 0))[1],
                                  "k_reloc_topk_ms": round(prof.get("k_reloc_topk", (0, 0))[0], 4),
                                  "probes": 27 * m_pts * n, "inlier_fraction": round(float(sc.sum()) / (m_pts * n), 4),
                                  "best": [res[0]["score"], res[0]["refined_score"]], "gpu": name, "power_limit": power}), flush=True)
        # the refine stage: n_hyp = K
        for K in (1, 16):
            H = hypotheses(pkg, pose7, K)
            run = lambda: ctx.prior_relocalise(H, f["less_sharp"], f["less_flat"], inlier_sq=0.25, max_score_points=256, refine=K, scores=False)
            run()
            ts = []
            for _ in range(a.repeats):
                t0 = time.perf_counter(); run(); ts.append((time.perf_counter() - t0) * 1e3)
            print(json.dumps({"map": wname, "refine": K, "n_hyp": K, "call_ms_median": round(float(np.median(ts)), 3),
                              "call_ms_range": [round(min(ts), 3), round(max(ts), 3)], "gpu": name, "power_limit": power}), flush=True)
        # the oracle's scoring rate on one host core, same scan and hypotheses
        import pyoracle
        # kd-trees over the map's clouds by type (for the built map its input clouds: the rate, not the scores, is measured)
        S = RC.FrozenScorer.__new__(RC.FrozenScorer)
        if wname == "built1M":
            S.trees = [pyoracle.KdTree(corner), pyoracle.KdTree(surf)]
        else:
            info = pkg.snapshot_store_clouds(blob)
            S.trees = [pyoracle.KdTree(info["corner"]), pyoracle.KdTree(info["surf"])]
        H = hypotheses(pkg, pose7, 200)
        for npts in points:
            pts = RC.scoring_points(f["less_sharp"], f["less_flat"], npts, *leaves)
            t0 = time.perf_counter()
            S.score_points(pts, H, 0.25)
            dt = time.perf_counter() - t0
            print(json.dumps({"map": wname, "oracle_one_core": True, "max_score_points": npts, "n_hyp": len(H),
                              "hyp_per_s": round(len(H) / dt, 1)}), flush=True)
        ctx.close()


if __name__ == "__main__":
    main()
