#!/usr/bin/env python
"""Cost of localising lane snapshots (aloam_lane_save_localising / aloam_lane_restore, format version 2) and of the prior-map digest.
The world is bench_localise.py's: HDL-32 32 x 2200 scans of one seeded trajectory; one lane maps its first --map-scans scans and its
snapshot is the prior map (about 76 k points at 60 scans).
1. Save and restore: a lane localising against that map, saved to a device tensor and to a pinned host tensor and restored from
   each; median microseconds of the synchronous calls (host clock) and the snapshot's size.  The restored lane saves the same bytes.
2. Digest: the first aloam_prior_map_digest call after a load or build (one launch over the map and a synchronisation; host clock
   around the call) on that map and on maps built (aloam_prior_map_build) from lattice clouds of 1 M and 8 M points, median of
   --repeats, and the map's points.
3. Time slicing: 32 localising trajectories over 16 lanes (trajectory t starts at scan t of the mapped run, armed with the map pose
   found there, and runs --scans scans) -- once in two groups of 16 run to their end, once round-robin in slices of 10 and of 5 scans
   with a save and a restore at every swap; useful scans per second of each (median of --repeats, alternating) and whether every
   trajectory's odometry and map poses are bit-identical between them.
Every line carries the GPU name and power limit read in the same run.  Needs a GPU: without one it fails.
usage: python tools/bench_localise_snapshot.py [--repeats 5] [--scans 20] [--map-scans 60]"""
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
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                         timeout=30).stdout.strip()
    name, power = [s.strip() for s in out.split(",")[:2]]
    return name, power


def _median_us(fn, reps, torch):
    us = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        us.append(1e6 * (time.perf_counter() - t0))
    return float(np.median(us))


def _ctx(maxn, batch):
    return pkg.Aloam(n_scans=32, max_points=maxn, max_map_points=600000, max_batch=batch, max_ring_points=2304)


def _call(ctx, lanes, plan):
    """plan = {lane: [(address, points, op), ...]}: one mapped lanes call -> {lane: (odometry, map poses) of its entries}"""
    steps = max(len(e) for e in plan.values())
    ptrs, counts, ops = np.zeros((steps, lanes), np.uint64), np.zeros((steps, lanes), np.int64), np.zeros((steps, lanes), np.int32)
    for lane, entries in plan.items():
        for k, (p, n, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    o, m = ctx.scan_stream_lanes(ptrs, counts, ops, True)
    return {lane: (o[:len(e), lane], m[:len(e), lane]) for lane, e in plan.items()}


def _entries(dev, i0, i1, start):
    return [(d.data_ptr(), d.shape[0], pkg.LANE_START if start and i == i0 else pkg.LANE_SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def bench_save_restore(torch, gpu, R, dev, maxn, blob, map_poses):
    ctx = _ctx(maxn, 1)
    ctx.prior_map_load(blob)
    ctx.lane_localise(0, map_poses[3][:4], map_poses[3][4:])
    _call(ctx, 1, {0: _entries(dev, 3, 8, True)})
    ref = ctx.lane_save_localising(0)
    n = len(ref)
    bufs = {"device": torch.empty(n, dtype=torch.uint8, device="cuda"), "pinned_host": torch.empty(n, dtype=torch.uint8).pin_memory()}
    res = {}
    for name, buf in bufs.items():
        save = _median_us(lambda: ctx.lane_save_localising(0, buf), R, torch)
        restore = _median_us(lambda: ctx.lane_restore(0, buf), R, torch)
        assert ctx.lane_save_localising(0).tobytes() == ref.tobytes(), name
        res[name] = {"save_us": round(save, 1), "restore_us": round(restore, 1)}
    print(json.dumps({"bench": "localise_snapshot", "bytes": n, "last_points": int((n - 256 - 128) // 16), **res,
                      "prior_map_points": int(pkg.snapshot_info(blob.cpu().numpy())["map_points"]), "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)
    ctx.close()


def _lattice(n_points):
    """a map-frame cloud of n_points on a 0.5 m lattice over the 1000 x 1000 m around the origin, two layers deep (every point in a
    voxel of its own at the 0.2 / 0.4 m leaves, 20 000 points per 50 m cube at 8 M): (corner = the first eighth, surf = the rest)"""
    side = 2000
    layers = max(1, -(-n_points // (side * side)))
    k = np.arange(n_points, dtype=np.int64)
    p = np.zeros((n_points, 4), np.float32)
    p[:, 0] = -500.0 + 0.5 * (k % side)
    p[:, 1] = -500.0 + 0.5 * ((k // side) % side)
    p[:, 2] = 0.5 * ((k // (side * side)) % layers)
    p[:, 3] = (k % 7).astype(np.float32)
    nc = n_points // 8
    return p[:nc], p[nc:]


def bench_digest(torch, gpu, R, maxn, blob):
    ctx = _ctx(maxn, 1)
    maps = [("snapshot", lambda: ctx.prior_map_load(blob))]
    for n in (1_000_000, 8_000_000):
        corner, surf = _lattice(n)
        c_dev, s_dev = torch.from_numpy(corner).cuda(), torch.from_numpy(surf).cuda()
        maps.append(("built_from_%dM_points" % (n // 1_000_000), lambda a=c_dev, b=s_dev: ctx.prior_map_build(a, b)))
    for name, install in maps:
        us, digest = [], None
        for _ in range(R + 1):   # the first one warms up
            install()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            d = ctx.prior_map_digest()
            us.append(1e6 * (time.perf_counter() - t0))
            assert digest is None or d == digest, name
            digest = d
        points = ctx.mapper_export_size(pkg.EXPORT_MAP, pkg.PRIOR_MAP)
        med = float(np.median(us[1:]))
        print(json.dumps({"bench": "prior_map_digest", "map": name, "map_points": int(points), "digest_call_us": round(med, 1),
                          "GB_per_s": round(16 * points / med / 1e3, 1), "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)
    ctx.close()


def run_unsliced(ctx, dev, lanes, plan, L):
    out = {}
    for g in range(0, len(plan), lanes):
        group = list(plan)[g:g + lanes]
        for i, t in enumerate(group):
            ctx.lane_localise(i, *plan[t][1])
        res = _call(ctx, lanes, {i: _entries(dev, plan[t][0], plan[t][0] + L, True) for i, t in enumerate(group)})
        out.update({t: res[i] for i, t in enumerate(group)})
    return out


def run_sliced(ctx, dev, lanes, plan, L, S):
    pos, saved, parts, order = {t: 0 for t in plan}, {}, {t: [] for t in plan}, list(plan)
    while any(p < L for p in pos.values()):
        group = [t for t in order if pos[t] < L][:lanes]
        calls = {}
        for i, t in enumerate(group):
            s0, init = plan[t]
            if t in saved:
                ctx.lane_restore(i, saved.pop(t))
            else:
                ctx.lane_localise(i, *init)
            calls[i] = _entries(dev, s0 + pos[t], s0 + min(pos[t] + S, L), not parts[t])
        res = _call(ctx, lanes, calls)
        for i, t in enumerate(group):
            parts[t].append(res[i])
            pos[t] += len(calls[i])
            if pos[t] < L:
                saved[t] = ctx.lane_save_localising(i)
        order = order[len(group):] + group
    return {t: (np.concatenate([p[0] for p in ps]), np.concatenate([p[1] for p in ps])) for t, ps in parts.items()}


def bench_slicing(torch, gpu, R, dev, maxn, blob, map_poses, L, slices):
    lanes, n = 16, 32
    plan = {t: (t, (map_poses[t][:4], map_poses[t][4:])) for t in range(n)}
    modes = ["whole"] + ["slice_%d" % s for s in slices]
    ctx = {}
    for m in modes:
        ctx[m] = _ctx(maxn, lanes)
        ctx[m].prior_map_load(blob)
    run = {"whole": lambda: run_unsliced(ctx["whole"], dev, lanes, plan, L)}
    for s in slices:
        run["slice_%d" % s] = lambda s=s: run_sliced(ctx["slice_%d" % s], dev, lanes, plan, L, s)
    secs, poses = {m: [] for m in modes}, {}
    for r in range(R + 1):   # run 0 warms up
        for m in (modes if r % 2 == 0 else modes[::-1]):
            ctx[m].reset_odometry()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            poses[m] = run[m]()
            torch.cuda.synchronize()
            if r > 0:
                secs[m].append(time.perf_counter() - t0)
    useful = n * L
    rate = {m: useful / float(np.median(v)) for m, v in secs.items()}
    for s in slices:
        m = "slice_%d" % s
        same = all(np.array_equal(poses["whole"][t][0], poses[m][t][0]) and np.array_equal(poses["whole"][t][1], poses[m][t][1]) for t in plan)
        print(json.dumps({"bench": "localise_time_slicing", "sensor": "HDL-32", "lanes": lanes, "trajectories": n, "scans_each": L, "slice": s,
                          "useful_scans_per_s_unsliced": round(rate["whole"], 1), "useful_scans_per_s_sliced": round(rate[m], 1),
                          "sliced_over_unsliced": round(rate[m] / rate["whole"], 3), "poses_identical": bool(same),
                          "gpu": gpu[0], "power_limit": gpu[1]}), flush=True)
    for c in ctx.values():
        c.close()


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--scans", type=int, default=20)
    ap.add_argument("--map-scans", type=int, default=60)
    a = ap.parse_args()
    if a.scans < 2 or a.repeats < 1 or a.map_scans < 32 + a.scans:
        ap.error("scans >= 2, repeats >= 1, map-scans >= 32 + scans (trajectory t runs scans t .. t + scans - 1)")
    if not torch.cuda.is_available():
        raise SystemExit("bench_localise_snapshot needs a CUDA device")
    gpu = gpu_info()
    scans = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 900, n_az=2200) for k in range(a.map_scans)]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    maxn = max(s.shape[0] for s in scans) + 1024
    # the prior map: one lane maps the first map_scans scans (bench_localise.py's world); its map poses arm the localising lanes
    mapper = _ctx(maxn, 1)
    _, map_poses = _call(mapper, 1, {0: _entries(dev, 0, a.map_scans, True)})[0]
    blob = mapper.lane_save(0, torch.empty(mapper.lane_save(0).size, dtype=torch.uint8, device="cuda"))
    mapper.close()
    bench_save_restore(torch, gpu, a.repeats * 4, dev, maxn, blob, map_poses)
    bench_digest(torch, gpu, a.repeats, maxn, blob)
    bench_slicing(torch, gpu, a.repeats, dev, maxn, blob, map_poses, a.scans, (10, 5))


if __name__ == "__main__":
    main()
