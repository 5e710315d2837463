"""GPU: odometry, mapping and the LM at non-default aloam_config values, against the oracle run with the same values.

* The association (aloam_odometry_associate) at every NEARBY_SCAN and DISTANCE_SQ_THRESHOLD of tests/config_cases.py on real
  VLP-16 / HDL-64 scan pairs, seam clouds whose int(intensity) descends, and hand-built clouds that plant nearer points just
  outside the ring window and candidates at float d2 = float(thr) and its neighbours: correspondences exact.
* Feature extraction at minimum_range 0, 1, 12.5 and 40 against the reference's own scanRegistration.cpp (oracle/_ref) and the
  oracle, with returns at exactly the range limit and one ulp inside it.
* aloam_solve at inner_iters x huber away from 4 x 0.1, and through the emulated-rank exchanges.
* Chains through scan_to_pose, scan_stream and a 4-lane scan_stream_batch, one context per setting; the mapped stream and a
  localising lane at outer_iters 1 / 3, inner_iters 8, huber 0.5; a snapshot taken under a non-default association."""
import math
import os
import struct

import numpy as np
import pytest

import config_cases as K
import edge_scenes as es
import lane_refs as R
import seam_cases as S
import test_gpu_lm_edges as LE
import test_gpu_localise as TL
from conftest import rot_angle
from refsource import ref_registration

pytestmark = pytest.mark.gpu

IDENT_Q, ZERO_T = np.array([0, 0, 0, 1.0]), np.zeros(3)
BAR = 1e-6
_FEAT = {}


def _features(orc, synth, sensor, t, k):
    """oracle features of scan k of trajectory t (VLP-16 at 900, HDL-64 at 600 azimuths), cached"""
    key = (sensor, t, k)
    if key not in _FEAT:
        raw = R.traj(synth, t, k + 1, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)[k]
        ns, _, mr = synth.SENSORS[sensor][:3]
        _FEAT[key] = (raw, orc.Features(raw, ns, mr))
    return _FEAT[key]


def _pairs(orc, synth):
    """(name, last corner, last surf, sharp, flat, q, t): real scan pairs at identity and moved, and the seam pairs"""
    q = np.array([0.001, -0.002, 0.008, 1.0]); q /= np.linalg.norm(q)
    out = []
    for sensor in ("VLP-16", "HDL-64"):
        (_, f0), (_, f1) = _features(orc, synth, sensor, 0, 0), _features(orc, synth, sensor, 0, 1)
        out.append((sensor, f0.less_sharp, f0.less_flat, f1.sharp, f1.flat, IDENT_Q, ZERO_T))
        out.append((sensor + "-moved", f0.less_sharp, f0.less_flat, f1.sharp, f1.flat, q, np.array([0.7, 0.02, -0.01])))
        ns, _, mr = synth.SENSORS[sensor][:3]
        g0, g1 = (orc.Features(S.trajectory_scan(synth, sensor, k), ns, mr) for k in (0, 1))
        assert S.descents(g0.less_sharp) + S.descents(g0.less_flat) > 0
        out.append(("seam-" + sensor, g0.less_sharp, g0.less_flat, g1.sharp, g1.flat, q, np.array([0.7, 0.02, -0.01])))
    return out


def _rows(cc, pc):
    return ([(int(a), int(b), int(c)) for a, b, c in cc], [tuple(int(v) for v in r) for r in pc])


def _check_assoc(ctx, orc, thr, nearby, distortion, name, lc, ls, sharp, flat, q, t):
    od = orc.Odometry(distortion=bool(distortion), dist_sq_thresh=thr, nearby_scan=nearby)
    od.set_last(lc, ls)
    cc, pc, _ = od.associate(sharp, flat, q, t)
    ctx.odometry_set_last(lc, ls)
    gcc, gpc = ctx.odometry_associate(sharp, flat, q, t)
    got = ([(i, a, b) for i, (a, b, v) in enumerate(gcc) if v], [(i, a, b, c) for i, (a, b, c, v) in enumerate(gpc) if v])
    want = _rows(cc, pc)
    for g, w, kind in zip(got, want, ("corner", "surf")):
        if g != w:
            diff = [(x, y) for x, y in zip(g, w) if x != y][:4]
            pytest.fail("%s thr=%r nearby=%r distortion=%d: %s rows differ (%d vs %d), first (got, expected): %s"
                        % (name, thr, nearby, distortion, kind, len(g), len(w), diff))
    return len(want[0]) + len(want[1])


@pytest.mark.parametrize("nearby", K.NEARBY, ids=K.NEARBY_IDS)
@pytest.mark.parametrize("distortion", [0, 1])
def test_association_at_every_ring_window(aloam, orc, synth, nearby, distortion):
    ctx = aloam.Aloam(n_scans=64, max_points=200000, nearby_scan=nearby, distortion=distortion)
    try:
        for case in _pairs(orc, synth):
            assert _check_assoc(ctx, orc, 25.0, nearby, distortion, *case) > 300
        last, queries = K.window_scene()
        assert _check_assoc(ctx, orc, 25.0, nearby, distortion, "window", last, last, queries, queries, IDENT_Q, ZERO_T) == 2 * len(queries)
    finally:
        ctx.close()


@pytest.mark.parametrize("thr", K.THRESH, ids=K.THRESH_IDS)
def test_association_at_every_threshold(aloam, orc, synth, thr):
    ctx = aloam.Aloam(n_scans=64, max_points=200000, dist_sq_thresh=thr)
    try:
        if thr < 3e38:   # finite in float32
            last, queries = K.threshold_scene(thr)
            _check_assoc(ctx, orc, thr, 2.5, 0, "planted", last, last, queries, queries, IDENT_Q, ZERO_T)
        # real scans a few metres apart: at 100 / 400 / 1e40 the sweeps grow bucket by bucket up to the whole circle
        q = np.array([0.0, 0.0, 0.05, 1.0]); q /= np.linalg.norm(q)
        for sensor in ("VLP-16", "HDL-64"):
            (_, f0), (_, f1) = _features(orc, synth, sensor, 0, 0), _features(orc, synth, sensor, 0, 1)
            for t in (np.zeros(3), np.array([3.0, -1.5, 0.2])):
                _check_assoc(ctx, orc, thr, 2.5, 0, sensor, f0.less_sharp, f0.less_flat, f1.sharp, f1.flat, q, t)
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------- features


def _at_norm(p, target):
    """p moved by a few ulps per coordinate so that float32 (x*x + y*y) + z*z == target (removeClosedPointCloud's expression)"""
    base = np.asarray(p, np.float32)
    for i in range(-4, 5):
        for j in range(-4, 5):
            for k in range(-4, 5):
                c = base.copy()
                for a, n in zip(range(3), (i, j, k)):
                    for _ in range(abs(n)):
                        c[a] = np.nextafter(c[a], np.float32(np.inf) if n > 0 else np.float32(-np.inf))
                if K.sqd(c, np.zeros(3, np.float32)) == target:
                    return c
    return None


def _range_scan(raw, thres, rng):
    """raw with 40 returns moved onto the range limit: 20 at float norm^2 == thres^2 (kept), 20 one float below (dropped)"""
    raw = raw.copy()
    t2 = np.float32(thres) * np.float32(thres)
    r = np.sqrt(np.sum(raw[:, :3].astype(np.float64) ** 2, axis=1))
    far = np.flatnonzero(r > 1.5 * thres)
    done = {True: 0, False: 0}
    for i in rng.permutation(far):
        keep = done[True] <= done[False]
        if done[keep] >= 20:
            keep = not keep
        if done[keep] >= 20:
            break
        target = t2 if keep else np.nextafter(t2, np.float32(0))
        p = _at_norm(raw[i, :3] * (float(thres) / r[i]), target)
        if p is not None:
            raw[i, :3] = p
            done[keep] += 1
    assert done == {True: 20, False: 20}, done
    return raw


def _check_features(got, ref, what):
    for name in ("full", "sharp", "less_sharp", "flat", "less_flat"):
        g, w = got[name], ref[name] if isinstance(ref, dict) else getattr(ref, name)
        assert g.shape == w.shape, (what, name, g.shape, w.shape)
        assert np.array_equal(g[:, :3], w[:, :3]), (what, name)
        assert np.array_equal(g[:, 3].astype(np.int32), w[:, 3].astype(np.int32)), (what, name)


@pytest.mark.parametrize("sensor,min_range", [("VLP-16", 0.0), ("VLP-16", 1.0), ("HDL-64", 12.5), ("VLP-16", 40.0), ("HDL-64", 40.0)])
def test_features_at_minimum_range(aloam, orc, synth, sensor, min_range):
    """at 40 m the scan is scaled by 4 (exact in float) so that enough returns lie beyond the limit"""
    ns = synth.SENSORS[sensor][0]
    raw = synth.scan(sensor, 1, n_az=900 if sensor == "VLP-16" else 600)
    if min_range >= 40:
        raw = raw.copy(); raw[:, :3] *= np.float32(4.0)
    if min_range > 0:
        raw = _range_scan(raw, min_range, np.random.default_rng(int(min_range * 10)))
    else:
        assert not np.any(np.all(raw[:, :3] == 0, axis=1))
    ctx = aloam.Aloam(n_scans=ns, max_points=raw.shape[0] + 1024, minimum_range=min_range)
    try:
        got = ctx.extract_features(raw)
        ref = ref_registration(ns, min_range).run(raw, orc.SORT_CANONICAL)
        _check_features(got, ref, ("reference source", sensor, min_range))
        _check_features(got, orc.Features(raw, ns, min_range), ("oracle", sensor, min_range))
        if min_range > 0:
            # the 20 returns at the limit are kept, the 20 one float inside are not
            n2 = K.sqd(raw[:, :3], np.zeros(3, np.float32))
            t2 = np.float32(min_range) * np.float32(min_range)
            kept = {bytes(p) for p in np.ascontiguousarray(got["full"][:, :3])}
            assert sum(bytes(p) in kept for p in np.ascontiguousarray(raw[n2 == t2, :3])) == 20
            assert not any(bytes(p) in kept for p in np.ascontiguousarray(raw[n2 == np.nextafter(t2, np.float32(0)), :3]))
        if min_range == 40.0:
            inside = synth.scan(sensor, 1, n_az=900 if sensor == "VLP-16" else 600).copy()
            inside[:, :3] *= np.float32(0.25)
            assert np.sqrt(np.sum(inside[:, :3].astype(np.float64) ** 2, axis=1)).max() < 40.0
            with pytest.raises(aloam.AloamError) as e:
                ctx.extract_features(inside)
            assert e.value.code == -3
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------- LM


def _lm_problems(orc):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "solve_hdl64_pair.npz"))
    out = [("golden", g["blocks"], g["x0"])]
    for name in ("gradient", "function", "iterations"):
        b, x0, _ = LE._problem(orc, name)
        out.append((name, b, x0))
    out.append(("rejected", es.near_parallel_planes(orc, 0), LE.IDENT))
    out.append(("huber", es.blocks(orc, np.random.default_rng(4), LE.X_TRUE, 400, noise=3.0), LE.IDENT))
    return out


def _compare_solve(ctx, orc, blocks, x0, inner, huber, what):
    xr, sr, tr = orc.solve(blocks, x0, max_iters=inner, huber=huber)
    xg, sg, tg = ctx.solve(blocks, x0)
    for k in ("termination", "num_iterations", "num_successful"):
        assert sg[k] == sr[k], (what, k, sg[k], sr[k])
    assert np.all(np.isfinite(xg)) and np.abs(xg - xr).max() < 1e-9, (what, np.abs(xg - xr).max())
    n = min(len(tr), 8)   # ALOAM_LM_MAX_TRACE rows
    assert len(tg) == n, (what, len(tg), len(tr))
    nb = len(blocks)
    assert np.all(np.abs(tg[:n, 0] - tr[:n, 0]) <= LE._cost_tol(tr[:n, 0], nb, 1e-8)), what     # cost, step by step
    assert np.allclose(tg[:n, 5], tr[:n, 5], rtol=1e-8, atol=0), what                              # trust-region radius
    assert np.array_equal(tg[:n, 6:], tr[:n, 6:]), what                                            # valid, successful
    return sg


@pytest.mark.parametrize("huber", [0.01, 1.0, 1e6])
@pytest.mark.parametrize("inner", [0, 1, 2, 7, 8, 12])
def test_solve_at_inner_iters_and_huber(aloam, orc, inner, huber):
    ctx = aloam.Aloam(n_scans=64, max_points=20000, inner_iters=inner, huber=huber)
    try:
        for name, blocks, x0 in _lm_problems(orc):
            _compare_solve(ctx, orc, blocks, x0, inner, huber, (name, inner, huber))
            if inner in (0, 7) and name in ("golden", "iterations", "rejected"):
                # the emulated one-rank world: per-evaluation kernels (a fixed schedule of 1 + inner_iters evaluations) and the
                # peer mailbox; "rejected" needs all 7 iterations.  Bars of DESIGN's emulated-rank row: identical stats, 1e-15.
                ref = ctx.solve(blocks, x0)
                for ex in (1, 2):
                    ctx.debug_shard_emulate(0, 1, ex)
                    got = ctx.solve(blocks, x0)
                    ctx.debug_shard_emulate(0, 0)
                    dx = float(np.abs(got[0] - ref[0]).max())
                    assert got[1]["termination"] == ref[1]["termination"], (name, inner, ex, got[1], ref[1])
                    for k in ("num_iterations", "num_successful"):
                        assert got[1][k] == ref[1][k], (name, inner, ex, k, got[1][k], ref[1][k])
                    assert dx <= 1e-15 * max(1.0, float(np.abs(ref[0]).max())), (name, inner, ex, dx)
                    assert got[2].shape == ref[2].shape and np.array_equal(got[2][:, 6:], ref[2][:, 6:]), (name, inner, ex)
    finally:
        ctx.close()


# ---------------------------------------------------------------------------------------------------------------- chains


SETTINGS = {"nearby1": dict(nearby_scan=1.0), "nearby4": dict(nearby_scan=4.0), "nearby_inf": dict(nearby_scan=math.inf),
            "thr9": dict(dist_sq_thresh=9.0), "thr100": dict(dist_sq_thresh=100.0), "outer1": dict(outer_iters=1),
            "outer3": dict(outer_iters=3), "outer4": dict(outer_iters=4), "inner1": dict(inner_iters=1), "inner8": dict(inner_iters=8),
            "huber0.5": dict(huber=0.5)}


def _odom(orc, cfg, distortion=0):
    return orc.Odometry(distortion=bool(distortion), dist_sq_thresh=cfg.get("dist_sq_thresh", 25.0), nearby_scan=cfg.get("nearby_scan", 2.5))


def _reg_kw(cfg):
    return dict(outer=cfg.get("outer_iters", 2), max_iters=cfg.get("inner_iters", 4), huber=cfg.get("huber", 0.1))


def _oracle_chain(orc, feats, cfg):
    """world poses and per-scan correspondence counts of the oracle chain run with the setting"""
    od = _odom(orc, cfg)
    q, t = IDENT_Q.copy(), ZERO_T.copy(); qw, tw = q.copy(), t.copy()
    poses, counts = [], []
    for k, f in enumerate(feats):
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t, **_reg_kw(cfg))
            qw, tw = orc.integrate_pose(qw, tw, q, t)
            counts.append((info["corner_corr"], info["plane_corr"]))
        od.set_last(f.less_sharp, f.less_flat)
        poses.append(np.concatenate([qw, tw]))
    return np.array(poses), counts


@pytest.mark.parametrize("sensor", ["VLP-16", "HDL-64"])
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_chains_and_streams_at_a_setting(aloam, orc, synth, sensor, setting):
    cfg = SETTINGS[setting]
    ns, n, lanes = synth.SENSORS[sensor][0], 5, 4
    trajs = [[_features(orc, synth, sensor, t, k) for k in range(n)] for t in range(lanes)]
    raws = [[np.ascontiguousarray(r) for r, _ in tr] for tr in trajs]
    maxpts = max(r.shape[0] for tr in raws for r in tr) + 1024
    ctx = aloam.Aloam(n_scans=ns, max_points=maxpts, **cfg)
    batch = aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=lanes, **cfg)
    worst = 0.0
    try:
        ref, counts = _oracle_chain(orc, [f for _, f in trajs[0]], cfg)
        per_scan = []
        for k, raw in enumerate(raws[0]):
            gq, gt, st = ctx.scan_to_pose(raw)
            per_scan.append(np.concatenate([gq, gt]))
            if k > 0:
                assert (st["n_corner_corr"], st["n_plane_corr"]) == counts[k - 1], (k, st, counts[k - 1])
        per_scan = np.array(per_scan)
        worst = max(float(np.abs(per_scan[:, 4:] - ref[:, 4:]).max()), max(rot_angle(per_scan[k, :4], ref[k, :4]) for k in range(n)))
        assert worst < BAR, worst
        assert float(np.abs(ref[:, 4:]).max()) > 0.05
        solo = []
        for tr in raws:
            ctx.reset_odometry()
            p, _ = ctx.scan_stream([r.ctypes.data for r in tr], [len(r) for r in tr], False)
            solo.append(p)
        assert np.array_equal(solo[0], per_scan), np.abs(solo[0] - per_scan).max()
        ptrs = np.array([[raws[b][k].ctypes.data for b in range(lanes)] for k in range(n)], np.uint64)
        cnts = np.array([[len(raws[b][k]) for b in range(lanes)] for k in range(n)], np.int32)
        got = batch.scan_stream_batch(ptrs, cnts, False)
        for b in range(lanes):
            assert np.array_equal(got[:, b], solo[b]), (b, np.abs(got[:, b] - solo[b]).max())
    finally:
        ctx.close(); batch.close()
    print("%s %s: worst pose deviation from the oracle chain %.2e" % (sensor, setting, worst))


MAP_SETTINGS = {"outer1": dict(outer_iters=1, inner_iters=8, huber=0.5), "outer3": dict(outer_iters=3, inner_iters=8, huber=0.5)}


@pytest.mark.parametrize("setting", list(MAP_SETTINGS))
def test_mapped_stream_at_a_setting(aloam, orc, synth, setting):
    cfg = MAP_SETTINGS[setting]
    ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
    scans = [np.ascontiguousarray(s) for s in R.traj(synth, 0, 6)]
    dev = R.to_device(scans)
    c = aloam.Aloam(n_scans=ns, max_points=R.maxn([scans]) + 1024, max_ring_points=4096, max_map_points=400000, **cfg)
    try:
        odom, mp = c.scan_stream_mapped(np.array([d.data_ptr() for d in dev], np.uint64), np.array([s.shape[0] for s in scans]), True)
    finally:
        c.close()
    od, cm = _odom(orc, cfg), orc.CubeMap()
    q, t = IDENT_Q.copy(), ZERO_T.copy(); qw, tw = q.copy(), t.copy()
    ro, rm = [], []
    optimised = 0
    for k, raw in enumerate(scans):
        f = orc.Features(raw, ns, mr)
        if k > 0:
            q, t, _ = od.register(f.sharp, f.flat, q, t, **_reg_kw(cfg))
            qw, tw = orc.integrate_pose(qw, tw, q, t)
        od.set_last(f.less_sharp, f.less_flat)
        ro.append(np.concatenate([qw, tw]))
        pose, info = cm.step(f.less_sharp, f.less_flat, qw, tw, line_res, plane_res, outer=cfg["outer_iters"], max_iters=cfg["inner_iters"],
                             huber=cfg["huber"])
        optimised += info["optimised"]
        rm.append(pose)
    assert optimised >= 4
    for got, ref, what in ((odom, np.array(ro), "odometry"), (mp, np.array(rm), "map")):
        dt, dr = R.deviation(got, ref)
        assert dt < BAR and dr < BAR, (setting, what, dt, dr)


@pytest.mark.parametrize("setting", list(MAP_SETTINGS))
def test_localising_lane_at_a_setting(aloam, orc, synth, setting):
    """a lane localising on a prior map mapped under the same setting, from 0.2 m and 2 degrees off, against the frozen oracle"""
    import pyfrozen
    cfg = MAP_SETTINGS[setting]
    W = TL._world(aloam, synth, "VLP-16", **cfg)
    n = len(W["scans"])
    init = TL._perturbed(np.array([0, 0, 0, 1.0, 0, 0, 0]), 0.2, 2.0)
    c = TL._localiser(aloam, W, 1, **cfg)
    try:
        c.lane_localise(0, *init)
        o, m = TL._call(c, 1, {0: TL._entries(W["dev"], 0, n)})[0]
        st = c.mapper_state(0)
    finally:
        c.close()
    blob = W["blob"].tobytes()
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    off = 256 + 16 * (nls + nlf)
    counts = np.frombuffer(blob, np.int32, 2 * 4851, off + 592).reshape(2, 4851)
    points = np.frombuffer(blob, np.float32, offset=off + 39424).reshape(-1, 4)
    frozen = pyfrozen.FrozenMap.from_export(struct.unpack_from("<3i", blob, off), counts, points)
    ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
    feats = [orc.Features(raw, ns, mr) for raw in W["scans"]]
    odom, _ = _oracle_chain(orc, feats, cfg)
    dt, dr = R.deviation(o, odom)
    assert dt < BAR and dr < BAR, ("odometry", dt, dr)
    loc = pyfrozen.Localiser(frozen, *init)
    ref = []
    for k, f in enumerate(feats):
        pose, info = loc.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], line_res, plane_res, outer=cfg["outer_iters"],
                              max_iters=cfg["inner_iters"], huber=cfg["huber"])
        assert info["optimised"] == 1
        ref.append(pose)
    dt, dr = R.deviation(m, np.array(ref))
    assert dt < BAR and dr < BAR, ("map", dt, dr)
    assert st["valid"] == loc.valid and st["centre"] == frozen.centre


def test_snapshot_under_a_non_default_association(aloam, synth):
    """a lane saved at nearby_scan 3 / dist_sq_thresh 16 continues bit-identical in a context of that configuration; a default
    context refuses the snapshot"""
    cfg = dict(nearby_scan=3.0, dist_sq_thresh=16.0)
    scans = R.traj(synth, 1, 8)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    whole = TL._ctx(aloam, M, 1, **cfg)
    first = TL._ctx(aloam, M, 1, **cfg)
    second = TL._ctx(aloam, M, 2, **cfg)
    default = TL._ctx(aloam, M, 1)
    try:
        o_all, m_all = TL._call(whole, 1, {0: TL._entries(dev, 0, 8)})[0]
        o1, m1 = TL._call(first, 1, {0: TL._entries(dev, 0, 4)})[0]
        blob = first.lane_save(0)
        second.lane_restore(1, blob)
        o2, m2 = TL._call(second, 2, {1: [(d.data_ptr(), d.shape[0], TL.SCAN) for d in dev[4:8]]})[1]
        assert np.array_equal(np.concatenate([o1, o2]), o_all) and np.array_equal(np.concatenate([m1, m2]), m_all)
        TL._expect(aloam, -11, lambda: default.lane_restore(0, blob))
    finally:
        for c in (whole, first, second, default):
            c.close()
