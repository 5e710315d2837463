"""GPU: per-row records of the mapped stream calls (aloam_set_map_rows, aloam_map_rows).  Checked here: every mapping row against
aloam_mapper_step replayed on a second context (stats bit for bit, flags, error word) and its sizes against the oracle's frame;
localising rows against the mapping frame of a scratch context restored from the prior snapshot, their sizes against the frozen
oracle and their scores integer-equal to the oracle's score at the row's map pose; START rows of lanes armed with relocalisation
results against those results; the lost-track scenario of tests/track_cases.py end to end, with recovery through
aloam_prior_relocalise; overflow attribution to the row that overflowed; nothing else changes with recording on; refusals."""
import ctypes as C
import struct

import numpy as np
import pytest

import lane_refs as R
import reloc_cases as RC
import track_cases as TC

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
IDLE, SCAN, START = 0, 1, 2
IDENT7 = np.array([0, 0, 0, 1.0, 0, 0, 0])
STAT_KEYS = ("n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps", "flags", "init_cost", "final_cost")


def _ctx(aloam, maxpts, batch=1, ns=16, **cfg):
    kw = {"max_ring_points": 4096, "max_map_points": 400000, **cfg}
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, **kw)


def _entries(dev, i0, i1):
    return [(d.data_ptr(), d.shape[0], START if i == i0 else SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def _grid(batch, lanes):
    steps = max(len(e) for e in lanes.values())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for lane, entries in lanes.items():
        for k, (p, n, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    return ptrs, counts, ops


def _call(ctx, batch, lanes, mapped=True, rows=True):
    """one aloam_scan_stream_lanes call; lanes = {lane: entries} -> (odometry (steps, batch, 7), map poses, rows or None)"""
    ptrs, counts, ops = _grid(batch, lanes)
    o, m = ctx.scan_stream_lanes(ptrs, counts, ops, True, mapped=mapped)
    return o, m, (ctx.map_rows(ops.size) if rows else None)


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def _row(rows, r):
    return {k: v[r] for k, v in rows.items()}


def _same_stats(row, st, what, flag_mask=-1):
    for k in STAT_KEYS:
        a, b = (row[k] & flag_mask, st[k] & flag_mask) if k == "flags" else (row[k], st[k])
        assert a == b, (what, k, row[k], st[k])
    assert list(row["termination"]) == list(st["termination"]), (what, row["termination"], st["termination"])


def _mapper_step(aloam, c, f, odom):
    """aloam_mapper_step through the C ABI: (return code, pose, stats) -- the stats of a frame that returns ALOAM_ERR_CAPACITY too"""
    a, ka = aloam._view(f["less_sharp"])
    b, kb = aloam._view(f["less_flat"])
    qo, to = np.ascontiguousarray(odom[:4]), np.ascontiguousarray(odom[4:])
    q, t, st = np.zeros(4), np.zeros(3), aloam.Stats()
    rc = aloam.lib().aloam_mapper_step(c._h, a, b, aloam._dp(qo), aloam._dp(to), aloam._dp(q), aloam._dp(t), C.byref(st))
    return rc, np.concatenate([q, t]), st.as_dict()


def _replay(aloam, feats, odom, kinds, rows, cfg, what, setup=None):
    """a trajectory's mapped rows against aloam_mapper_step on a fresh context with the same config, fed the same clouds and odometry
    poses: pose bit for bit, stats field for field (costs bit for bit), flags, the error word's bit 0 against the frame's return
    code.  Returns the replay's stats of the mapped rows."""
    c = aloam.Aloam(**cfg)
    c.mapper_reset()
    if setup:
        setup(c)
    out = []
    for j, (f, kind) in enumerate(zip(feats, kinds)):
        if kind != aloam.ROW_MAPPED:
            continue
        rc, pose, st = _mapper_step(aloam, c, f, odom[j])
        row = _row(rows, j)
        assert rc in (0, ERR_CAPACITY), rc
        assert bool(row["err"] & 1) == (rc == ERR_CAPACITY), (what, j, row["err"], rc)
        _same_stats(row, st, (what, j))
        out.append((j, pose, st))
    c.close()
    return out


def _cfg(ctx):
    cfg = ctx.cfg
    return {k: getattr(cfg, k) for k, _ in type(cfg)._fields_}


_WORLD = {}


def _world(aloam, synth, sensor="VLP-16"):
    """as tests/test_gpu_relocalise.py: scans of trajectory 0, the snapshot of the lane that mapped the first N_MAP of them, its map
    poses, the prior map as the oracle's FrozenMap and scorer, every scan's clouds from the device's feature extraction"""
    if sensor not in _WORLD:
        import pyfrozen
        ns = synth.SENSORS[sensor][0]
        scans = R.traj(synth, 0, RC.N_MAP + 6, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)
        M = R.maxn([scans]) + 1024
        dev = R.to_device(scans)
        c = _ctx(aloam, M, 1, ns)
        _, m, _ = _call(c, 1, {0: _entries(dev, 0, RC.N_MAP)}, rows=False)
        blob = c.lane_save(0)
        c.close()
        b = blob.tobytes()
        nls, nlf = struct.unpack_from("<ii", b, 28)
        S = 256 + 16 * (nls + nlf)
        counts = np.frombuffer(b, np.int32, 2 * 4851, S + 592).reshape(2, 4851)
        points = np.frombuffer(b, np.float32, offset=S + 39424).reshape(-1, 4)
        frozen = pyfrozen.FrozenMap.from_export(struct.unpack_from("<3i", b, S), counts, points)
        fx = _ctx(aloam, M, 1, ns)
        feats = [fx.extract_features(s) for s in scans]
        fx.close()
        _WORLD[sensor] = {"scans": scans, "dev": dev, "M": M, "ns": ns, "blob": blob, "map": m[:, 0], "frozen": frozen,
                          "scorer": RC.FrozenScorer(frozen), "feats": feats, "res": synth.SENSORS[sensor][3:5]}
    return _WORLD[sensor]


def _localiser(aloam, W, batch=1):
    c = _ctx(aloam, W["M"], batch, W["ns"])
    c.prior_map_load(W["blob"])
    return c


# five lanes: staggered STARTs, a trajectory that ends and a lane that starts again, idle lanes at either end of the call
def _schedule(dev, n):
    return {0: _entries(dev, 0, n),
            1: [(0, 0, IDLE)] * 2 + _entries(dev, 1, n - 1),
            2: _entries(dev, 3, 3 + n // 2) + [(0, 0, IDLE)] + _entries(dev, 0, n - n // 2 - 1),
            3: [(0, 0, IDLE)] * (n - 4) + _entries(dev, 2, 6),
            4: [(0, 0, IDLE)] * n}


@pytest.mark.parametrize("sensor,skip", [("VLP-16", 1), ("HDL-32", 1), ("VLP-16", 3)])
def test_mapping_rows_equal_the_mapper_step_replay_and_the_oracle(aloam, synth, orc, sensor, skip):
    """a 5-lane call with staggered STARTs, IDLEs and (skip 3) skipped rows: kinds follow the schedule, every mapped row equals
    aloam_mapper_step replayed with the lane's clouds and odometry poses, and its sizes equal the oracle's frame over the same
    trajectory"""
    ns, _, mr, line_res, plane_res = synth.SENSORS[sensor]
    n = 9
    scans = R.traj(synth, 0, n, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)
    M = R.maxn([scans]) + 1024
    dev = R.to_device(scans)
    c = _ctx(aloam, M, 5, ns, mapping_skip_frame=skip)
    c.set_map_rows(True)
    sched = _schedule(dev, n)
    ptrs, counts, ops = _grid(5, sched)
    odom, mp, rows = _call(c, 5, sched)
    ids = {d.data_ptr(): i for i, d in enumerate(dev)}
    cfg = {**_cfg(c), "max_batch": 1}
    for lane in range(5):
        # the lane's trajectories: runs from a START to the step before the next START or IDLE
        runs, cur = [], None
        for k in range(ops.shape[0]):
            op = ops[k, lane]
            if op == START:
                cur = []
                runs.append(cur)
            if op == IDLE:
                cur = None
            if cur is not None:
                cur.append(k)
        for k in range(ops.shape[0]):
            r = k * 5 + lane
            if ops[k, lane] == IDLE:
                assert rows["kind"][r] == aloam.ROW_IDLE and all(rows[f][r].sum() == 0 for f in rows if f != "kind"), (lane, k)
        for run in runs:
            kinds = [aloam.ROW_MAPPED if j % skip == 0 else aloam.ROW_SKIPPED for j in range(len(run))]
            got = [rows["kind"][k * 5 + lane] for k in run]
            assert got == kinds, (lane, got, kinds)
            sub = {f: v[[k * 5 + lane for k in run]] for f, v in rows.items()}
            for j, k in enumerate(run):
                if kinds[j] == aloam.ROW_SKIPPED:
                    assert sub["score"][j] == -1 and sub["n_score"][j] == 0 and sub["flags"][j] == 0 and sub["lm_iters"][j] == 0
                else:
                    assert sub["score"][j] == -1 and sub["n_score"][j] == 0
            raw = [scans[ids[int(ptrs[k, lane])]] for k in run]
            feats = []
            fx = aloam.Aloam(n_scans=ns, max_points=M)
            for s in raw:
                feats.append(fx.extract_features(s))
            fx.close()
            rep = _replay(aloam, feats, odom[run, lane], kinds, sub, cfg, (sensor, lane))
            for j, pose, _ in rep:
                assert np.array_equal(pose, mp[run[j], lane]), (lane, j)
            # sizes against the oracle's frame over the same trajectory (oracle features and odometry)
            od, cm = orc.Odometry(), orc.CubeMap()
            q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
            for j, s in enumerate(raw):
                f = orc.Features(s, ns, mr)
                if j > 0:
                    q, t, _ = od.register(f.sharp, f.flat, q, t)
                    qw, tw = orc.integrate_pose(qw, tw, q, t)
                od.set_last(f.less_sharp, f.less_flat)
                if kinds[j] != aloam.ROW_MAPPED:
                    continue
                _, info = cm.step(f.less_sharp, f.less_flat, qw, tw, line_res, plane_res)
                got = (sub["n_valid"][j], *sub["n_sub"][j], *sub["n_stack"][j], not sub["flags"][j] & aloam.FLAG_MAP_TOO_THIN)
                ref = (info["n_valid"], info["corner_from_map"], info["surf_from_map"], info["corner_stack"], info["surf_stack"], bool(info["optimised"]))
                assert got == ref, (sensor, lane, j, got, ref)
    c.close()


def _patched(W, T):
    """the prior snapshot with its T_wmap_wodom replaced by T"""
    blob = bytearray(W["blob"].tobytes())
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    S = 256 + 16 * (nls + nlf)
    struct.pack_into("<4d", blob, S + 536, *T[:4])
    struct.pack_into("<3d", blob, S + 568, *T[4:])
    return np.frombuffer(bytes(blob), np.uint8)


@pytest.mark.parametrize("inlier_sq,max_pts", [(TC.ISQ, TC.PTS), (1.0, 1 << 20)])
def test_localising_rows_equal_the_mapping_frame_and_the_oracle_score(aloam, synth, inlier_sq, max_pts):
    """frame j of a localising lane: its row equals aloam_mapper_step on a scratch context restored from the prior snapshot with the
    lane's T_wmap_wodom; its sizes equal the frozen oracle's frame; its score equals the oracle's score at the row's map pose
    (max_pts = 2^20: more scoring points than the stacks hold)"""
    import pyfrozen
    W = _world(aloam, synth)
    s0, n = 2, 6
    loc = _localiser(aloam, W)
    loc.set_map_rows(True, inlier_sq, max_pts)
    T = W["map"][s0] + [0, 0, 0, 0, 0.2, -0.1, 0]
    loc.lane_localise(0, T[:4], T[4:])
    n2 = 0.0
    for v in T[:4]:   # the arming's normalisation: q / sqrt(q . q), summed in index order
        n2 += float(v) * float(v)
    T[:4] = T[:4] / np.sqrt(n2)
    oracle = pyfrozen.Localiser(W["frozen"], T[:4], T[4:])
    scratch = _ctx(aloam, W["M"])
    entries = _entries(W["dev"], s0, s0 + n)
    for j in range(n):
        o, m, rows = _call(loc, 1, {0: [entries[j]]})
        row = _row(rows, 0)
        assert row["kind"] == aloam.ROW_LOCALISED and row["err"] == 0
        scratch.lane_restore(0, _patched(W, T))
        f = W["feats"][s0 + j]
        rc, pose, st = _mapper_step(aloam, scratch, f, o[0, 0])
        assert rc == 0 and np.array_equal(pose, m[0, 0]), j
        # the mapping frame also inserts the scan into the restored store, whose full slabs raise ALOAM_FLAG_CUBE_OVERFLOW: a
        # localising frame inserts nothing
        _same_stats(row, st, j, ~aloam.FLAG_CUBE_OVERFLOW)
        assert not row["flags"] & aloam.FLAG_CUBE_OVERFLOW
        _, info = oracle.step(f["less_sharp"], f["less_flat"], o[0, 0, :4], o[0, 0, 4:], *W["res"])
        assert (row["n_valid"], *row["n_sub"], *row["n_stack"]) == (info["n_valid"], info["corner_from_map"], info["surf_from_map"],
                                                                    info["corner_stack"], info["surf_stack"]), (j, row, info)
        sp = RC.scoring_points(f["less_sharp"], f["less_flat"], max_pts, *W["res"])
        assert row["n_score"] == len(sp[0]) + len(sp[1]) and (max_pts < 1 << 20 or row["n_score"] == sum(row["n_stack"]))
        ref = W["scorer"].score(f["less_sharp"], f["less_flat"], m[0, 0][None], inlier_sq, max_pts, *W["res"], normalise=False)[0]
        assert row["score"] == ref and row["score"] > 0, (j, row["score"], ref)
        s = loc.mapper_state(0)
        T = np.concatenate([s["q_wmap_wodom"], s["t_wmap_wodom"]])
    for c in (loc, scratch):
        c.close()


def test_start_rows_of_lanes_armed_with_relocalise_results(aloam, synth):
    W = _world(aloam, synth)
    s = 5
    f = W["feats"][s]
    hyps = RC.search_grid(aloam, W["map"][s], offset=(0.2, 0.1, 0), half=2.0, step=1.0, n_yaw=8)
    K = 8
    c = _localiser(aloam, W, K)
    res, _ = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=K)
    c.set_map_rows(True, 0.5, 256)
    for l, r in enumerate(res):
        c.lane_localise(l, hyps[r["hyp"], :4], hyps[r["hyp"], 4:])
    _, m, rows = _call(c, K, {l: _entries(W["dev"], s, s + 1) for l in range(K)})
    for l, r in enumerate(res):
        assert rows["kind"][l] == aloam.ROW_LOCALISED
        assert rows["score"][l] == r["refined_score"], (l, rows["score"][l], r["refined_score"])
        assert np.array_equal(m[0, l], r["pose"]), l
    c.close()


def test_a_lost_lane_is_seen_relocalised_and_tracks_again(aloam, synth):
    """lane 0 armed at the true map pose, lane 1 armed 45 degrees and 3 m off, lane 2 armed off the map: lane 1's rows fall below
    LOST_RATIO, lane 2's are thin with zero stats.  Relocalising lane 1 on its next scan from a search around its last map pose and
    re-arming it brings it back onto lane 0's poses and above TRACK_RATIO."""
    W = _world(aloam, synth)
    s0, s1, end = TC.START, TC.START + 6, len(W["dev"])
    c = _localiser(aloam, W, 3)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    true = W["map"][s0]
    for lane, init in enumerate((true, TC.mis_armed(true), TC.off_map(true))):
        c.lane_localise(lane, init[:4], init[4:])
    _, m, rows = _call(c, 3, {l: _entries(W["dev"], s0, s1) for l in range(3)})
    sc, n = rows["score"].reshape(-1, 3), rows["n_score"].reshape(-1, 3)
    assert (sc[:, 0] > TC.TRACK_RATIO * n[:, 0]).all(), (sc[:, 0], n[:, 0])
    assert (sc[:, 1] < TC.LOST_RATIO * n[:, 1]).all(), (sc[:, 1], n[:, 1])
    thin = rows["flags"].reshape(-1, 3)[:, 2]
    assert (thin == aloam.FLAG_MAP_TOO_THIN).all() and (sc[:, 2] == 0).all() and (n[:, 2] > 0).all()
    for k in ("lm_iters", "n_corner_corr", "n_plane_corr", "accepted_steps", "init_cost", "final_cost"):
        assert (rows[k].reshape(-1, 3)[:, 2] == 0).all(), k
    assert (rows["termination"].reshape(-1, 3, 4)[:, 2] == 0).all()
    # relocalise lane 1 on its next scan from a search around its last (wrong) map pose, re-arm it and START it on that scan
    f = W["feats"][s1]
    hyps = RC.search_grid(aloam, m[-1, 1], offset=(0.0, 0.0, 0.0))
    res, _ = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=TC.ISQ, max_score_points=TC.PTS, refine=4)
    c.lane_localise(1, res[0]["pose"][:4], res[0]["pose"][4:])
    _, m2, rows2 = _call(c, 3, {0: [(p, n_, SCAN) for p, n_, _ in _entries(W["dev"], s1, end)], 1: _entries(W["dev"], s1, end)})
    assert rows2["score"].reshape(-1, 3)[0, 1] == res[0]["refined_score"]
    dt, dr = R.deviation(m2[1:, 1], m2[1:, 0])
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    sc2, n2 = rows2["score"].reshape(-1, 3), rows2["n_score"].reshape(-1, 3)
    assert (sc2[:, 1] > TC.TRACK_RATIO * n2[:, 1]).all(), (sc2[:, 1], n2[:, 1])
    assert (rows2["kind"].reshape(-1, 3)[:, 2] == aloam.ROW_IDLE).all()
    c.close()


def test_cube_overflow_is_on_the_row_that_overflowed(aloam, synth):
    """a submap truncated at a small cfg.max_map_points raises ALOAM_FLAG_CUBE_OVERFLOW (error bit 3) on exactly the rows where the
    mapper_step replay reports it"""
    scans = R.traj(synth, 0, 8)
    M = R.maxn([scans]) + 1024
    dev = R.to_device(scans)
    c = _ctx(aloam, M, 1, max_map_points=4000)
    c.set_map_rows(True)
    odom, mp, rows = _call(c, 1, {0: _entries(dev, 0, 8)})
    fx = aloam.Aloam(n_scans=16, max_points=M)
    feats = [fx.extract_features(s) for s in scans]
    fx.close()
    rep = _replay(aloam, feats, odom[:, 0], [aloam.ROW_MAPPED] * 8, rows, _cfg(c), "truncated")
    flagged = [bool(st["flags"] & aloam.FLAG_CUBE_OVERFLOW) for _, _, st in rep]
    assert any(flagged) and not all(flagged), flagged
    assert [bool(e & 8) for e in rows["err"]] == flagged
    c.close()


def test_key_overflow_is_on_the_row_that_overflowed(aloam, synth):
    """tests/test_gpu_cubemap.py's cube beyond the sort key's width, put into the store before the call: the call returns
    ALOAM_ERR_CAPACITY, the rows stay readable and error bit 0 is set on exactly the rows whose replayed frame returns it"""
    from test_gpu_cubemap import W as CW, H as CH, _overflow_box
    raws = [synth.scan("VLP-16", k, n_az=900) for k in range(3)]
    maxn = max(r.shape[0] for r in raws)
    box = _overflow_box(np.random.default_rng(59), (87.113, 87.113, 37.113))
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    cfg = dict(n_scans=16, max_points=maxn + 1024, max_map_points=400000, line_res=0.02, plane_res=0.02)
    c = aloam.Aloam(**cfg)
    c.mapper_reset()
    _expect(aloam, ERR_CAPACITY, lambda: c.mapper_step(empty, box, ident, np.zeros(3)))
    c.set_map_rows(True)
    ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
    _expect(aloam, ERR_CAPACITY, lambda: c.scan_stream_mapped(ptrs, counts, False))
    assert 12 + CW * 12 + CW * CH * 6 in c.mapper_state()["valid"]
    rows = c.map_rows(3)
    assert (rows["kind"] == aloam.ROW_MAPPED).all()
    c.close()
    c = aloam.Aloam(**cfg)   # the odometry poses of the mapped call, bit for bit
    odom, _ = c.scan_stream(ptrs, counts, False)
    feats = [c.extract_features(r) for r in raws]
    c.close()
    rep = _replay(aloam, feats, odom, [aloam.ROW_MAPPED] * 3, rows, cfg, "key overflow",
                  setup=lambda s: _expect(aloam, ERR_CAPACITY, lambda: s.mapper_step(empty, box, ident, np.zeros(3))))
    assert len(rep) == 3 and (rows["err"] & 1).any()


def _launches(fn, c):
    a = c.launch_count()
    out = fn()
    return out, c.launch_count() - a


def test_recording_changes_nothing_else(aloam, synth):
    """a mapping lane (skip 2), a localising lane and an odometry-only lane; the same schedule with recording off, rows only, rows and
    scores, and off again after on: identical odometry and map poses, registered clouds, stores and prior map; launches equal with
    recording off, +1 per frame with rows and +1 more per localising frame with scores; odometry-only calls unaffected; a relocalise
    call between stream calls answers the same"""
    import torch
    W = _world(aloam, synth)
    f = W["feats"][5]
    hyps = RC.search_grid(aloam, W["map"][5], offset=(0.2, 0.1, 0), half=1.0, step=1.0, n_yaw=4)
    init = W["map"][2]
    out = []
    for mode in ("off", "rows", "score", "on-off"):
        c = _ctx(aloam, W["M"], 3, W["ns"], mapping_skip_frame=2)
        store = aloam.snapshot_store_clouds(W["blob"])   # (a snapshot taken at skip 1 does not load at skip 2)
        c.prior_map_build(store["corner"], store["surf"], store["centre"])
        sink = torch.zeros((20 * W["M"], 4), dtype=torch.float32, device="cuda")
        c.set_registered_sink(sink)
        if mode == "rows":
            c.set_map_rows(True)
        elif mode == "score":
            c.set_map_rows(True, TC.ISQ, TC.PTS)
        elif mode == "on-off":
            c.set_map_rows(True, TC.ISQ, TC.PTS)
            c.set_map_rows(False)
        rec = mode in ("rows", "score")
        res = []
        o, n0 = _launches(lambda: _call(c, 3, {2: _entries(W["dev"], 0, 3)}, mapped=False, rows=False), c)
        res.append(("odo", o[0], n0))
        reloc_a = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=2)
        c.lane_localise(1, init[:4], init[4:])
        for lanes in ({0: _entries(W["dev"], 0, 5), 1: _entries(W["dev"], 2, 7)},
                      {0: [(p, n, SCAN) for p, n, _ in _entries(W["dev"], 5, 9)], 1: [(p, n, SCAN) for p, n, _ in _entries(W["dev"], 7, 11)]}):
            (o, m, rows), n1 = _launches(lambda: _call(c, 3, lanes, rows=rec), c)
            begin, count = c.registered_rows(o.shape[0] * 3)
            clouds = [sink[b:b + k].cpu().numpy().copy() for b, k in zip(begin, count)]
            res.append(("map", o, m, clouds, n1, rows))
            if not rec:
                _expect(aloam, ERR_STATE, lambda: c.map_rows(o.shape[0] * 3))
        reloc_b = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=2)
        o, n2 = _launches(lambda: _call(c, 3, {2: _entries(W["dev"], 3, 6)}, mapped=False, rows=False), c)
        res.append(("odo", o[0], n2))
        if rec:   # an odometry-only call leaves the last mapped call's rows readable
            assert c.map_rows(res[-2][1].shape[0] * 3)["kind"].size == res[-2][1].shape[0] * 3
        store = c.mapper_export(aloam.EXPORT_MAP, 0).tobytes()
        prior = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes()
        out.append((mode, res, reloc_a, reloc_b, store, prior))
        c.close()
    base = out[0]
    for mode, res, ra, rb, store, prior in out[1:]:
        assert store == base[4] and prior == base[5], mode
        for (a, b) in zip(res, base[1]):
            if a[0] == "odo":
                assert np.array_equal(a[1], b[1], equal_nan=True) and a[2] == b[2], mode
                continue
            _, o, m, clouds, n, rows = a
            assert np.array_equal(o, b[1], equal_nan=True) and np.array_equal(m, b[2], equal_nan=True), mode
            assert all(np.array_equal(x, y) for x, y in zip(clouds, b[3])), mode
            frames = loc_frames = 0
            if rows is not None:
                kinds = rows["kind"].reshape(-1, 3)
                frames = sum(int(((k == aloam.ROW_MAPPED).any())) + int((k == aloam.ROW_LOCALISED).any()) for k in kinds)
                loc_frames = int((kinds == aloam.ROW_LOCALISED).any(axis=1).sum())
                assert (kinds[:, 0] != aloam.ROW_LOCALISED).all() and (kinds[:, 1] != aloam.ROW_MAPPED).all()
                assert ((kinds == aloam.ROW_SKIPPED).any()) and (kinds[:, 2] == aloam.ROW_IDLE).all()
                scored = rows["score"].reshape(-1, 3)[kinds == aloam.ROW_LOCALISED]
                assert (scored > 0).all() if mode == "score" else (scored == -1).all(), mode
            assert n == b[4] + frames + (loc_frames if mode == "score" else 0), (mode, n, b[4], frames, loc_frames)
        for x, y in ((ra, base[2]), (rb, base[3])):
            assert np.array_equal(x[1], y[1]) and all(np.array_equal(p["pose"], q["pose"]) for p, q in zip(x[0], y[0])), mode


def test_refusals_leave_the_context_as_it_was(aloam, synth):
    W = _world(aloam, synth)
    c = _ctx(aloam, W["M"], 2, W["ns"])
    lib = aloam.lib()
    row = (aloam.MapRow * 4)()
    assert lib.aloam_map_rows(c._h, row, 2) == ERR_STATE                 # before any mapped stream call
    for on, isq, pts in ((2, 1.0, 0), (-1, 1.0, 0), (1, 1.0, -1), (1, 0.0, 16), (1, -1.0, 16), (1, 1.0001, 16), (1, float("nan"), 16),
                         (0, 2.0, 16)):
        assert lib.aloam_set_map_rows(c._h, on, isq, pts) == ERR_INVALID_ARG, (on, isq, pts)
    assert lib.aloam_set_map_rows(c._h, 1, 5.0, 0) == 0                  # no scoring: inlier_sq is not read
    _call(c, 2, {0: _entries(W["dev"], 0, 2)}, rows=False)
    rows = c.map_rows(4)
    assert lib.aloam_map_rows(c._h, None, 4) == ERR_INVALID_ARG
    for n in (3, 5, 0):
        assert lib.aloam_map_rows(c._h, row, n) == ERR_INVALID_ARG, n
    again = c.map_rows(4)
    assert all(np.array_equal(rows[k], again[k]) for k in rows)
    # a mapped call with recording off: nothing to read
    c.set_map_rows(False)
    _call(c, 2, {0: [(p, n, SCAN) for p, n, _ in _entries(W["dev"], 2, 3)]}, rows=False)
    assert lib.aloam_map_rows(c._h, row, 2) == ERR_STATE
    # a call that fails with an empty scan: nothing to read
    c.set_map_rows(True)
    ptrs, counts, ops = _grid(2, {0: _entries(W["dev"], 0, 1)})
    counts[0, 0] = 0
    with pytest.raises(aloam.AloamError):
        c.scan_stream_lanes(ptrs, counts, ops, True)
    assert lib.aloam_map_rows(c._h, row, 2) == ERR_STATE
    # sharded ranks and emulating contexts refuse, and emulation turns recording off
    assert lib.aloam_debug_shard_emulate(c._h, 0, 2, 0, 0) == 0
    assert lib.aloam_set_map_rows(c._h, 1, 1.0, 0) == ERR_STATE and lib.aloam_set_map_rows(c._h, 0, 1.0, 0) == ERR_STATE
    assert lib.aloam_debug_shard_emulate(c._h, 0, 0, 0, 0) == 0
    c.reset_odometry()
    _call(c, 2, {0: _entries(W["dev"], 0, 1)}, rows=False)
    assert lib.aloam_map_rows(c._h, row, 2) == ERR_STATE               # recording was turned off by the emulation
    c.close()
