"""GPU: relocalisation against a prior map (aloam_prior_relocalise).  Hypotheses of one scan are scored against the whole prior map
on the device, the best K are refined by one localising frame each.  Checked here: every coarse score integer-equal to the
oracle's (tests/reloc_cases.py) on VLP-16 and HDL-32 worlds, a crafted map at the d^2 edges, far and single hypotheses and one call
of more than 2^20 hypotheses; ranking and ties; the refined poses bit for bit against lanes armed with the winners and STARTed on the
scan, and against the frozen oracle; recovery of the pose of a mapped scan from a 21 x 21 m x 72-heading search, and an off-map
scan scoring far below; relocalise calls between stream calls change nothing; refusals change nothing."""
import struct

import numpy as np
import pytest

import lane_refs as R
import prior_build_cases as PB
import reloc_cases as RC

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
IDLE, SCAN, START = 0, 1, 2
IDENT7 = np.array([0, 0, 0, 1.0, 0, 0, 0])


def _ctx(aloam, maxpts, batch=1, ns=16, **cfg):
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, max_ring_points=4096, max_map_points=400000, **cfg)


def _entries(dev, i0, i1):
    return [(d.data_ptr(), d.shape[0], START if i == i0 else SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def _call(ctx, batch, lanes, mapped=True):
    """one aloam_scan_stream_lanes call; lanes = {lane: entries} -> {lane: (odometry rows, map rows)}"""
    steps = max(len(e) for e in lanes.values())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for lane, entries in lanes.items():
        for k, (p, n, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    o, m = ctx.scan_stream_lanes(ptrs, counts, ops, True, mapped=mapped)
    return {lane: (o[:len(e), lane], m[:len(e), lane] if mapped else None) for lane, e in lanes.items()}


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


_WORLD = {}


def _world(aloam, synth, sensor="VLP-16"):
    """scans of trajectory 0, the snapshot of the lane that mapped the first N_MAP of them, its map poses, the prior map as the
    oracle's FrozenMap and scorer, and every scan's less-sharp / less-flat clouds from the device's feature extraction"""
    if sensor not in _WORLD:
        import pyfrozen
        ns = synth.SENSORS[sensor][0]
        scans = R.traj(synth, 0, RC.N_MAP + 6, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)
        M = R.maxn([scans]) + 1024
        dev = R.to_device(scans)
        c = _ctx(aloam, M, 1, ns)
        o, m = _call(c, 1, {0: _entries(dev, 0, RC.N_MAP)})[0]
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
        _WORLD[sensor] = {"scans": scans, "dev": dev, "M": M, "ns": ns, "blob": blob, "map": m, "frozen": frozen,
                          "scorer": RC.FrozenScorer(frozen), "feats": feats, "res": synth.SENSORS[sensor][3:5]}
    return _WORLD[sensor]


def _localiser(aloam, W, batch=1):
    c = _ctx(aloam, W["M"], batch, W["ns"])
    c.prior_map_load(W["blob"])
    return c


def _far(n):
    """hypotheses that put the scan outside the buffer, in empty cubes of it, or under a non-unit quaternion"""
    return np.array([[0, 0, 0, 1.0, 1e4, 0, 0], [0, 0, 0, 1.0, 300.0, 300.0, 0], [0, 0, 0, 1.0, -520.0, 0, 50.0],
                     [0, 0, 0.3, 2.0, 1.0, 0.5, 0]] * n)[:n]


@pytest.mark.parametrize("sensor,inlier_sq,max_pts", [("VLP-16", 1.0, 1024), ("VLP-16", 0.25, 64), ("HDL-32", 0.5, 1 << 20)])
def test_scores_equal_the_oracle(aloam, synth, sensor, inlier_sq, max_pts):
    W = _world(aloam, synth, sensor)
    s = 5
    f = W["feats"][s]
    hyps = np.concatenate([RC.search_grid(aloam, W["map"][s], offset=(0.3, -0.2, 0), half=3.0, step=1.0, n_yaw=36), _far(4)])
    c = _localiser(aloam, W)
    res, sc = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=inlier_sq, max_score_points=max_pts, refine=4)
    ref = W["scorer"].score(f["less_sharp"], f["less_flat"], hyps, inlier_sq, max_pts, *W["res"])
    bad = np.nonzero(sc != ref)[0]
    assert not len(bad), (len(bad), bad[:8], sc[bad[:8]], ref[bad[:8]])
    assert sc.max() > 0 and (sc[-4:] == ref[-4:]).all()
    # n_hyp = 1
    r1, s1 = c.prior_relocalise(hyps[-1:], f["less_sharp"], f["less_flat"], inlier_sq=inlier_sq, max_score_points=max_pts, refine=1)
    assert s1[0] == ref[-1] and r1[0]["hyp"] == 0 and r1[0]["score"] == ref[-1]
    # the refined poses scored again: the oracle's score at the returned pose
    for r in res:
        assert r["refined_score"] == W["scorer"].score(f["less_sharp"], f["less_flat"], r["pose"][None], inlier_sq, max_pts, *W["res"],
                                                       normalise=False)[0]
    c.close()


def test_scores_at_the_d2_edges_of_a_crafted_map(aloam):
    """a map built from crafted clouds: neighbours at float d2 == inlier_sq, one ulp of the offset below and above, across a cube
    boundary and a cell face, and none at all for one type"""
    pts, corner, surf = RC.edge_case_clouds()
    c = aloam.Aloam(n_scans=16, max_points=4096, max_map_points=400000)
    c.prior_map_build(corner, surf)
    frozen = PB.oracle_build(corner, surf, c.cfg.line_res, c.cfg.plane_res)[0].frozen()
    S = RC.FrozenScorer(frozen)
    hyps = np.array([IDENT7, IDENT7 + [0, 0, 0, 0, 0, 0.1, 0], IDENT7 + [0, 0, 0, 0, 30.0, 0, 0]])
    for isq in (RC.EDGE_SQ, 1.0):
        _, sc = c.prior_relocalise(hyps, pts[0], pts[1], inlier_sq=isq, max_score_points=1 << 20, refine=1)
        ref = S.score(pts[0], pts[1], hyps, isq, 1 << 20, c.cfg.line_res, c.cfg.plane_res)
        assert np.array_equal(sc, ref), (isq, sc, ref)
    # an empty corner map: corner points never count
    c.prior_map_build(np.zeros((0, 4), np.float32), surf)
    _, sc = c.prior_relocalise(hyps, pts[0], pts[1], inlier_sq=RC.EDGE_SQ, max_score_points=1 << 20, refine=1)
    ref = RC.FrozenScorer(PB.oracle_build(np.zeros((0, 4), np.float32), surf, c.cfg.line_res, c.cfg.plane_res)[0].frozen()).score(
        pts[0], pts[1], hyps, RC.EDGE_SQ, 1 << 20, c.cfg.line_res, c.cfg.plane_res)
    assert np.array_equal(sc, ref), (sc, ref)
    c.close()


def test_a_call_of_more_than_2_20_hypotheses(aloam, synth):
    W = _world(aloam, synth)
    s = 5
    f = W["feats"][s]
    hyps = RC.search_grid(aloam, W["map"][s], offset=(0.0, 0.0, 0), half=15.0, step=0.5, n_yaw=288)
    assert len(hyps) >= 1 << 20
    c = _localiser(aloam, W)
    res, sc = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.25, max_score_points=256, refine=16)
    sample = np.random.default_rng(11).choice(len(hyps), 300, replace=False)
    ref = W["scorer"].score(f["less_sharp"], f["less_flat"], hyps[sample], 0.25, 256, *W["res"])
    assert np.array_equal(sc[sample], ref)
    order = np.lexsort((np.arange(len(sc)), -sc))[:16]
    assert sorted(r["hyp"] for r in res) == sorted(order.tolist())
    c.close()


def test_ranking_ties_and_the_refining_frames(aloam, synth):
    """duplicated hypotheses rank by index; K = 1 and 16; each refined pose == the START row of a lane armed with the winner (bit
    for bit) and the frozen oracle's frame from it (1e-6); refined ties keep the coarse rank"""
    import pyfrozen
    W = _world(aloam, synth)
    s = 5
    f = W["feats"][s]
    grid = RC.search_grid(aloam, W["map"][s], offset=(0.2, 0.1, 0), half=2.0, step=1.0, n_yaw=8)
    best = int(np.argmax(W["scorer"].score(f["less_sharp"], f["less_flat"], grid, 0.5, 256, *W["res"])))
    scaled = grid[best:best + 1].copy()
    scaled[:, :4] *= 3.0
    hyps = np.concatenate([grid, grid[best:best + 1], scaled])   # two copies of the best, one not normalised
    c = _localiser(aloam, W, 16)
    r1, sc = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=1)
    assert r1[0]["hyp"] == best and sc[best] == sc[-1] == sc[-2] == sc.max()
    res, sc16 = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=16)
    assert np.array_equal(sc, sc16)
    rank = {int(h): i for i, h in enumerate(np.lexsort((np.arange(len(sc)), -sc))[:16])}
    assert set(r["hyp"] for r in res) == set(rank)
    for a, b in zip(res, res[1:]):   # (refined score descending, coarse rank ascending)
        assert (a["refined_score"], -rank[a["hyp"]]) > (b["refined_score"], -rank[b["hyp"]])
    dup = [r for r in res if r["hyp"] in (best, len(grid), len(grid) + 1)]
    assert len(dup) == 3 and all(np.array_equal(d["pose"], dup[0]["pose"]) for d in dup)   # the same frame three times
    # every result against a lane armed with its hypothesis and STARTed on the scan, all 16 in one call
    for l, r in enumerate(res):
        c.lane_localise(l, hyps[r["hyp"], :4], hyps[r["hyp"], 4:])
    rows = _call(c, 16, {l: _entries(W["dev"], s, s + 1) for l in range(16)})
    for l, r in enumerate(res):
        assert np.array_equal(rows[l][1][0], r["pose"]), l
        loc = pyfrozen.Localiser(W["frozen"], hyps[r["hyp"], :4], hyps[r["hyp"], 4:])
        pose, info = loc.step(f["less_sharp"], f["less_flat"], IDENT7[:4], IDENT7[4:], *W["res"])
        R.assert_near(r["pose"][None], pose[None], "refined pose %d" % l)
        assert r["flags"] == 0
    c.reset_odometry()
    # a thin window: the pose stays the (normalised) hypothesis
    thin = np.array([[0, 0, 0, 2.0, 400.0, 0, 0]])
    rt, _ = c.prior_relocalise(thin, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=1)
    assert rt[0]["flags"] == aloam.FLAG_MAP_TOO_THIN and np.array_equal(rt[0]["pose"], [0, 0, 0, 1.0, 400.0, 0, 0])
    c.close()


def test_recovery_of_a_mapped_scan_and_an_off_map_scan(aloam, synth):
    W = _world(aloam, synth)
    s = RC.SCAN
    hyps = RC.search_grid(aloam, W["map"][s])
    c = _localiser(aloam, W)
    res, sc = c.prior_relocalise(hyps, raw=W["scans"][s], inlier_sq=RC.INLIER_SQ, max_score_points=RC.MAX_PTS, refine=4)
    dt, dr = R.deviation(res[0]["pose"][None], W["map"][s:s + 1])
    assert dt < RC.NEAR_M and dr < RC.NEAR_RAD, (dt, dr)
    # a lane armed with the answer and STARTed on this scan follows the mapped trajectory
    c.lane_localise(0, res[0]["pose"][:4], res[0]["pose"][4:])
    _, m = _call(c, 1, {0: _entries(W["dev"], s, s + 6)})[0]
    dt, dr = R.deviation(m[1:], W["map"][s + 1:s + 6])
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    c.reset_odometry()
    off = synth.scan("VLP-16", RC.OFF_MAP, seed=synth.BASE_SEED + 50, n_az=900)
    _, so = c.prior_relocalise(hyps, raw=off, inlier_sq=RC.INLIER_SQ, max_score_points=RC.MAX_PTS, refine=1)
    assert so.max() < RC.OFF_MAP_RATIO * sc.max(), (so.max(), sc.max())
    c.close()


def test_relocalise_calls_between_stream_calls_change_nothing(aloam, synth):
    """a mapping, a localising and an odometry lane; the same schedule with and without relocalise calls between the stream calls:
    every row, the prior map's bytes and the launches of every stream call are the same"""
    W = _world(aloam, synth)
    f = W["feats"][5]
    hyps = RC.search_grid(aloam, W["map"][5], offset=(0.2, 0.1, 0), half=2.0, step=1.0, n_yaw=8)
    init = W["map"][2]
    out = []
    for reloc in (False, True):
        c = _localiser(aloam, W, 3)
        before = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes()
        rows, launches, got = [], [], []

        def between():
            if reloc:
                got.append(c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=3))

        def stream(lanes, mapped=True):
            a = c.launch_count()
            r = _call(c, 3, lanes, mapped)
            launches.append(c.launch_count() - a)
            rows.append(r)
        between()
        stream({2: _entries(W["dev"], 0, 3)}, mapped=False)
        between()
        c.lane_localise(1, init[:4], init[4:])
        stream({0: _entries(W["dev"], 0, 3), 1: _entries(W["dev"], 2, 5)})
        between()
        stream({0: [(p, n, SCAN) for p, n, _ in _entries(W["dev"], 3, 6)], 1: [(p, n, SCAN) for p, n, _ in _entries(W["dev"], 5, 8)]})
        between()
        stream({2: _entries(W["dev"], 3, 5)}, mapped=False)   # its trajectory ended at its first idle step: a new one
        assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == before
        out.append((rows, launches, got))
        c.close()
    (ra, la, _), (rb, lb, got) = out
    assert la == lb
    for a, b in zip(ra, rb):
        for lane in a:
            assert np.array_equal(a[lane][0], b[lane][0]) and (a[lane][1] is None or np.array_equal(a[lane][1], b[lane][1])), lane
    # and the relocaliser answers the same whatever ran before it
    for res, sc in got[1:]:
        assert np.array_equal(sc, got[0][1]) and all(np.array_equal(x["pose"], y["pose"]) for x, y in zip(res, got[0][0]))


def test_refusals_leave_the_context_as_it_was(aloam, synth):
    W = _world(aloam, synth)
    f = W["feats"][5]
    hyps = RC.search_grid(aloam, W["map"][5], offset=(0.2, 0.1, 0), half=1.0, step=1.0, n_yaw=4)
    c = _ctx(aloam, W["M"], 2, W["ns"])
    run = lambda h=hyps, **k: c.prior_relocalise(h, f["less_sharp"], f["less_flat"], **{"inlier_sq": 0.5, "max_score_points": 256, "refine": 2, **k})
    _expect(aloam, ERR_STATE, run)                                  # no prior map
    c.prior_map_load(W["blob"])
    before = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes()
    good = run()
    for bad in ({"inlier_sq": 0.0}, {"inlier_sq": -1.0}, {"inlier_sq": 1.0001}, {"inlier_sq": float("nan")}, {"refine": 0}, {"refine": 17},
                {"max_score_points": 0}):
        _expect(aloam, ERR_INVALID_ARG, lambda: run(**bad))
    _expect(aloam, ERR_INVALID_ARG, lambda: run(hyps[:2], refine=3))   # K > n_hyp
    for row in (np.array([0, 0, 0, 0, 1.0, 0, 0]), np.array([0, 0, np.nan, 1.0, 0, 0, 0]), np.array([0, 0, 0, 1.0, 0, np.inf, 0])):
        h = hyps.copy()
        h[1] = row
        _expect(aloam, ERR_INVALID_ARG, lambda: run(h))
    big = np.zeros((W["M"] + 1, 4), np.float32)
    _expect(aloam, ERR_CAPACITY, lambda: c.prior_relocalise(hyps, big, f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=2))
    again = run()
    assert np.array_equal(again[1], good[1]) and all(np.array_equal(x["pose"], y["pose"]) for x, y in zip(again[0], good[0]))
    assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == before
    assert aloam.lib().aloam_debug_shard_emulate(c._h, 0, 2, 0, 0) == 0   # an emulating context
    _expect(aloam, ERR_STATE, run)
    c.close()
