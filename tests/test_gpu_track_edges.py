"""GPU parity at the edges of the per-row records (aloam_set_map_rows, aloam_map_rows): k_track_score's staging and record
dimension, its 27-cell walk on crafted thin-map scenes, and k_map_rows over whole row tables.  The scenes are in
tests/track_edge_cases.py, whose properties tests/test_oracle_track_edges.py checks on the CPU.
  * A: START rows of localising lanes on the VLP-16 world of tests/track_cases.py with m = 1 .. 513 and 5214 scoring points, the
    corner / surf switch at lanes 31 / 0 / 1 of a warp, max_score_points 1, n_c - 1, n_c, n_c + 1 and above both stacks, the
    largest stack a synthetic sensor reaches (subsampled), and one 16-lane step with 16 scans and stack sizes, one lane off the map;
  * B: thin frames on crafted maps, armed so that one stack point of a real scan lands on the walk scene's query: the inlier at
    every flat walk index of tests/reloc_cases.py, d2 at inlier_sq and one float below, inlier_sq 1 and the smallest float, far and
    aliasing poses;
  * C: 64 x 16 and 256 x 16 (kMaxStreamScans) calls of every row kind at mapping_skip_frame 2, a smaller call after the largest,
    outer_iters 1 and 4, and a localising frame whose stack filter overflows its key.
References: the oracle's score at the row's map pose on the device's own features (integer-equal), the numpy brute force on the
crafted scenes, aloam_prior_relocalise's score of the single hypothesis at that pose where the pose is a fixed point of its
normalisation, and the aloam_mapper_step replay of tests/test_gpu_map_rows.py for mapped rows."""
import ctypes as C

import numpy as np
import pytest

import prior_build_cases as PB
import reloc_cases as RC
import test_gpu_map_rows as MR
import track_cases as TC
import track_edge_cases as TE

pytestmark = pytest.mark.gpu

IDLE, SCAN, START = 0, 1, 2
EMPTY = np.zeros((0, 4), np.float32)
N_SCANS = {"VLP-16": 16, "HDL-32": 32, "HDL-64": 64}


def _kinds(aloam):
    return dict(IDLE=aloam.ROW_IDLE, MAPPED=aloam.ROW_MAPPED, LOCALISED=aloam.ROW_LOCALISED, SKIPPED=aloam.ROW_SKIPPED)


def _store(aloam, W):
    if "store" not in W:
        W["store"] = aloam.snapshot_store_clouds(W["blob"])
    return W["store"]


def _scorer(aloam, W, leaves):
    """the oracle's scorer of the world's prior map rebuilt at `leaves` (what prior_map_build makes of the store's clouds)"""
    key = ("scorer", tuple(leaves))
    if key not in W:
        s = _store(aloam, W)
        W[key] = RC.FrozenScorer(PB.oracle_build(s["corner"], s["surf"], leaves[0], leaves[1], s["centre"])[0].frozen())
    return W[key]


def _world_ctx(aloam, W, sensor, leaves, batch, maxpts, **cfg):
    s = _store(aloam, W)
    c = aloam.Aloam(n_scans=N_SCANS[sensor], max_points=maxpts, max_batch=batch, max_ring_points=4096, max_map_points=400000,
                    line_res=leaves[0], plane_res=leaves[1], **cfg)
    c.prior_map_build(s["corner"], s["surf"], s["centre"])
    return c


def _start(c, batch, scans, lanes):
    """one step: lane l STARTs on device scan scans[i] for (l, i) in lanes -> (odometry, map poses, rows)"""
    return MR._call(c, batch, {l: [(scans[i].data_ptr(), scans[i].shape[0], START)] for l, i in lanes})


def _fixed_point(pose):
    return RC.normalised(pose)[0].tobytes() == np.asarray(pose, np.float64).tobytes()


def _check_scored(aloam, c, row, pose, f, S, isq, mp, leaves, raw=None, what=""):
    """row: localised, its stack sizes those of the oracle's filter on the device's features, its score the oracle's at the
    row's map pose, and where the pose is a fixed point of relocalisation's normalisation, aloam_prior_relocalise's score of that
    single hypothesis from the same raw scan -> (score, m_c, m)"""
    assert row["kind"] == aloam.ROW_LOCALISED, what
    pts = RC.scoring_points(f["less_sharp"], f["less_flat"], mp, *leaves)
    st = [len(RC.scoring_points(f["less_sharp"], f["less_flat"], TE.BIG, *leaves)[k]) for k in (0, 1)]
    assert list(row["n_stack"]) == st, (what, row["n_stack"], st)
    assert row["n_score"] == len(pts[0]) + len(pts[1]), (what, row["n_score"], len(pts[0]), len(pts[1]))
    ref = S.score_points(pts, pose[None], isq, normalise=False)[0]
    assert row["score"] == ref, (what, row["score"], ref)
    if raw is not None and _fixed_point(pose):
        _, sc = c.prior_relocalise(pose[None], raw=raw, inlier_sq=isq, max_score_points=mp, refine=1)
        assert sc[0] == row["score"], (what, sc[0], row["score"])
    return int(ref), len(pts[0]), len(pts[0]) + len(pts[1])


# ------------------------------------------------------------------------------------------------------ A. staging and records
_CTX = {}


@pytest.fixture(scope="module")
def stage_ctx(aloam, synth):
    W = MR._world(aloam, synth)

    def get(sensor, leaves):
        key = (sensor, tuple(leaves))
        if key not in _CTX:
            maxpts = 262144 if sensor == "HDL-64" else 65536
            _CTX[key] = (_world_ctx(aloam, W, sensor, leaves, 1, maxpts), _scorer(aloam, W, leaves))
        return _CTX[key]
    yield W, get
    for c, _ in _CTX.values():
        c.close()
    _CTX.clear()


_REACHED = {"m": set(), "mc": set(), "mp": set()}


def _stage_run(aloam, synth, W, get, sensor, n_az, index, leaves, mp, what):
    c, S = get(sensor, leaves)
    raw = TE.raw_scan(synth, sensor, n_az, index)
    f = c.extract_features(raw)
    import torch
    dev = torch.from_numpy(raw).cuda()
    c.set_map_rows(True, TC.ISQ, mp)
    T = W["map"][index]
    c.lane_localise(0, T[:4], T[4:])
    _, m, rows = _start(c, 1, [dev], [(0, 0)])
    row = MR._row(rows, 0)
    assert row["err"] == 0 and not row["flags"] & aloam.FLAG_MAP_TOO_THIN, (what, row)
    return row, _check_scored(aloam, c, row, m[0, 0], f, S, TC.ISQ, mp, leaves, raw=raw, what=what)


@pytest.mark.parametrize("case", TE.STAGE_CASES, ids=lambda k: "%s-%d-s%d-mp%s" % k)
def test_staging_of_a_start_row(aloam, synth, stage_ctx, case):
    W, get = stage_ctx
    sensor, n_az, index, spec = case
    n_c, n_s = TE.stacks(synth, sensor, n_az, index, TE.DEFAULT_LEAVES)
    mp = TE.resolve_mp(spec, n_c, n_s)
    row, (score, m_c, m) = _stage_run(aloam, synth, W, get, sensor, n_az, index, TE.DEFAULT_LEAVES, mp, case)
    assert (m_c, m) == TE.staging(n_c, n_s, mp), (case, m_c, m)
    assert score > 0, case
    _REACHED["m"].add(m)
    _REACHED["mp"].add(spec if isinstance(spec, str) else ("1" if spec == 1 else "int"))
    if m - m_c > 0 and m_c % 32:
        _REACHED["mc"].add(m_c % 32)
    elif m - m_c > 0:
        _REACHED["mc"].add(0)


def test_staging_reached_every_residue():
    """(runs after the staging cases) the values of m, m_c mod 32 with surf points after the switch, and max_score_points"""
    if len(_REACHED["m"]) == 0:
        pytest.skip("the staging cases did not run in this session")
    assert set(TE.STAGE_M) <= _REACHED["m"], sorted(_REACHED["m"])
    assert set(TE.STAGE_MC_RES) <= _REACHED["mc"], _REACHED["mc"]
    assert {"1", "nc-1", "nc", "nc+1", "big"} <= _REACHED["mp"], _REACHED["mp"]


def test_the_largest_stack_subsampled(aloam, synth, stage_ctx):
    W, get = stage_ctx
    sensor, n_az, index, leaves, mp = TE.LARGE_CASE
    row, (score, m_c, m) = _stage_run(aloam, synth, W, get, sensor, n_az, index, leaves, mp, "large")
    assert row["n_stack"][1] >= TE.LARGE_MIN and m - m_c == mp < row["n_stack"][1], row
    assert score > 0
    print("\nlargest stack reached: %d surf points (%s, %d azimuth steps, plane_res %g), %d scored, %d inliers"
          % (row["n_stack"][1], sensor, n_az, leaves[1], m - m_c, score))


def test_sixteen_localising_lanes_each_score_their_own_row(aloam, synth):
    """16 lanes START on 16 scans in one step (one k_track_score launch of 16 records): lane 0 has the smallest stacks, lane 15
    the largest, lane WIDE_OFF is armed off the map (a thin frame: score 0); every row's score is the oracle's of its own scan at
    its own map pose"""
    import torch
    W = MR._world(aloam, synth)
    raws = [TE.raw_scan(synth, "VLP-16", n_az, k) for n_az, k in TE.WIDE_LANES]
    c = _world_ctx(aloam, W, "VLP-16", TE.DEFAULT_LEAVES, 16, max(r.shape[0] for r in raws) + 1024)
    S = _scorer(aloam, W, TE.DEFAULT_LEAVES)
    c.set_map_rows(True, TC.ISQ, TE.BIG)
    for l, (_, k) in enumerate(TE.WIDE_LANES):
        T = TC.off_map(W["map"][k]) if l == TE.WIDE_OFF else W["map"][k]
        c.lane_localise(l, T[:4], T[4:])
    dev = [torch.from_numpy(r).cuda() for r in raws]
    _, m, rows = _start(c, 16, dev, [(l, l) for l in range(16)])
    got = []
    for l in range(16):
        f = c.extract_features(raws[l])
        row = MR._row(rows, l)
        got.append(_check_scored(aloam, c, row, m[0, l], f, S, TC.ISQ, TE.BIG, TE.DEFAULT_LEAVES, what=l))
        assert bool(row["flags"] & aloam.FLAG_MAP_TOO_THIN) == (l == TE.WIDE_OFF), (l, row["flags"])
    sc, ms = [g[0] for g in got], [g[2] for g in got]
    assert sc[TE.WIDE_OFF] == 0 and all(s > 0 for l, s in enumerate(sc) if l != TE.WIDE_OFF), sc
    assert ms[15] == max(ms) and ms[0] == min(ms) and len(set(ms)) == 16, ms
    c.close()


# ----------------------------------------------------------------------------------------------- B. crafted thin-map scenes
_SCENES = TE.thin_scenes()
_SCENE_FEATS = {}


def _scene_feats(aloam, synth):
    if "f" not in _SCENE_FEATS:
        raw = TE.raw_scan(synth, *TE.SCENE_SCAN)
        fx = aloam.Aloam(n_scans=16, max_points=raw.shape[0] + 1024, line_res=RC.WALK_LEAF, plane_res=RC.WALK_LEAF)
        _SCENE_FEATS["f"] = (raw, fx.extract_features(raw))
        fx.close()
    return _SCENE_FEATS["f"]


@pytest.mark.parametrize("t", [0, 1], ids=["corner", "surf"])
@pytest.mark.parametrize("k", range(len(_SCENES)), ids=[s[0] for s in _SCENES])
def test_a_thin_start_row_scores_the_crafted_scene(aloam, synth, k, t):
    """the scene's map as type t, the other type one far point: the frame is thin and the START row's map pose is the armed pose
    bit for bit; the chosen stack point lands on the query (or offset from it) and is an inlier exactly as claimed; the row's
    score == the oracle's == the brute force's == aloam_prior_relocalise's, every stack point counted"""
    import torch
    name, s, isq, off, expect = _SCENES[k]
    raw, f = _scene_feats(aloam, synth)
    leaves = (RC.WALK_LEAF, RC.WALK_LEAF)
    pts = RC.scoring_points(f["less_sharp"], f["less_flat"], TE.BIG, *leaves)
    i = TE.pick(len(pts[0]), t, (7 * k + 31 * t) % 32, len(pts[t]))
    p = pts[t][i]
    pose = TE.arming(s["query"][0], p, off)
    maps = (s["map"], TE.OTHER_MAP) if t == 0 else (TE.OTHER_MAP, s["map"])
    c = aloam.Aloam(n_scans=16, max_points=raw.shape[0] + 1024, max_map_points=20000, line_res=RC.WALK_LEAF, plane_res=RC.WALK_LEAF)
    c.prior_map_build(*maps)
    S = RC.FrozenScorer(PB.oracle_build(maps[0], maps[1], *leaves)[0].frozen())
    c.set_map_rows(True, isq, TE.BIG)
    c.lane_localise(0, pose[:4], pose[4:])
    _, m, rows = _start(c, 1, [torch.from_numpy(raw).cuda()], [(0, 0)])
    row = MR._row(rows, 0)
    assert row["flags"] & aloam.FLAG_MAP_TOO_THIN and row["err"] == 0, row
    assert m[0, 0].tobytes() == pose.tobytes(), (m[0, 0], pose)
    moved = RC.transform(pose, p[None])[0]
    if not any(off):
        assert moved.tobytes() == s["query"][0, :3].tobytes(), (moved, s["query"])
    own = [EMPTY, EMPTY]
    own[t] = p[None]
    assert RC.brute_score(maps[0], maps[1], own, pose[None], isq)[0] == int(expect), name
    score, _, _ = _check_scored(aloam, c, row, pose, f, S, isq, TE.BIG, leaves, raw=raw, what=name)
    assert _fixed_point(pose)
    brute = RC.brute_score(maps[0], maps[1], pts, pose[None], isq)[0]
    assert score == brute and score >= int(expect), (name, score, brute)
    c.close()


# ------------------------------------------------------------------------------------------------------------- C. row tables
ARMED = {1: 2, 4: 0, 6: 5, 9: 1, 12: 3, 14: 6}   # lane -> scan of its first (localising) trajectory


def _run_table(aloam, W, c, ops, idx, armed):
    for l, s in armed.items():
        c.lane_localise(l, W["map"][s][:4], W["map"][s][4:])
    lanes = {}
    for l in range(ops.shape[1]):
        lanes[l] = [(W["dev"][idx[k, l]].data_ptr(), W["dev"][idx[k, l]].shape[0], int(ops[k, l])) if ops[k, l] else (0, 0, IDLE)
                    for k in range(ops.shape[0])]
    return MR._call(c, ops.shape[1], lanes)


def _check_table(aloam, W, c, ops, idx, armed, skip, odom, mp, rows, S):
    """every row against the kind its schedule gives; idle and skipped rows empty; mapped rows against the mapper-step replay;
    localised rows against the oracle's score"""
    K = _kinds(aloam)
    steps, nb = ops.shape
    want = TE.expected_kinds(ops, armed, skip, K["IDLE"], K["MAPPED"], K["LOCALISED"], K["SKIPPED"])
    kinds = rows["kind"].reshape(steps, nb)
    assert np.array_equal(kinds, want), np.argwhere(kinds != want)[:8]
    zero = [k for k in rows if k not in ("kind", "score")]
    for r in np.flatnonzero(rows["kind"] == K["IDLE"]):
        assert rows["score"][r] == 0 and all(not np.any(rows[k][r]) for k in zero), r
    for r in np.flatnonzero(rows["kind"] == K["SKIPPED"]):
        assert rows["score"][r] == -1 and all(not np.any(rows[k][r]) for k in zero), r
    for r in np.flatnonzero(rows["kind"] == K["MAPPED"]):
        assert rows["score"][r] == -1 and rows["n_score"][r] == 0, r
    cfg = {**MR._cfg(c), "max_batch": 1}
    n_rep = n_loc = 0
    for l in range(nb):
        starts = list(np.flatnonzero(ops[:, l] == START)) + [steps]
        for a, b in zip(starts[:-1], starts[1:]):
            run = [k for k in range(a, b) if ops[k, l]]
            run = run[:next((j for j in range(1, len(run)) if run[j] != run[j - 1] + 1), len(run))]
            kr = [int(want[k, l]) for k in run]
            if K["LOCALISED"] in kr:
                for k in run:
                    if want[k, l] == K["LOCALISED"]:
                        r = k * nb + l
                        row = MR._row(rows, r)
                        assert row["err"] == 0, (k, l)
                        _check_scored(aloam, c, row, mp[k, l], W["feats"][idx[k, l]], S, TC.ISQ, TC.PTS, W["res"], what=(k, l))
                        n_loc += 1
                continue
            sub = {f: v[[k * nb + l for k in run]] for f, v in rows.items()}
            feats = [W["feats"][idx[k, l]] for k in run]
            rep = MR._replay(aloam, feats, odom[run, l], kr, sub, cfg, (l, a))
            for j, pose, _ in rep:
                assert np.array_equal(pose, mp[run[j], l]), (l, run[j])
            n_rep += len(rep)
    return n_rep, n_loc


def _table_ctx(aloam, W, nb=16, **cfg):
    c = _world_ctx(aloam, W, "VLP-16", W["res"], nb, W["M"], mapping_skip_frame=2, **cfg)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    return c


@pytest.mark.parametrize("steps", [64, 256])
def test_a_row_table_of_every_kind(aloam, synth, steps):
    """steps x 16 rows (256 x 16 = kMaxStreamScans) at mapping_skip_frame 2: lanes idle, map, localise and skip in every mix, lane
    0 idle at first so records and lanes differ.  After the 256-step call a 8 x 4 call on the same context equals that call on a
    fresh context, row for row"""
    W = MR._world(aloam, synth)
    S = _scorer(aloam, W, W["res"])
    K = _kinds(aloam)
    ops, idx = TE.schedule(steps, 16, len(W["dev"]), ARMED)
    c = _table_ctx(aloam, W)
    odom, mp, rows = _run_table(aloam, W, c, ops, idx, ARMED)
    assert rows["kind"].size == steps * 16
    n_rep, n_loc = _check_table(aloam, W, c, ops, idx, ARMED, 2, odom, mp, rows, S)
    kinds = rows["kind"].reshape(steps, 16)
    every = [k for k in range(steps) if len(set(kinds[k])) == 4]
    assert every and n_loc >= 20 and n_rep >= 100, (len(every), n_loc, n_rep)
    if steps == 256:
        ops2 = np.array([[START, START, START, IDLE]] + [[SCAN, SCAN, SCAN, IDLE]] * 7, np.int32)
        idx2 = np.array([[k, k + 3, k + 2, 0] for k in range(8)])
        armed2 = {2: 2}
        got = _run_table(aloam, W, c, ops2, idx2, armed2)
        fresh = _table_ctx(aloam, W, 16)
        ref = _run_table(aloam, W, fresh, ops2, idx2, armed2)
        fresh.close()
        for k in got[2]:
            assert np.array_equal(got[2][k], ref[2][k]), k
        assert np.array_equal(got[1], ref[1], equal_nan=True)
        _check_table(aloam, W, c, ops2, idx2, armed2, 2, got[0], got[1], got[2], S)
        assert (got[2]["kind"] == K["LOCALISED"]).sum() == 4 and (got[2]["kind"] == K["MAPPED"]).sum() == 8
    c.close()


@pytest.mark.parametrize("outer", [1, 4])
def test_outer_iterations_of_the_rows(aloam, synth, outer):
    """outer_iters 1 and 4 (k_map_rows copies min(outer, 4) summary heads): every mapped row's stats, termination included, equal
    the replay's; the terminations past outer_iters are 0; localised rows score as the oracle"""
    W = MR._world(aloam, synth)
    S = _scorer(aloam, W, W["res"])
    ops, idx = TE.schedule(14, 4, len(W["dev"]), {2: 1}, seed=5)
    c = _table_ctx(aloam, W, 4, outer_iters=outer)
    odom, mp, rows = _run_table(aloam, W, c, ops, idx, {2: 1})
    n_rep, n_loc = _check_table(aloam, W, c, ops, idx, {2: 1}, 2, odom, mp, rows, S)
    assert n_rep >= 8 and n_loc >= 3, (n_rep, n_loc)
    done = rows["kind"] == aloam.ROW_MAPPED
    # (a trajectory's first mapped frame sees an empty store: a thin frame with zero stats)
    assert not rows["termination"][:, outer:].any() and (rows["lm_iters"][done] > 0).sum() >= 4
    c.close()


def test_a_localising_key_overflow_is_on_its_row(aloam, synth):
    """a localising lane over four scans of the world, the second with two returns moved out so that its less-sharp stack's box
    needs more than 31 key bits: the call returns ALOAM_ERR_CAPACITY, error bit 0 is set on exactly that row, its stack is the
    unfiltered cloud and its score the oracle's on that unfiltered stack"""
    import torch
    W = MR._world(aloam, synth)
    raw4, _ = TE.overflow_scan(synth)
    scans = [W["scans"][3], raw4, W["scans"][5], W["scans"][6]]
    dev = [torch.from_numpy(s).cuda() for s in scans]
    c = MR._localiser(aloam, W)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    T = W["map"][3]
    c.lane_localise(0, T[:4], T[4:])
    ptrs, counts, ops = MR._grid(1, {0: [(d.data_ptr(), d.shape[0], START if i == 0 else SCAN) for i, d in enumerate(dev)]})
    odom, mp = np.zeros((4, 1, 7)), np.zeros((4, 1, 7))
    st = (aloam.Stats * 1)()
    opsc = np.ascontiguousarray(ops, np.int32)
    rc = aloam.lib().aloam_scan_stream_lanes(c._h, aloam._views(ptrs, counts, 4), opsc.ctypes.data_as(C.POINTER(C.c_int)), 4, 1, 1,
                                             aloam._dp(odom), aloam._dp(mp), st)
    assert rc == MR.ERR_CAPACITY, rc
    rows = c.map_rows(4)
    assert (rows["kind"] == aloam.ROW_LOCALISED).all()
    assert [int(e & 1) for e in rows["err"]] == [0, 1, 0, 0], rows["err"]
    for k in range(4):
        f = c.extract_features(scans[k])
        pts = RC.scoring_points(f["less_sharp"], f["less_flat"], TC.PTS, *W["res"])
        if k == 1:
            assert TE.seg_box(f["less_sharp"], W["res"][0])[1]
            assert row_stack(rows, k) == [len(f["less_sharp"]), len(RC.scoring_points(EMPTY, f["less_flat"], TE.BIG, *W["res"])[1])]
            pts = (RC.subsample(f["less_sharp"], TC.PTS), pts[1])
        else:
            assert row_stack(rows, k) == [len(x) for x in RC.scoring_points(f["less_sharp"], f["less_flat"], TE.BIG, *W["res"])]
        ref = W["scorer"].score_points(pts, mp[k, 0][None], TC.ISQ, normalise=False)[0]
        assert rows["score"][k] == ref and ref > 0, (k, rows["score"][k], ref)
        assert rows["n_score"][k] == len(pts[0]) + len(pts[1])
    c.close()


def row_stack(rows, r):
    return [int(v) for v in rows["n_stack"][r]]
