"""GPU parity at the edges of relocalisation (reloc.cu: k_reloc_score, any_in_block27, k_reloc_topk and the refinement), on
crafted scenes (tests/reloc_cases.py, whose properties tests/test_oracle_reloc_edges.py checks on the CPU) and on the VLP-16 world
of tests/test_gpu_relocalise.py:
  * staging: m = m_c + m_s of 31 .. 6145 scoring points, the corner / surf boundary inside a chunk and across a stage;
  * the subsample of a 60 000-point stack at max_score_points 50 000 (i * n beyond 2^31);
  * the 27-cell walk: one inlier alone in its cell at flat walk index 0, 31, 32, 33, 63, 64, 1500 and last, behind thousands of near
    misses; no inlier; d2 == inlier_sq and one float below inside a dense cell;
  * far and odd hypotheses: keys that alias map cells through the unmasked z field, saturated cells, infinite coordinates, -q,
    non-unit quaternions;
  * the top K at n_hyp = 2^24: 17 winners in one warp, winners over the warps of a CTA and over CTAs, a tie at ranks K / K + 1
    across CTAs, a winner at n_hyp - 1, every score 0;
  * empty stacks, calls in sequence against a fresh context, and a stack filter whose key overflows.
Comparators: the oracle scorer (integer equality), the numpy brute force, the host ranking np.lexsort((index, -score)), the refined
pose of a lane armed with the hypothesis and STARTed on the scan (bit for bit), or the frozen oracle's frame on crafted clouds."""
import ctypes as C
import time

import numpy as np
import pytest

import lane_refs as R
import prior_build_cases as PB
import pyoracle
import reloc_cases as RC

pytestmark = pytest.mark.gpu

ERR_CAPACITY = -4
LEAVES = (0.2, 0.4)


def _ctx(aloam, maxpts=8192, batch=1, **cfg):
    return aloam.Aloam(n_scans=16, max_points=maxpts, max_batch=batch, max_ring_points=4096, max_map_points=20000, **cfg)


def _built(c, corner, surf):
    """builds the prior map of c from the clouds -> the oracle's scorer of the same build"""
    c.prior_map_build(corner, surf)
    return RC.FrozenScorer(PB.oracle_build(corner, surf, c.cfg.line_res, c.cfg.plane_res)[0].frozen())


def _check_ranking(res, sc, K):
    """(H): the K (hyp, score) pairs of the host ranking, out ordered by (refined score desc, coarse rank asc)"""
    top = RC.host_top(sc, K)
    rank = {int(h): i for i, h in enumerate(top)}
    assert sorted((r["hyp"], r["score"]) for r in res) == sorted((int(h), int(sc[h])) for h in top), ([r["hyp"] for r in res], top)
    keys = [(-r["refined_score"], rank[r["hyp"]]) for r in res]
    assert keys == sorted(keys), keys


def _check_refined_crafted(S, c, res, sharp, flat, isq, mp):
    """every refined score == the oracle's score at the refined pose"""
    for r in res:
        assert r["refined_score"] == S.score(sharp, flat, r["pose"][None], isq, mp, c.cfg.line_res, c.cfg.plane_res, normalise=False)[0]


# ---------------------------------------------------------------------------------------------------------------- 1. staging
@pytest.fixture(scope="module")
def stage_world(aloam):
    scan, maps = RC.stage_pool(*LEAVES)
    c = _ctx(aloam)
    S = _built(c, maps[0], maps[1])
    yield c, S, scan
    c.close()


@pytest.mark.parametrize("case", RC.STAGE_CASES, ids=lambda k: "m%d-mc%d" % (min(k[0], k[2]) + min(k[1], k[2]), min(k[0], k[2])))
def test_stage_and_chunk_boundaries(stage_world, case):
    c, S, scan = stage_world
    n_c, n_s, mp = case
    sharp, flat = scan[0][:n_c], scan[1][:n_s]
    hyps = RC.stage_hyps()
    res, sc = c.prior_relocalise(hyps, sharp, flat, inlier_sq=0.25, max_score_points=mp, refine=4)
    ref = S.score(sharp, flat, hyps, 0.25, mp, *LEAVES)
    bad = np.flatnonzero(sc != ref)
    assert not len(bad), (case, len(bad), bad[:8], sc[bad[:8]], ref[bad[:8]])
    assert len(np.unique(sc)) > 5 and sc.max() > 0.3 * (min(n_c, mp) + min(n_s, mp)), np.unique(sc)
    _check_ranking(res, sc, 4)
    _check_refined_crafted(S, c, res, sharp, flat, 0.25, mp)


# ------------------------------------------------------------------------------------------------------ 2. the 64-bit subsample
def test_the_subsample_of_a_stack_beyond_2_31_over_n(aloam):
    (corner, surf), (mc, ms) = RC.big_stack()
    c = _ctx(aloam, maxpts=65536)
    S = _built(c, mc, ms)
    hyps = np.array([RC.IDENT7, RC.shift(0.2), RC.shift(-0.35), [0, 0, np.sin(0.01), np.cos(0.01), 0.1, 0.1, 0], RC.FAR_POSE])
    res, sc = c.prior_relocalise(hyps, corner, surf, inlier_sq=0.25, max_score_points=50000, refine=2)
    ref = S.score(corner, surf, hyps, 0.25, 50000, *LEAVES)
    assert np.array_equal(sc, ref), (sc, ref)
    assert sc[0] > 20000 and sc[-1] == 0
    _check_ranking(res, sc, 2)
    c.close()


# --------------------------------------------------------------------------------------------- 3. dense cells and the walk's exit
@pytest.fixture(scope="module")
def walk_ctx(aloam):
    c = _ctx(aloam, line_res=RC.WALK_LEAF, plane_res=RC.WALK_LEAF)
    yield c
    c.close()


def _walk_run(c, m, q, isq, t):
    """the scene's map and query as type t; the other type holds one far point each"""
    far_map = np.array([[30.0, 30.0, 30.0, 7.0]], np.float32)
    far_scan = np.array([[-30.0, -30.0, -30.0, 1.0]], np.float32)
    maps = (m, far_map) if t == 0 else (far_map, m)
    scan = (q, far_scan) if t == 0 else (far_scan, q)
    S = _built(c, *maps)
    hyps = np.array([RC.IDENT7, [0, 0, 0, 3.0, 0, 0, 0], RC.FAR_POSE])
    res, sc = c.prior_relocalise(hyps, scan[0], scan[1], inlier_sq=isq, max_score_points=1 << 20, refine=1)
    ref = S.score(scan[0], scan[1], hyps, isq, 1 << 20, c.cfg.line_res, c.cfg.plane_res)
    brute = RC.brute_score(maps[0], maps[1], scan, hyps, isq)
    return sc, ref, brute, res


@pytest.mark.parametrize("t", [0, 1], ids=["corner", "surf"])
@pytest.mark.parametrize("scene", RC.WALK_SCENES, ids=lambda s: "lane%s-flat%d-of%d" % s)
def test_the_walk_finds_the_inlier_wherever_it_lies(walk_ctx, scene, t):
    s = RC.walk_scene(*scene)
    sc, ref, brute, _ = _walk_run(walk_ctx, s["map"], s["query"], s["inlier_sq"], t)
    expect = 0 if scene[0] is None else 1
    assert sc.tolist() == [expect, expect, 0] and np.array_equal(sc, ref) and np.array_equal(sc, brute), (sc, ref, brute)


@pytest.mark.parametrize("below", [False, True])
def test_d2_at_inlier_sq_inside_a_dense_cell(walk_ctx, below):
    s = RC.edge_walk_scene(below)
    sc, ref, brute, _ = _walk_run(walk_ctx, s["map"], s["query"], RC.EDGE_WALK_SQ, 0)
    assert sc.tolist() == [s["score"], s["score"], 0] and np.array_equal(sc, ref) and np.array_equal(sc, brute), (sc, ref, brute)


# ------------------------------------------------------------------------------------------------- 4. far and odd hypotheses
def test_far_and_odd_hypotheses(aloam, synth):
    import test_gpu_relocalise as TR
    W = TR._world(aloam, synth)
    s = 5
    f = W["feats"][s]
    base = W["map"][s]
    q, t0 = base[:4], base[4:]
    cs = float(RC.MAP_CELL)
    offs = [(2.0**20 * cs, 0, 0), (0, 2.0**20 * cs, 0), (0, 0, 2.0**20 * cs), (0, -cs, 2.0**21 * cs), (2.0**21 * cs,) * 3,
            (0, 0, -2.0**21 * cs), (1e30, 0, 0), (-1e30, -1e30, -1e30), (1e300, 0, 0), (0, 0, -1e300)]
    hyps = [np.r_[q, t0 + np.array(o)] for o in offs]
    hyps += [np.r_[q, t0], np.r_[-q, t0], np.r_[q * 1e-3, t0], np.r_[q * 1e3, t0]]
    hyps = np.array(hyps)
    K = len(hyps)
    c = TR._localiser(aloam, W, 16)   # the world snapshot's configuration
    res, sc = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=K)
    pts = RC.scoring_points(f["less_sharp"], f["less_flat"], 256, *W["res"])
    brute = RC.brute_score(W["scorer"].clouds[0], W["scorer"].clouds[1], pts, hyps, 0.5)
    assert np.array_equal(sc, brute), (sc, brute)
    near = np.abs(hyps[:, 4:]).max(axis=1) < 1e7
    ref = W["scorer"].score(f["less_sharp"], f["less_flat"], hyps[near], 0.5, 256, *W["res"])
    assert np.array_equal(sc[near], ref)
    assert (sc[:len(offs)] == 0).all() and sc[-4] > 0 and (sc[-4:] == sc[-4]).all()
    _check_ranking(res, sc, K)
    # every refined pose and flag against a lane armed with its hypothesis and STARTed on the scan
    for l, r in enumerate(res):
        c.lane_localise(l, hyps[r["hyp"], :4], hyps[r["hyp"], 4:])
    rows = TR._call(c, 16, {l: TR._entries(W["dev"], s, s + 1) for l in range(K)})
    for l, r in enumerate(res):
        assert rows[l][1][0].tobytes() == r["pose"].tobytes(), (l, r["hyp"], rows[l][1][0], r["pose"])
        if r["hyp"] < len(offs):
            assert r["flags"] == aloam.FLAG_MAP_TOO_THIN
    c.close()


# ------------------------------------------------------------------------------------------------------------------- 5. top K
def _line_world(aloam, **kw):
    scan, maps = RC.line_scene(**kw)
    c = _ctx(aloam, batch=1)
    S = _built(c, maps[0], maps[1])
    return c, S, scan, maps


def _levels(scan, maps):
    """shift -> score of the line scene at shifts that keep every distance away from the radius"""
    shifts = [0.025 + 0.05 * k for k in range(-9, 25)]
    sc = RC.brute_score(maps[0], maps[1], scan, np.array([RC.shift(s) for s in shifts]), 0.25)
    return dict(zip(shifts, sc.tolist()))


def test_top_k_at_the_hypothesis_limit(aloam):
    """one call of exactly 2^24 hypotheses: 17 copies of the best pose in warp 0 of CTA 0 (h = j 8 SMs 840, 840 = lcm(1..8) covers
    every blocks-per-SM) and one at n_hyp - 1: the first 16 come back"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    c, S, scan, maps = _line_world(aloam)
    lv = _levels(scan, maps)
    best = max(lv, key=lambda s: (lv[s], -s))
    n = 1 << 24
    stride = 8 * sms * 840
    copies = [j * stride for j in range(17)] + [n - 1]
    assert copies[16] < n - 1
    hyps = np.empty((n, 7))
    hyps[:] = RC.FAR_POSE
    hyps[copies] = RC.shift(best)
    c.profile_enable()
    t0 = time.perf_counter()
    res, sc = c.prior_relocalise(hyps, scan[0], scan[1], inlier_sq=0.25, max_score_points=1 << 20, refine=16)
    wall = time.perf_counter() - t0
    prof = c.profile_read()
    print("\n2^24 hypotheses on %s: call %.3f s (host normalisation and copies included), k_reloc_score %s, k_reloc_topk %s"
          % (torch.cuda.get_device_name(0), wall, prof.get("k_reloc_score"), prof.get("k_reloc_topk")))
    assert np.flatnonzero(sc).tolist() == copies and (sc[copies] == lv[best]).all()
    _check_ranking(res, sc, 16)
    assert sorted(r["hyp"] for r in res) == copies[:16]
    sample = np.random.default_rng(9).choice(n, 200, replace=False)
    rows = np.concatenate([copies, sample])
    assert np.array_equal(sc[rows], S.score(scan[0], scan[1], hyps[rows], 0.25, 1 << 20, *LEAVES))
    _check_refined_crafted(S, c, res, scan[0], scan[1], 0.25, 1 << 20)
    c.close()


def test_top_k_across_warps_and_ctas(aloam):
    """graded winners over the 8 warps of CTA 1 and over CTAs 2 .. 7 and at n_hyp - 1 (15 above the tie), a tie at ranks 16 / 17
    (K / K + 1) between CTAs 8 and 9, lower winners after it; K = 16 and K = 1"""
    c, S, scan, maps = _line_world(aloam)
    lv = _levels(scan, maps)
    levels = sorted(set(lv.values()), reverse=True)
    T = levels[len(levels) // 2]
    above = [s for s in lv if lv[s] > T]
    at = [s for s in lv if lv[s] == T]
    below = [s for s in lv if 0 < lv[s] < T]
    n = 200_003
    hyps = np.empty((n, 7))
    hyps[:] = RC.FAR_POSE
    top = [8 + w for w in range(8)] + [8 * b + b % 8 for b in range(2, 8)] + [n - 1]
    for i, h in enumerate(top):
        hyps[h] = RC.shift(above[i % len(above)])
    tie = [8 * 8 + 3, 8 * 9 + 1]
    for h in tie:
        hyps[h] = RC.shift(at[0])
    low = [8 * b + (b * 3) % 8 for b in range(10, 14)]
    for i, h in enumerate(low):
        hyps[h] = RC.shift(below[i % len(below)])
    planted = sorted(top + tie + low)
    for K in (16, 1):
        res, sc = c.prior_relocalise(hyps, scan[0], scan[1], inlier_sq=0.25, max_score_points=1 << 20, refine=K)
        _check_ranking(res, sc, K)
        assert np.flatnonzero(sc).tolist() == planted
        assert np.array_equal(sc[planted], S.score(scan[0], scan[1], hyps[planted], 0.25, 1 << 20, *LEAVES))
        _check_refined_crafted(S, c, res, scan[0], scan[1], 0.25, 1 << 20)
        if K == 16:
            got = {r["hyp"] for r in res}
            assert tie[0] in got and tie[1] not in got and set(top) <= got
    c.close()


def test_top_k_when_every_score_is_zero(aloam):
    """2^19 far hypotheses: at most 8 blocks of 8 warps per SM, so every warp ranks more than 32 zero keys in its list of 16"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    c, S, scan, maps = _line_world(aloam)
    n = 1 << 19
    assert n // (sms * 8 * 8) > 32
    hyps = np.tile(RC.FAR_POSE, (n, 1))
    hyps[:, 5] = np.arange(n) * 0.5
    for K in (16, 3):
        res, sc = c.prior_relocalise(hyps, scan[0], scan[1], inlier_sq=0.25, max_score_points=1 << 20, refine=K)
        assert not sc.any()
        assert [r["hyp"] for r in res] == list(range(K)) and all(r["score"] == 0 for r in res)
    c.close()


# ----------------------------------------------------------------------------------------------------------- 6. empty stacks
@pytest.mark.parametrize("K", [1, 16])
@pytest.mark.parametrize("empty", ["sharp", "flat", "both"])
def test_empty_stacks(aloam, synth, empty, K):
    """a VLP-16 scan with its less-sharp cloud, its less-flat cloud or both replaced by an empty cloud, on the world's prior map
    (not thin, so the refining frames solve on whatever stack is left): scores == the oracle's, refined poses and flags == the
    frozen oracle's localising frame from each winner"""
    import pyfrozen
    import test_gpu_relocalise as TR
    W = TR._world(aloam, synth)
    s = 5
    f = W["feats"][s]
    none = np.zeros((0, 4), np.float32)
    sharp = none if empty in ("sharp", "both") else f["less_sharp"]
    flat = none if empty in ("flat", "both") else f["less_flat"]
    hyps = np.concatenate([np.tile(RC.FAR_POSE, (3, 1)), RC.search_grid(aloam, W["map"][s], offset=(0.2, 0.1, 0), half=1.0, step=1.0, n_yaw=2)])
    c = TR._localiser(aloam, W)
    res, sc = c.prior_relocalise(hyps, sharp, flat, inlier_sq=0.5, max_score_points=256, refine=K)
    ref = W["scorer"].score(sharp, flat, hyps, 0.5, 256, *W["res"])
    assert np.array_equal(sc, ref), (sc, ref)
    if empty == "both":
        assert not sc.any() and [r["hyp"] for r in res] == list(range(K))
    else:
        assert sc.max() > 0
    _check_ranking(res, sc, K)
    for r in res:
        assert r["refined_score"] == W["scorer"].score(sharp, flat, r["pose"][None], 0.5, 256, *W["res"], normalise=False)[0]
        loc = pyfrozen.Localiser(W["frozen"], hyps[r["hyp"], :4], hyps[r["hyp"], 4:])
        pose, info = loc.step(sharp, flat, RC.IDENT7[:4], RC.IDENT7[4:], *W["res"])
        R.assert_near(r["pose"][None], pose[None], "refined pose of %d" % r["hyp"])
        assert r["flags"] == (0 if info["optimised"] else aloam.FLAG_MAP_TOO_THIN)
        if empty != "both":   # a winner on the map solves on the stack left and moves; a far one sees a thin window
            on = r["hyp"] >= 3
            assert bool(info["optimised"]) == on and np.array_equal(r["pose"], RC.normalised(hyps[r["hyp"]])[0]) != on, r["hyp"]
    c.close()


# ------------------------------------------------------------------------------------------------------ 7. calls in sequence
def test_calls_in_sequence_answer_as_a_fresh_context(aloam, synth):
    """K = 1 small, K = 16 large, K = 3 small, a rebuilt prior map, then the first map loaded again: each answer == that of a fresh
    context making only that call"""
    import test_gpu_relocalise as TR
    W = TR._world(aloam, synth)
    f = W["feats"][5]
    small = RC.search_grid(aloam, W["map"][5], offset=(0.2, 0.1, 0), half=1.0, step=1.0, n_yaw=8)
    large = RC.search_grid(aloam, W["map"][5], offset=(0.0, 0.0, 0), half=6.0, step=0.25, n_yaw=96)
    scan, maps = RC.line_scene(slope=0.03)
    lv = np.array([RC.shift(0.025 + 0.05 * k) for k in range(-9, 25)])

    def load(c):
        c.prior_map_load(W["blob"])

    def build(c):
        c.prior_map_build(maps[0], maps[1])

    calls = [(load, small, f["less_sharp"], f["less_flat"], 1), (None, large, f["less_sharp"], f["less_flat"], 16),
             (None, small, f["less_sharp"], f["less_flat"], 3), (build, lv, scan[0], scan[1], 5),
             ("reload", small, f["less_sharp"], f["less_flat"], 4)]

    def run(c, hyps, a, b, K):
        res, sc = c.prior_relocalise(hyps, a, b, inlier_sq=0.5, max_score_points=256, refine=K)
        return sc.copy(), [(r["hyp"], r["score"], r["refined_score"], r["flags"], r["pose"].tobytes()) for r in res]

    c = TR._ctx(aloam, W["M"], 1, W["ns"])   # the world snapshot's configuration
    seq = []
    for prep, hyps, a, b, K in calls:
        if prep == "reload":
            c.prior_map_clear()
            load(c)
        elif prep is not None:
            prep(c)
        seq.append(run(c, hyps, a, b, K))
    c.close()
    for i, (prep, hyps, a, b, K) in enumerate(calls):
        fresh = TR._ctx(aloam, W["M"], 1, W["ns"])
        (build if prep is build else load)(fresh)
        sc, out = run(fresh, hyps, a, b, K)
        fresh.close()
        assert np.array_equal(seq[i][0], sc) and seq[i][1] == out, i


# --------------------------------------------------------------------------------------------------- 8. stack key overflow
def test_a_stack_key_overflow_writes_the_outputs(aloam):
    """a surf cloud whose stack-filter box needs more than 31 key bits at plane_res (1291^3 > 2^31 voxels while PCL's own test,
    1290^3, passes): ALOAM_ERR_CAPACITY with scores and out written.  The stack is kept unfiltered: two surf points share a voxel
    next to a map point, so each scores on its own where the filtered stack would score their centroid once"""
    corners = np.array([[-0.1] * 3, [515.7] * 3])   # floor(x / 0.4): -1 .. 1289 (1291 voxels), (515.8 / 0.4) + 1 = 1290
    pair = np.array([[100.05, 50.05, 0.05, 2.0], [100.15, 50.15, 0.15, 2.0]], np.float32)   # one 0.4 m voxel
    scan, maps = RC.line_scene()
    flat = np.concatenate([scan[1], np.c_[corners, [2.0, 2.0]].astype(np.float32), pair])
    map_surf = np.concatenate([maps[1], np.array([[100.1, 50.1, 0.1, 7.0]], np.float32)])
    c = _ctx(aloam)
    c.prior_map_build(maps[0], map_surf)
    L = aloam.lib()
    a, ka = aloam._view(scan[0])
    b, kb = aloam._view(flat)
    hyps = np.ascontiguousarray([RC.shift(0.375), RC.IDENT7, RC.FAR_POSE])
    opts = aloam.RelocOpts(0.25, 1 << 20, 2)
    out = (aloam.RelocResult * 2)()
    for r in out:
        r.hyp, r.score, r.refined_score, r.flags = -7, -7, -7, -7
    sc = np.full(3, -7, np.int32)
    rc = L.aloam_prior_relocalise(c._h, a, b, aloam._dp(hyps), 3, C.byref(opts), sc.ctypes.data_as(C.POINTER(C.c_int)), out)
    assert rc == ERR_CAPACITY, rc
    corner_stack = pyoracle.voxel_grid(scan[0], LEAVES[0])
    brute = RC.brute_score(maps[0], map_surf, (corner_stack, flat), hyps, 0.25)
    filtered = RC.brute_score(maps[0], map_surf, (corner_stack, pyoracle.voxel_grid(flat, LEAVES[1])), hyps, 0.25)
    assert (brute[:2] == filtered[:2] + 1).all()   # the pair scores twice unfiltered, its centroid once filtered
    assert np.array_equal(sc, brute), (sc, brute, filtered)
    assert sorted(r.hyp for r in out) == [0, 1]
    rank = RC.host_top(sc, 2).tolist()
    keys = []
    for r in out:
        pose = np.array(r.pose[:])
        assert r.score == sc[r.hyp] and r.flags == aloam.FLAG_MAP_TOO_THIN   # 16 surf map points: a thin window
        assert np.array_equal(pose, RC.normalised(hyps[r.hyp])[0])
        assert r.refined_score == RC.brute_score(maps[0], map_surf, (corner_stack, flat), pose[None], 0.25)[0]
        keys.append((-r.refined_score, rank.index(r.hyp)))
    assert keys == sorted(keys)
    c.close()
