"""CPU: the oracle's relocalisation score (tests/reloc_cases.py) against an independent numpy brute force, and the recovery scenario
of the GPU tests run on the oracle alone: the synthetic canyon repeats itself (cross walls every 40 m, wall gaps every 20 m, poles
every 10 m), so whether the search region and radius pick the true pose over its translated and turned copies is shown here."""
import importlib

import numpy as np
import pytest

import prior_build_cases as PB
import reloc_cases as RC

LEAVES = (0.2, 0.4)


def _hyps():
    return np.array([[0, 0, 0, 1.0, 0, 0, 0], [0, 0, 0, 1.0, 0, 0.1, 0], [0, 0, 0, 3.0, 30.0, 0, 0], [0, 0, np.sin(0.05), np.cos(0.05), 0.2, -0.1, 0.0]])


@pytest.mark.parametrize("inlier_sq,expect", [(RC.EDGE_SQ, 6), (1.0, 12)])
def test_score_at_the_d2_edges(inlier_sq, expect):
    """d2 == inlier_sq is out, one float below is in, one above is out; neighbours in the next cube and across a cell face count"""
    pts, corner, surf = RC.edge_case_clouds()
    S = RC.FrozenScorer(PB.oracle_build(corner, surf, *LEAVES)[0].frozen())
    got = S.score(pts[0], pts[1], _hyps(), inlier_sq, 1 << 20, *LEAVES)
    assert np.array_equal(got, RC.brute_score(corner, surf, pts, _hyps(), inlier_sq))
    assert got[0] == expect


def test_score_on_an_empty_corner_map():
    pts, corner, surf = RC.edge_case_clouds()
    empty = np.zeros((0, 4), np.float32)
    S = RC.FrozenScorer(PB.oracle_build(empty, surf, *LEAVES)[0].frozen())
    got = S.score(pts[0], pts[1], _hyps(), 1.0, 1 << 20, *LEAVES)
    assert np.array_equal(got, RC.brute_score(empty, surf, pts, _hyps(), 1.0)) and got[0] == 6


@pytest.mark.parametrize("max_pts", [1, 37, 300, 301, 5000])
def test_score_with_stacks_below_at_and_above_max_score_points(max_pts):
    """random clouds (300 corner and 301 surf points after the stack filter, which moves them onto centroids of their voxels) on a
    map made of the same points jittered; the subsample takes stack point floor(i n / m)"""
    rng = np.random.default_rng(5)
    scan = [np.concatenate([rng.uniform(-30, 30, (n, 3)) * [1, 1, 0.1], np.ones((n, 1))], 1).astype(np.float32) for n in (300, 301)]
    stacks = [PB.voxel_model(s, leaf) for s, leaf in zip(scan, LEAVES)]
    assert [len(s) for s in stacks] == [300, 301]
    maps = [(s + np.concatenate([rng.normal(0, 0.4, (len(s), 3)), np.zeros((len(s), 1))], 1)).astype(np.float32) for s in scan]
    S = RC.FrozenScorer(PB.oracle_build(maps[0], maps[1], *LEAVES)[0].frozen())
    pts = RC.scoring_points(scan[0], scan[1], max_pts, *LEAVES)
    assert [len(p) for p in pts] == [min(300, max_pts), min(301, max_pts)]
    m = min(301, max_pts)
    assert np.array_equal(pts[1], stacks[1][[i * 301 // m for i in range(m)]])
    got = S.score(scan[0], scan[1], _hyps(), 0.5, max_pts, *LEAVES)
    assert np.array_equal(got, RC.brute_score(S.clouds[0], S.clouds[1], pts, _hyps(), 0.5))
    assert 0 < got[0] <= len(pts[0]) + len(pts[1])


def test_the_recovery_scenario_picks_the_true_pose():
    """the GPU recovery test's search (reloc_cases: +-10 m at 1 m around a guess 3.7 m off, 72 headings, inlier_sq 0.25, 256 points
    per type) on the oracle's map of the first N_MAP scans: the best hypothesis is the lattice point next to the true pose and
    beats every translated or turned copy by a clear margin; a scan from 160 m further on scores far below it everywhere"""
    import pyoracle
    aloam = importlib.import_module("a-loam_b200")
    synth = importlib.import_module("a-loam_b200.synth")
    scans, feats, poses, frozen = RC.oracle_world(synth)
    S = RC.FrozenScorer(frozen)
    ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
    true = poses[RC.SCAN]
    hyps = RC.search_grid(aloam, true)
    f = feats[RC.SCAN]
    sc = S.score(f.less_sharp, f.less_flat, hyps, RC.INLIER_SQ, RC.MAX_PTS, line_res, plane_res)
    order = np.lexsort((np.arange(len(sc)), -sc))
    best = hyps[order[0]]
    dxy = np.abs(best[4:6] - true[4:6]).max()
    dyaw = abs(RC.yaw_of(best[:4]) - RC.yaw_of(true[:4]))
    assert dxy < 0.15 and dyaw < np.radians(0.2), (dxy, np.degrees(dyaw))
    # every hypothesis more than a metre or 10 degrees away scores at most 80 % of the best
    far = (np.abs(hyps[:, 4:6] - true[4:6]).max(axis=1) > 1.0) | (np.abs(np.angle(np.exp(1j * (RC.yaw_of(hyps[:, :4].T) - RC.yaw_of(true[:4]))))) > np.radians(10))
    assert sc[far].max() < 0.8 * sc[order[0]], (sc[far].max(), sc[order[0]])
    off = pyoracle.Features(synth.scan("VLP-16", RC.OFF_MAP, seed=synth.BASE_SEED + 50, n_az=900), ns, mr)
    so = S.score(off.less_sharp, off.less_flat, hyps, RC.INLIER_SQ, RC.MAX_PTS, line_res, plane_res)
    assert so.max() < RC.OFF_MAP_RATIO * sc.max(), (so.max(), sc.max())
