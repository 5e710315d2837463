"""CPU: the thresholds of the lost-track scenario (tests/track_cases.py), fixed on the oracle alone.  Localising lanes run the frozen
oracle's frames from their own odometry; every frame's map pose is scored as aloam_map_rows scores a localising row.  A lane armed
at a scan's true map pose keeps scoring nearly every scoring point; the same lane armed 45 degrees and 3 m off stays lost and
scores below LOST_RATIO; a lane armed off the map has thin frames and scores 0.  The score is checked against the numpy brute
force at the d^2 edges."""
import importlib

import numpy as np
import pytest

import prior_build_cases as PB
import reloc_cases as RC
import track_cases as TC

_W = {}


def _world():
    if not _W:
        synth = importlib.import_module("a-loam_b200.synth")
        scans, feats, poses, frozen = RC.oracle_world(synth)
        _W.update(feats=feats, poses=poses, frozen=frozen, scorer=RC.FrozenScorer(frozen), res=synth.SENSORS["VLP-16"][3:5])
    return _W


def _run(init):
    W = _world()
    return TC.track(W["frozen"], W["scorer"], W["feats"], init, TC.START, len(W["feats"]), W["res"])


def test_a_lane_armed_at_the_true_pose_keeps_track():
    W = _world()
    poses, infos, sc, n = _run(W["poses"][TC.START])
    assert all(i["optimised"] for i in infos)
    assert (sc > TC.TRACK_RATIO * n).all(), (sc, n)
    # on the mapped stretch it follows the mapping run
    k = RC.N_MAP - TC.START
    dt = np.abs(poses[:k, 4:] - W["poses"][TC.START:, 4:]).max()
    assert dt < 0.1, dt


def test_a_grossly_mis_armed_lane_stays_lost():
    W = _world()
    good = _run(W["poses"][TC.START])[2]
    poses, infos, sc, n = _run(TC.mis_armed(W["poses"][TC.START]))
    assert (sc < TC.LOST_RATIO * n).all(), (sc, n)
    assert (sc < 0.6 * good).all(), (sc, good)
    # and its map poses stay far from the true ones
    k = RC.N_MAP - TC.START
    assert np.abs(poses[:k, 4:6] - W["poses"][TC.START:, 4:6]).max(axis=1).min() > 1.0


def test_a_lane_armed_off_the_map_is_thin_and_scores_zero():
    W = _world()
    poses, infos, sc, n = _run(TC.off_map(W["poses"][TC.START]))
    assert not any(i["optimised"] for i in infos)
    assert (sc == 0).all() and (n > 0).all()


@pytest.mark.parametrize("inlier_sq", [RC.EDGE_SQ, 1.0])
def test_the_score_at_the_d2_edges_equals_the_brute_force(inlier_sq):
    """the crafted edge map at tracked poses (not normalised, as a row's map pose is scored): float d2 == inlier_sq is out, one
    float below is in"""
    pts, corner, surf = RC.edge_case_clouds()
    S = RC.FrozenScorer(PB.oracle_build(corner, surf, 0.2, 0.4)[0].frozen())
    poses = np.array([[0, 0, 0, 1.0, 0, 0, 0], [0, 0, 0, 1.0, 0, 0.1, 0], [0, 0, np.sin(0.01), np.cos(0.01), 0.05, 0, 0]])
    got = S.score(pts[0], pts[1], poses, inlier_sq, 1 << 20, 0.2, 0.4, normalise=False)
    assert np.array_equal(got, RC.brute_score(corner, surf, pts, poses, inlier_sq))
    assert got[0] == (6 if inlier_sq == RC.EDGE_SQ else 12)
