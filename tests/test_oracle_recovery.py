"""CPU: the constants of the recovery scenario (tests/recovery_cases.py), fixed on the oracle alone, as tests/test_oracle_track_score.py
fixes the lost-track thresholds.  On the VLP-16 world of tests/reloc_cases.py, with recovery at TRIGGER / ACCEPT over the candidate
lattice: the lane armed 45 degrees and 3 m off adopts on its START row and from FRAMES_TO_TRACK on follows the truly armed lane; the
truly armed lane never triggers; the lane armed off the map triggers on every row and never adopts.  The candidates' oracle scores
equal the numpy brute force on a subset, and the host model's pieces hold their defining identities."""
import importlib

import numpy as np
import pytest

import recovery_cases as RV
import reloc_cases as RC
import track_cases as TC

_W = {}


def _world():
    if not _W:
        synth = importlib.import_module("a-loam_b200.synth")
        aloam = importlib.import_module("a-loam_b200")
        scans, feats, poses, frozen = RC.oracle_world(synth)
        _W.update(feats=feats, poses=poses, frozen=frozen, scorer=RC.FrozenScorer(frozen), res=synth.SENSORS["VLP-16"][3:5],
                  D=RV.deltas(aloam))
    return _W


def _run(init):
    W = _world()
    key = tuple(np.round(init, 12))
    if key not in W:
        W[key] = RV.recover_track(W["frozen"], W["scorer"], W["feats"], init, TC.START, len(W["feats"]), W["res"], W["D"])
    return W[key]


def _dev(a, b):
    from lane_refs import deviation
    return deviation(np.array(a), np.array(b))


def test_the_mis_armed_lane_adopts_on_its_start_row_and_tracks():
    W = _world()
    true = _run(W["poses"][TC.START])
    mis = _run(TC.mis_armed(W["poses"][TC.START]))
    assert mis[0]["triggered"] and mis[0]["adopted"], mis[0]
    assert not any(r["triggered"] for r in mis[1:]), [r["score"] for r in mis]
    k = RV.FRAMES_TO_TRACK
    dt, dr = _dev([r["pose"] for r in mis[k:]], [r["pose"] for r in true[k:]])
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    assert all(r["score"] > TC.TRACK_RATIO * r["n_score"] for r in mis[k:]), [(r["score"], r["n_score"]) for r in mis]


def test_the_truly_armed_lane_never_triggers():
    W = _world()
    rows = _run(W["poses"][TC.START])
    assert not any(r["triggered"] for r in rows), [(r["score"], r["n_score"]) for r in rows]


def test_the_off_map_lane_triggers_on_every_row_and_never_adopts():
    W = _world()
    rows = _run(TC.off_map(W["poses"][TC.START]))
    assert all(r["triggered"] and not r["adopted"] and r["best_score"] == 0 and r["best"] == 0 for r in rows)


def test_candidate_scores_on_a_subset_equal_the_brute_force():
    """the START row's candidates of the mis-armed lane: the best and every 97th, scored by the oracle and by the brute force"""
    W = _world()
    mis = _run(TC.mis_armed(W["poses"][TC.START]))
    f = W["feats"][TC.START]
    sp = RC.scoring_points(f.less_sharp, f.less_flat, TC.PTS, *W["res"])
    cand = RV.candidates(mis[0]["pose"], W["D"])
    idx = sorted(set(range(0, len(cand), 97)) | {mis[0]["best"]})
    got = W["scorer"].score_points(sp, cand[idx], TC.ISQ, normalise=False)
    mc, ms = RC.map_clouds(W["frozen"])
    assert np.array_equal(got, RC.brute_score(mc, ms, sp, cand[idx], TC.ISQ))
    assert got[idx.index(mis[0]["best"])] == mis[0]["best_score"]


def test_the_host_model_pieces():
    rng = np.random.default_rng(5)
    P = np.concatenate([RV.normalise(rng.normal(size=4)), rng.normal(size=3)])
    D = np.concatenate([rng.normal(size=(50, 4)), rng.normal(size=(50, 3))], axis=1)
    C = RV.candidates(P, D)
    # headings turn about the sensor's position, offsets are in the map frame
    assert np.array_equal(C[:, 4:], P[4:] + D[:, 4:])
    assert np.allclose(np.linalg.norm(C[:, :4], axis=1), 1.0, atol=1e-15)
    # the identity delta gives the pose itself (normalised)
    assert np.allclose(RV.candidates(P, np.array([[0, 0, 0, 1.0, 0, 0, 0]]))[0], P, atol=1e-15)
    # transformUpdate: T * odom = x
    x = C[0]
    odom = np.concatenate([RV.normalise(rng.normal(size=4)), rng.normal(size=3)])
    T = RV.transform_update(x, odom)
    back = np.concatenate([RV.qmul(T[:4], odom[:4]), RV.qrot(T[:4], odom[4:]) + T[4:]])
    assert np.allclose(back, x, atol=1e-12)
    # the float32 tests at their edges
    assert RV.triggers(255, 512, 0.5) and not RV.triggers(256, 512, 0.5) and not RV.triggers(0, 0, 1.0)
    assert RV.accepts(384, 0, 512, 0.75) and not RV.accepts(383, 0, 512, 0.75) and not RV.accepts(10, 10, 10, 0.0)
    assert RV.best_of(np.array([3, 7, 7, 1])) == (1, 7)


@pytest.mark.parametrize("frac", [0.0, 1.0])
def test_trigger_fractions_at_the_ends(frac):
    """trigger_frac 0 never triggers; 1 triggers every row that misses a point"""
    assert RV.triggers(0, 10, frac) == (frac == 1.0)
    assert not RV.triggers(10, 10, frac)
