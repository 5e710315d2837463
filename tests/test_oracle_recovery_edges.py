"""CPU: the scenes of the recovery edge-case tests (tests/recovery_edge_cases.py, used by tests/test_gpu_recovery_edges.py) have the
properties the GPU tests rely on: every f_lo / f_hi pair is adjacent in float32 and straddles the trigger and accept tests of the
host model; the vectorised hypotheses are the host model's bits; on the oracle the gate scenario triggers as claimed and a lane's
stale candidates score differently on later scans; the 16-lane schedule puts localising records off their lanes; the lost armings
lose track and the spread armings spread; the size and tie layouts land where they claim for any SM count; records stage once and
in chunks; the far deltas score 0 and the odd ones normalise."""
import numpy as np
import pytest

import pyfrozen
import recovery_cases as RV
import recovery_edge_cases as RE
import reloc_cases as RC
import track_cases as TC
import track_edge_cases as TE
from test_oracle_recovery import _world

F32 = np.float32


@pytest.mark.parametrize("n", [1, 7, 300, 512, 513, 600, 2048, 5214, 30256])
def test_fraction_pairs_are_adjacent_and_straddle_the_decision(n):
    scores = range(n) if n <= 2048 else sorted(set(np.random.default_rng(n).integers(0, n, 700).tolist()) | {0, 1, n - 1})
    n_exact = 0
    for s in scores:
        lo, hi = RE.frac_pair(s, n)
        assert lo.dtype == np.float32 and np.nextafter(lo, F32(2)) == hi and F32(0) <= lo < hi <= F32(1), (s, n)
        # the row (s, n) does not trigger at f_lo and triggers at f_hi
        assert not RV.triggers(s, n, lo) and RV.triggers(s, n, hi), (s, n, lo, hi)
        # a best score s above the row's score is accepted at f_lo and not at f_hi
        if s > 0:
            assert RV.accepts(s, s - 1, n, lo) and not RV.accepts(s, s - 1, n, hi), (s, n)
        n_exact += int(lo * F32(n) == F32(s))
    if n in (512, 2048):   # a power of two: score == f_lo * n exactly on every row
        assert n_exact == len(scores)
    if n == 600:           # and not on every row otherwise
        assert 0 < n_exact < len(scores)


def test_a_zero_score_triggers_at_the_smallest_float():
    lo, hi = RE.frac_pair(0, 512)
    assert lo == 0 and hi == np.nextafter(F32(0), F32(1)) and RV.triggers(0, 512, hi) and not RV.triggers(0, 512, lo)


def test_vectorised_hypotheses_are_the_host_models_bits(aloam):
    P = np.concatenate([RV.normalise(np.random.default_rng(1).normal(size=4)), [12.5, -3.25, 0.75]])
    D = np.concatenate([RE.random_deltas(500), RE.far_deltas(100), RV.deltas(aloam)[::7], np.array([d for _, d in RE.odd_deltas()])])
    assert RE.hypotheses(P, D).tobytes() == RV.products(P, RC.normalised(D)).tobytes()


def test_odd_deltas_normalise_and_reach_their_edges():
    odd = dict(RE.odd_deltas())
    D = np.array(list(odd.values()))
    Dn = RC.normalised(D)
    assert np.isfinite(Dn).all() and np.allclose(np.linalg.norm(Dn[:, :4], axis=1), 1.0, atol=1e-15)
    assert np.linalg.norm(odd["scaled-1e-3"][:4]) < 2e-3 and np.linalg.norm(odd["scaled-1e3"][:4]) > 500
    assert odd["negated"][3] < 0 and odd["half-turn"][3] == 0 and odd["x-axis"][2] == 0 and odd["x-axis"][0] != 0
    assert len(set(odd["111-axis"][:3])) == 1 and np.abs(odd["t+1e4"][4:]).max() == 1e4 and (odd["t-1e4"][4:] == -1e4).all()
    P = np.concatenate([RV.normalise([0.1, -0.2, 0.3, 0.9]), [1.0, 2.0, 3.0]])
    C = RV.candidates(P, D)
    assert np.allclose(np.linalg.norm(C[:, :4], axis=1), 1.0, atol=1e-15)


def test_the_gate_scenario_on_the_oracle():
    """lane A mis-armed triggers on its START row only, lane B off the map on every row; A's START candidates scored on each later
    scan differ from its START-row scores, so scores of a dropped gate would show"""
    W = _world()
    n = 5
    a = RV.recover_track(W["frozen"], W["scorer"], W["feats"], TC.mis_armed(W["poses"][TC.START]), TC.START, TC.START + n, W["res"], W["D"])
    b = RV.recover_track(W["frozen"], W["scorer"], W["feats"], TC.off_map(W["poses"][TC.START]), TC.START, TC.START + n, W["res"], W["D"])
    assert [r["triggered"] for r in a] == [True] + [False] * (n - 1) and a[0]["adopted"]
    assert all(r["triggered"] and not r["adopted"] for r in b)
    cand = RV.candidates(a[0]["pose"], W["D"])
    scores = []
    for j in range(n):
        f = W["feats"][TC.START + j]
        sp = RC.scoring_points(f.less_sharp, f.less_flat, TC.PTS, *W["res"])
        scores.append(W["scorer"].score_points(sp, cand, TC.ISQ, normalise=False))
    assert scores[0].max() == a[0]["best_score"]
    for j in range(1, n):
        assert not np.array_equal(scores[j], scores[0]), j


def test_localising_records_are_not_their_lanes():
    ops, idx = RE.records_schedule(RC.N_MAP + 6)
    armed = RE.records_armed(np.array([0, 0, 0, 1.0, 0, 0, 0]))
    assert set(armed) | set(RE.MAPPING) == set(range(16)) and not set(armed) & set(RE.MAPPING)
    kinds = TE.expected_kinds(ops, armed, RE.SKIP)
    recs = RE.localising_records(kinds)
    moved = sum(1 for r in recs for i, l in r if i != l)
    assert moved >= 0.9 * sum(len(r) for r in recs) and all(any(i != l for i, l in r) for r in recs if r)
    # lanes idle at first, mapping lanes interleaved, skipped rows
    assert (ops[0] == 0).sum() >= 6 and set(np.flatnonzero(kinds[0] == 1)) == set(RE.MAPPING) and (kinds == 3).any()
    # every kind of localising lane has a registered START row whose record is not its lane
    for group in (RE.MIS, RE.OFF, RE.TRUE):
        assert all(any(i != l for i, l in recs[RE.start_step(ll)] if l == ll) for ll in group), group
    assert idx[ops > 0].max() < RC.N_MAP


def _start_rows(W, armings):
    """the oracle's START rows (score, n_score) of lanes armed with `armings` on scan TC.START"""
    f = W["feats"][TC.START]
    sp = RC.scoring_points(f.less_sharp, f.less_flat, TC.PTS, *W["res"])
    out = []
    for a in armings:
        loc = pyfrozen.Localiser(W["frozen"], a[:4], a[4:])
        pose, _ = loc.step(f.less_sharp, f.less_flat, np.array([0, 0, 0, 1.0]), np.zeros(3), *W["res"])
        out.append((int(W["scorer"].score_points(sp, pose[None], TC.ISQ, normalise=False)[0]), len(sp[0]) + len(sp[1])))
    return out


def test_the_lost_armings_lose_track_and_the_spread_armings_spread():
    W = _world()
    lost = _start_rows(W, RE.lost_armings(W["poses"][TC.START]))
    assert all(s < TC.LOST_RATIO * n for s, n in lost), lost
    spread = _start_rows(W, RE.spread_armings(W["poses"][TC.START]))
    ratios = {s / n for s, n in spread if 0 < s < n}
    assert len(ratios) >= 5 and min(ratios) < TC.LOST_RATIO < max(ratios) and any(s == 0 for s, _ in spread), spread


@pytest.mark.parametrize("sms", [16, 78, 114, 132, 144])
def test_size_and_tie_layouts(sms):
    W = RE.wave(sms)
    n = RE.sizes(sms)
    assert n == sorted(n) and len(set(n)) == len(n) and n[-1] < RE.MAX_DELTA and {W - 1, W, W + 1} <= set(n)
    assert RE.ctas(W, sms) == RE.ctas(W + 1, sms) == sms * RE.RELOC_CTAS_PER_SM and RE.ctas(W - 1, sms) == sms * RE.RELOC_CTAS_PER_SM
    # past one wave the grid-stride loop wraps: hypothesis W is the first CTA's again
    assert RE.cta_warp(W, W + 1, sms) == (0, 0) and RE.cta_warp(2 * W + 2, 2 * W + 3, sms)[0] == 0
    # k_recover_cand's last CTA is partial below, at and past one CTA, and around the wave
    assert n[2] == RE.CAND_THREADS and n[1] % RE.CAND_THREADS and n[3] % RE.CAND_THREADS and any(k % RE.CAND_THREADS for k in n[4:])
    nt, early, late = RE.tie_layout(sms)
    ce, we = RE.cta_warp(early, nt, sms)
    cl, wl = RE.cta_warp(late, nt, sms)
    assert early < late < nt and ce < cl == RE.ctas(nt, sms) - 1 and we != wl
    t = RE.tail_layout(sms)
    assert RE.cta_warp(t - 1, t, sms)[0] == RE.ctas(t, sms) - 1 and t % RE.CAND_THREADS


def test_records_stage_once_and_in_chunks(synth):
    m = [sum(min(k, TE.BIG) for k in TE.stacks(synth, "VLP-16", n_az, k, TE.DEFAULT_LEAVES)) for n_az, k in TE.WIDE_LANES]
    assert min(m) <= 2048 < max(m) and sum(x <= 2048 for x in m) >= 3 and sum(x > 2048 for x in m) >= 3, m
    sensor, n_az, index, leaves, mp = TE.LARGE_CASE
    n_c, n_s = TE.stacks(synth, sensor, n_az, index, leaves)
    assert min(n_c, mp) + min(n_s, mp) > 2048 * 10 and n_s > mp


def test_far_deltas_score_zero_and_settings_fit(aloam):
    W = _world()
    P = W["poses"][TC.START]
    f = W["feats"][TC.START]
    sp = RC.scoring_points(f.less_sharp, f.less_flat, TC.PTS, *W["res"])
    D = RE.far_deltas(64)
    assert not W["scorer"].score_points(sp, RV.candidates(P, D), TC.ISQ, normalise=False).any()
    # the lattice's best around the true pose scores well, so a planted copy of it stands out among far deltas
    cand = RV.candidates(P, W["D"])
    assert W["scorer"].score_points(sp, cand, TC.ISQ, normalise=False).max() > TC.TRACK_RATIO * (len(sp[0]) + len(sp[1]))
    sets = RE.settings(aloam)
    assert [len(d) for _, d in sets] == [3, 20808, 5, RE.MAX_DELTA]
    assert all(np.isfinite(RC.normalised(d)).all() for _, d in sets)
    # random deltas' scores agree with the brute force on a subset
    D = RE.random_deltas(16, seed=9)
    c = RV.candidates(TC.mis_armed(P), D)
    mc, ms = RC.map_clouds(W["frozen"])
    assert np.array_equal(W["scorer"].score_points(sp, c, TC.ISQ, normalise=False), RC.brute_score(mc, ms, sp, c, TC.ISQ))
