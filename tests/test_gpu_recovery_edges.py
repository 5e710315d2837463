"""GPU parity at the edges of the recovery of localising lanes (recover.cu: k_recover_cand; reloc.cu: the gated multi-record
k_reloc_score / k_reloc_topk; cubemap.cu: k_recover_adopt), on the VLP-16 world of tests/test_gpu_map_rows.py.  The scenes are in
tests/recovery_edge_cases.py, whose properties tests/test_oracle_recovery_edges.py checks on the CPU.
  * A: the trigger and accept tests at their float32 boundaries (f_lo and the next float up, exact products included), and the
    identity candidate tied with the row's own k_track_score score (never adopted);
  * B: a 16-lane call at mapping_skip_frame 2 whose localising records are not its lanes, against solo runs, and the gate: a lane
    that triggered once keeps that row's scores while another lane triggers on every later frame;
  * C: n_delta of 1 .. 2W + 3 around one resident wave W of k_reloc_score and 65 536 over 16 triggering lanes, ties across CTAs
    and a winner at n - 1, records that stage once and in chunks in one launch (and an HDL-64 stack subsampled at 30 000), odd
    deltas;
  * D: re-setting recovery over a context's life against fresh contexts, and a row whose stack filter overflows its key.
References: the host model of tests/recovery_cases.py bit for bit, aloam_prior_relocalise's coarse scores of the host-composed
hypotheses on the row's scan (integer-equal), and the oracle scorer and numpy brute force on subsets of the candidates."""
import ctypes as C

import numpy as np
import pytest

import recovery_cases as RV
import recovery_edge_cases as RE
import reloc_cases as RC
import test_gpu_map_rows as MR
import test_gpu_track_edges as TG
import track_cases as TC
import track_edge_cases as TE

pytestmark = pytest.mark.gpu

ROW_KEYS = ("kind", "err", "n_valid", "score", "n_score", "flags", "lm_iters", "init_cost", "final_cost")
LARGE_STAGE = 2048   # k_reloc_score stages at most this many scoring points at once (kRelocStage)


@pytest.fixture(scope="module")
def world(aloam, synth):
    return MR._world(aloam, synth)


@pytest.fixture(scope="module")
def sms():
    import torch
    n = torch.cuda.get_device_properties(0).multi_processor_count
    print("\nk_reloc_score: %d SMs x %d CTAs per SM (its launch bound) x %d warps: one resident wave W = %d hypotheses"
          % (n, RE.RELOC_CTAS_PER_SM, RE.RELOC_WARPS, RE.wave(n)))
    return n


def _arm(c, inits):
    for lane, init in inits.items():
        c.lane_localise(lane, init[:4], init[4:])


def _start_all(c, W, armings, scan=TC.START):
    """every lane of the context armed and STARTed on the same scan in one step -> (odometry, map poses, rows)"""
    _arm(c, dict(enumerate(armings)))
    d = W["dev"][scan]
    return MR._call(c, len(armings), {l: [(d.data_ptr(), d.shape[0], MR.START)] for l in range(len(armings))})


def _ref_scores(c, P, D, f, mp=TC.PTS, isq=TC.ISQ):
    """aloam_prior_relocalise's coarse scores of the candidates around map pose P on the scan with features f"""
    _, sc = c.prior_relocalise(RE.hypotheses(P, D), f["less_sharp"], f["less_flat"], inlier_sq=isq, max_score_points=mp, refine=1)
    return sc


def _T(c, lane):
    st = c.mapper_state(lane)
    return np.concatenate([st["q_wmap_wodom"], st["t_wmap_wodom"]])


def _check_best(c, rec, r, row_score, n_score, P, odom, D, ref, accept, lane, what):
    """a triggered row's best candidate, score, pose and adoption against the host model on the reference scores; the adopted
    T_wmap_wodom against transformUpdate bit for bit"""
    h, bs = RV.best_of(ref)
    assert (rec["best"][r], rec["best_score"][r]) == (h, bs), (what, rec["best"][r], rec["best_score"][r], h, bs)
    cand = RV.candidates(P, D[h:h + 1])[0]
    assert rec["pose"][r].tobytes() == cand.tobytes(), (what, rec["pose"][r], cand)
    assert bool(rec["adopted"][r]) == RV.accepts(bs, row_score, n_score, accept), (what, bs, row_score, n_score)
    if rec["adopted"][r]:
        T = _T(c, lane)
        assert T.tobytes() == RV.transform_update(cand, odom).tobytes(), (what, T)
    return h, bs


# ------------------------------------------------------------------------------------------------ A. float boundaries
@pytest.fixture(scope="module")
def spread(aloam, world):
    """a 16-lane localiser and the spread armings of the START scan"""
    c = MR._localiser(aloam, world, 16)
    yield c, RE.spread_armings(world["map"][TC.START])
    c.close()


def _chosen(scores, n, k=3):
    """up to k rows with 0 < score < n and distinct ratios: the lowest, the middle and the highest ratio"""
    cand = sorted({(s / m, int(s), int(m)) for s, m in zip(scores, n) if 0 < s < m})
    if len(cand) <= k:
        return [(s, m) for _, s, m in cand]
    return [(cand[i][1], cand[i][2]) for i in (0, len(cand) // 2, len(cand) - 1)]


@pytest.mark.parametrize("mp", [TC.PTS, 300])
def test_trigger_flips_at_its_float_boundary(aloam, world, spread, mp):
    """START rows learnt with recovery off; for chosen rows f_lo (largest float with f * n <= score: no trigger) and f_hi = the
    next float (trigger).  Every row of every run equals the learnt one and triggers exactly as the host model says; at
    max_score_points 256 n = 512 and f_lo * n == score exactly; a zero score triggers at the smallest positive float"""
    c, arms = spread
    c.set_map_rows(True, TC.ISQ, mp)
    c.set_recovery(False)
    _, m0, base = _start_all(c, world, arms)
    pairs = _chosen(base["score"], base["n_score"])
    assert len(pairs) == 3, (base["score"], base["n_score"])
    if mp == TC.PTS:
        z = [int(n) for s, n in zip(base["score"], base["n_score"]) if s == 0 and n > 0]
        assert z, base["score"]
        pairs.append((0, z[0]))
    exact = 0
    D = RV.deltas(aloam)
    for score, n in pairs:
        lo, hi = RE.frac_pair(score, n)
        exact += int(lo * np.float32(n) == np.float32(score))
        for f, want in ((lo, False), (hi, True)):
            c.set_recovery(True, f, 1.0, D)
            _, m, rows = _start_all(c, world, arms)
            rec = c.recovery_rows(16)
            assert np.array_equal(m, m0)
            for k in ROW_KEYS:
                assert np.array_equal(rows[k], base[k]), (k, f)
            trig = [RV.triggers(s, k, f) for s, k in zip(rows["score"], rows["n_score"])]
            assert list(rec["triggered"].astype(bool)) == trig, (score, n, float(f), rec["triggered"], trig)
            hit = [l for l in range(16) if rows["score"][l] == score and rows["n_score"][l] == n]
            assert all(bool(rec["triggered"][l]) == want for l in hit) and hit, (score, n, float(f))
    if mp == TC.PTS:
        assert exact == len(pairs), exact


def test_accept_flips_at_its_float_boundary(aloam, world, spread):
    """best scores learnt at trigger_frac 1, accept_frac 1; for chosen rows a_lo (largest float with a * n <= best_score: adopts)
    and the next float (does not).  Adoption follows the host model on every row, and an adopted T_wmap_wodom is transformUpdate
    at the best candidate with the row's odometry pose, bit for bit"""
    c, arms = spread
    D = RV.deltas(aloam)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, 1.0, 1.0, D)
    _, m0, base = _start_all(c, world, arms)
    rec0 = c.recovery_rows(16)
    ok = [l for l in range(16) if rec0["triggered"][l] and base["score"][l] < rec0["best_score"][l] < base["n_score"][l]]
    pairs = _chosen(rec0["best_score"][ok], base["n_score"][ok])
    assert len(pairs) >= 2, (rec0["best_score"], base["score"])
    n_adopted = 0
    for bs, n in pairs:
        lo, hi = RE.frac_pair(bs, n)
        for a, want in ((lo, True), (hi, False)):
            c.set_recovery(True, 1.0, a, D)
            o, m, rows = _start_all(c, world, arms)
            rec = c.recovery_rows(16)
            assert np.array_equal(m, m0) and np.array_equal(rows["score"], base["score"])
            for k in ("triggered", "best", "best_score", "pose"):
                assert np.array_equal(rec[k], rec0[k]), (k, float(a))
            for l in range(16):
                if not rec["triggered"][l]:
                    continue
                assert bool(rec["adopted"][l]) == RV.accepts(rec["best_score"][l], rows["score"][l], rows["n_score"][l], a), (l, float(a))
                if rec["adopted"][l]:
                    T = _T(c, l)
                    assert T.tobytes() == RV.transform_update(rec["pose"][l], o[0, l]).tobytes(), (l, T)
                    n_adopted += 1
                if l in ok and rec["best_score"][l] == bs and rows["n_score"][l] == n:
                    assert bool(rec["adopted"][l]) == want, (bs, n, float(a), l)
    assert n_adopted > 0


def test_the_identity_candidate_ties_with_the_row(aloam, world, spread):
    """deltas = [identity], trigger_frac 1, accept_frac 0: on rows whose map pose is a fixed point of the normalisation the
    candidate is the map pose itself, so k_reloc_score's score equals k_track_score's; s > score is strict, so none adopts"""
    c, arms = spread
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, 1.0, 0.0, np.array([[0, 0, 0, 1.0, 0, 0, 0]]))
    _, m, rows = _start_all(c, world, arms)
    rec = c.recovery_rows(16)
    n_fixed = 0
    for l in range(16):
        trig = RV.triggers(rows["score"][l], rows["n_score"][l], 1.0)
        assert bool(rec["triggered"][l]) == trig, l
        if not trig:
            continue
        assert bool(rec["adopted"][l]) == (rec["best_score"][l] > rows["score"][l]), l
        if TG._fixed_point(m[0, l]):
            assert rec["pose"][l].tobytes() == m[0, l].tobytes(), l
            sc = c.debug_recovery_scores(l)
            assert sc[0] == rows["score"][l] == rec["best_score"][l] and not rec["adopted"][l], (l, sc, rows["score"][l])
            n_fixed += 1
    assert n_fixed >= 1, n_fixed


# ---------------------------------------------------------------------------------------- B. records that are not lanes
def _records_run(aloam, W, D, lanes, batch):
    """lanes: {slot: lane of RE's schedule}; the schedule's columns on a context of `batch` lanes at mapping_skip_frame 2 ->
    (odometry, map poses, rows, recovery rows, debug scores per slot or None)"""
    ops, idx = RE.records_schedule(len(W["dev"]))
    armed = RE.records_armed(W["map"][TC.START])
    c = TG._world_ctx(aloam, W, "VLP-16", W["res"], batch, W["M"], mapping_skip_frame=RE.SKIP)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
    _arm(c, {s: armed[l] for s, l in lanes.items() if l in armed})
    entries = {s: [(W["dev"][idx[k, l]].data_ptr(), W["dev"][idx[k, l]].shape[0], int(ops[k, l])) if ops[k, l] else (0, 0, MR.IDLE)
                   for k in range(RE.STEPS)] for s, l in lanes.items()}
    o, m, rows = MR._call(c, batch, entries)
    rec = c.recovery_rows(RE.STEPS * batch)
    dbg = {}
    for s in lanes:
        try:
            dbg[s] = c.debug_recovery_scores(s)
        except aloam.AloamError as e:
            assert e.code == MR.ERR_STATE, e.code
            dbg[s] = None
    return c, (o, m, rows, rec, dbg), ops, idx


def test_records_that_are_not_lanes(aloam, world):
    """16 lanes, mapping lanes 0 / 5 / 10 among them, localising lanes STARTed at steps 0, 1 and 2 (idle before), at
    mapping_skip_frame 2: localising record l is not lane l on most frames.  Every lane equals its solo run (poses, rows,
    recovery rows, debug scores); a lane's debug scores are aloam_prior_relocalise's at its latest triggered row; lanes with no
    triggered row answer ALOAM_ERR_STATE"""
    W = world
    D = RV.deltas(aloam)
    c, (o, m, rows, rec, dbg), ops, idx = _records_run(aloam, W, D, {l: l for l in range(16)}, 16)
    kinds = rows["kind"].reshape(RE.STEPS, 16)
    want = TE.expected_kinds(ops, RE.records_armed(W["map"][TC.START]), RE.SKIP, aloam.ROW_IDLE, aloam.ROW_MAPPED,
                             aloam.ROW_LOCALISED, aloam.ROW_SKIPPED)
    assert np.array_equal(kinds, want)
    trig = rec["triggered"].reshape(RE.STEPS, 16)
    moved = [(k, i, l) for k, recs in enumerate(RE.localising_records(kinds, aloam.ROW_LOCALISED)) for i, l in recs if trig[k, l] and i != l]
    assert len(moved) >= 6, moved
    assert trig[:, list(RE.MIS)].sum(axis=0).min() >= 1 and not trig[:, list(RE.TRUE)].any() and not trig[:, list(RE.MAPPING)].any()
    assert rec["adopted"].reshape(RE.STEPS, 16)[:, list(RE.MIS)].any(axis=0).all()
    for l in RE.OFF:
        assert (trig[:, l] == (kinds[:, l] == aloam.ROW_LOCALISED)).all(), l
    latest_moved = 0
    for l in range(16):
        ks = np.flatnonzero(trig[:, l])
        if not len(ks):
            assert dbg[l] is None, l
            continue
        k = int(ks[-1])
        ref = _ref_scores(c, m[k, l], D, W["feats"][idx[k, l]])
        assert dbg[l] is not None and np.array_equal(dbg[l], ref), (l, k)
        latest_moved += int(any(kk == k and ll == l for kk, _, ll in moved))
    assert latest_moved >= 3, latest_moved
    c.close()
    for l in range(16):
        s, (so, sm, srows, srec, sdbg), _, _ = _records_run(aloam, W, D, {0: l}, 1)
        s.close()
        assert np.array_equal(o[:, l], so[:, 0], equal_nan=True) and np.array_equal(m[:, l], sm[:, 0], equal_nan=True), l
        for k in ROW_KEYS:
            assert np.array_equal(rows[k].reshape(RE.STEPS, 16)[:, l], srows[k]), (l, k)
        for k in srec:
            assert np.array_equal(rec[k].reshape((RE.STEPS, 16) + rec[k].shape[1:])[:, l], srec[k]), (l, k)
        assert (dbg[l] is None) == (sdbg[0] is None) and (dbg[l] is None or np.array_equal(dbg[l], sdbg[0])), l


def test_the_gate_keeps_an_untriggered_lanes_scores(aloam, world):
    """lane 0 mis-armed triggers and adopts on its START row only; lane 1 off the map triggers on every row, so every later frame's
    gated k_reloc_score runs with lane 0's record gated off.  Lane 0's scores stay those of its START row -- which differ from its
    stale candidates scored on any later scan -- and lane 1's are those of its last row"""
    W = world
    D = RV.deltas(aloam)
    n = 5
    c = MR._localiser(aloam, W, 2)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
    true = W["map"][TC.START]
    _arm(c, {0: TC.mis_armed(true), 1: TC.off_map(true)})
    o, m, rows = MR._call(c, 2, {l: MR._entries(W["dev"], TC.START, TC.START + n) for l in range(2)})
    rec = c.recovery_rows(2 * n)
    assert list(rec["triggered"][0::2]) == [1] + [0] * (n - 1) and rec["adopted"][0], rec["triggered"]
    assert rec["triggered"][1::2].all()
    a, b = c.debug_recovery_scores(0), c.debug_recovery_scores(1)
    ref = _ref_scores(c, m[0, 0], D, W["feats"][TC.START])
    assert np.array_equal(a, ref)
    assert np.array_equal(b, _ref_scores(c, m[n - 1, 1], D, W["feats"][TC.START + n - 1]))
    for j in range(1, n):
        stale = _ref_scores(c, m[0, 0], D, W["feats"][TC.START + j])
        assert not np.array_equal(stale, ref), j
    c.close()


# ---------------------------------------------------------------------------------------------------- C. candidate sets
@pytest.fixture(scope="module")
def pair_ctx(aloam, world):
    """a 2-lane localiser: lane 0 mis-armed, lane 1 a few degrees and tenths of a metre off"""
    c = MR._localiser(aloam, world, 2)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    true = world["map"][TC.START]
    yield c, [TC.mis_armed(true), RE.turned(true, 8.0, (0.6, -0.4, 0.0))]
    c.close()


def _pair_run(c, W, arms, D, trigger=1.0, accept=RV.ACCEPT):
    c.set_recovery(True, trigger, accept, D)
    o, m, rows = _start_all(c, W, arms)
    return o, m, rows, c.recovery_rows(len(arms))


SIZE_NAMES = ["1", "255", "256", "257", "W-1", "W", "W+1", "2W+3"]


@pytest.mark.parametrize("name", SIZE_NAMES)
def test_candidate_set_sizes(aloam, world, pair_ctx, sms, name):
    """n_delta around k_recover_cand's 256-thread CTAs and one resident wave W of k_reloc_score (the grid-stride loop wraps past
    W): every score of every triggered lane equals aloam_prior_relocalise's, best / best_score / pose / adoption the host model's"""
    c, arms = pair_ctx
    n = RE.sizes(sms)[SIZE_NAMES.index(name)]
    D = RE.random_deltas(n, seed=n)
    o, m, rows, rec = _pair_run(c, world, arms, D)
    assert rec["triggered"][0], rows["score"]
    f = world["feats"][TC.START]
    for l in range(2):
        if not rec["triggered"][l]:
            continue
        sc = c.debug_recovery_scores(l)
        ref = _ref_scores(c, m[0, l], D, f)
        assert len(sc) == n and np.array_equal(sc, ref), (name, l, np.flatnonzero(sc != ref)[:8])
        _check_best(c, rec, l, rows["score"][l], rows["n_score"][l], m[0, l], o[0, l], D, ref, RV.ACCEPT, l, (name, l))


def test_the_limit_over_sixteen_triggering_lanes(aloam, world):
    """n_delta 65 536 and 16 lanes that all trigger on their START rows in one step (one k_reloc_score launch of 16 x 65 536
    candidates): every lane's scores equal aloam_prior_relocalise's, its best the host model's; on subsets the oracle scorer and
    the brute force agree"""
    W = world
    D = RE.random_deltas(RE.MAX_DELTA, seed=11)
    c = MR._localiser(aloam, W, 16)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, 1.0, RV.ACCEPT, D)
    o, m, rows = _start_all(c, W, RE.lost_armings(W["map"][TC.START]))
    rec = c.recovery_rows(16)
    assert rec["triggered"].all(), (rows["score"], rows["n_score"])
    scores = [c.debug_recovery_scores(l) for l in range(16)]
    f = W["feats"][TC.START]
    sp = RC.scoring_points(f["less_sharp"], f["less_flat"], TC.PTS, *W["res"])
    mc, ms = RC.map_clouds(W["frozen"])
    rng = np.random.default_rng(3)
    for l in range(16):
        ref = _ref_scores(c, m[0, l], D, f)
        assert np.array_equal(scores[l], ref), (l, np.flatnonzero(scores[l] != ref)[:8])
        h, _ = _check_best(c, rec, l, rows["score"][l], rows["n_score"][l], m[0, l], o[0, l], D, ref, RV.ACCEPT, l, l)
        if l in (0, 7):
            idx = np.unique(np.r_[rng.choice(RE.MAX_DELTA, 300, replace=False), h, RE.MAX_DELTA - 1])
            cand = RV.candidates(m[0, l], D[idx])
            assert np.array_equal(W["scorer"].score_points(sp, cand, TC.ISQ, normalise=False), scores[l][idx]), l
            few = idx[:12].tolist() + [h]
            assert np.array_equal(RC.brute_score(mc, ms, sp, RV.candidates(m[0, l], D[few]), TC.ISQ), scores[l][few]), l
    c.close()


def test_ties_across_ctas_and_the_last_candidate(aloam, world, pair_ctx, sms):
    """the best delta of the recovery lattice for the mis-armed lane's START row planted among deltas that score 0: at `late`
    (last CTA of the first wave) and `early` < late (another CTA and warp) the best is `early`; planted at n - 1 alone (the last
    CTA, k_recover_cand's partial last CTA) it is n - 1; a lane whose every score is 0 has best 0"""
    c, arms = pair_ctx
    arms = [arms[0], TC.off_map(world["map"][TC.START])]
    f = world["feats"][TC.START]
    D0 = RV.deltas(aloam)
    _, m0, _, rec0 = _pair_run(c, world, arms, D0)
    h0, bs0 = int(rec0["best"][0]), int(rec0["best_score"][0])
    assert bs0 > 0 and rec0["triggered"].all()
    n, early, late = RE.tie_layout(sms)
    assert RE.cta_warp(early, n, sms)[0] != RE.cta_warp(late, n, sms)[0] and RE.cta_warp(early, n, sms)[1] != RE.cta_warp(late, n, sms)[1]
    nt = RE.tail_layout(sms)
    assert RE.cta_warp(nt - 1, nt, sms)[0] == RE.ctas(nt, sms) - 1 and nt % RE.CAND_THREADS
    for D, want in ((RE.far_deltas(n), (early, late)), (RE.far_deltas(nt, seed=1), (nt - 1,)), (RE.far_deltas(nt, seed=2), ())):
        for h in want:
            D[h] = D0[h0]
        o, m, rows, rec = _pair_run(c, world, arms, D)
        assert np.array_equal(m, m0) and rec["triggered"].all()
        sc = c.debug_recovery_scores(0)
        ref = _ref_scores(c, m[0, 0], D, f)
        assert np.array_equal(sc, ref), np.flatnonzero(sc != ref)[:8]
        assert sorted(np.flatnonzero(ref == ref.max()).tolist()) == (list(want) if want else list(range(len(D)))), want
        _check_best(c, rec, 0, rows["score"][0], rows["n_score"][0], m[0, 0], o[0, 0], D, ref, RV.ACCEPT, 0, want)
        assert (rec["best"][0], rec["best_score"][0]) == ((min(want), bs0) if want else (0, 0)), (rec["best"][0], want)
        assert (rec["best"][1], rec["best_score"][1]) == (0, 0) and not c.debug_recovery_scores(1).any()


def test_records_that_stage_once_and_in_chunks_share_a_launch(aloam, synth, world):
    """16 lanes START on the 16 scans of TE.WIDE_LANES at max_score_points above every stack and trigger_frac 1: records of at
    most 2048 scoring points (staged once) and of more (staged in chunks) in one gated k_reloc_score launch, each lane's scores
    aloam_prior_relocalise's at the same max_score_points; then one HDL-64 lane subsampled at 30 000 points"""
    import torch
    W = world
    D = RE.random_deltas(48, seed=2)
    raws = [TE.raw_scan(synth, "VLP-16", n_az, k) for n_az, k in TE.WIDE_LANES]
    c = TG._world_ctx(aloam, W, "VLP-16", TE.DEFAULT_LEAVES, 16, max(r.shape[0] for r in raws) + 1024)
    c.set_map_rows(True, TC.ISQ, TE.BIG)
    c.set_recovery(True, 1.0, RV.ACCEPT, D)
    for l, (_, k) in enumerate(TE.WIDE_LANES):
        T = TC.off_map(W["map"][k]) if l == TE.WIDE_OFF else W["map"][k]
        c.lane_localise(l, T[:4], T[4:])
    dev = [torch.from_numpy(r).cuda() for r in raws]
    o, m, rows = TG._start(c, 16, dev, [(l, l) for l in range(16)])
    rec = c.recovery_rows(16)
    scores = {l: c.debug_recovery_scores(l) for l in range(16) if rec["triggered"][l]}
    kinds = set()
    for l in range(16):
        assert bool(rec["triggered"][l]) == RV.triggers(rows["score"][l], rows["n_score"][l], 1.0), l
        if not rec["triggered"][l]:
            MR._expect(aloam, MR.ERR_STATE, lambda: c.debug_recovery_scores(l))
            continue
        _, ref = c.prior_relocalise(RE.hypotheses(m[0, l], D), raw=raws[l], inlier_sq=TC.ISQ, max_score_points=TE.BIG, refine=1)
        assert np.array_equal(scores[l], ref), (l, scores[l], ref)
        _check_best(c, rec, l, rows["score"][l], rows["n_score"][l], m[0, l], o[0, l], D, ref, RV.ACCEPT, l, l)
        kinds.add(rows["n_score"][l] > LARGE_STAGE)
    assert kinds == {False, True}, kinds
    c.close()
    sensor, n_az, index, leaves, mp = TE.LARGE_CASE
    raw = TE.raw_scan(synth, sensor, n_az, index)
    c = TG._world_ctx(aloam, W, sensor, leaves, 1, 262144)
    c.set_map_rows(True, TC.ISQ, mp)
    c.set_recovery(True, 1.0, RV.ACCEPT, D[:16])
    T = W["map"][index]
    c.lane_localise(0, T[:4], T[4:])
    o, m, rows = TG._start(c, 1, [torch.from_numpy(raw).cuda()], [(0, 0)])
    rec = c.recovery_rows(1)
    assert rec["triggered"][0] and rows["n_stack"][0][1] >= TE.LARGE_MIN and rows["n_score"][0] > mp, (rows["n_stack"], rows["score"])
    sc = c.debug_recovery_scores(0)
    _, ref = c.prior_relocalise(RE.hypotheses(m[0, 0], D[:16]), raw=raw, inlier_sq=TC.ISQ, max_score_points=mp, refine=1)
    assert np.array_equal(sc, ref), (sc, ref)
    _check_best(c, rec, 0, rows["score"][0], rows["n_score"][0], m[0, 0], o[0, 0], D[:16], ref, RV.ACCEPT, 0, "HDL-64")
    c.close()


def test_odd_deltas(aloam, world, pair_ctx):
    """quaternions scaled by 1e-3 and 1e3, negated, a half turn (w = 0), turns about x and (1, 1, 1), translations of +-1e4: each
    alone, the reported candidate pose is the host model's bit for bit and its score aloam_prior_relocalise's; all together,
    every score and the best"""
    c, arms = pair_ctx
    f = world["feats"][TC.START]
    odd = RE.odd_deltas()
    for name, d in odd:
        D = d[None]
        o, m, rows, rec = _pair_run(c, world, arms, D)
        assert rec["triggered"][0], name
        for l in range(2):
            if not rec["triggered"][l]:
                continue
            assert rec["best"][l] == 0, (name, l)
            cand = RV.candidates(m[0, l], D)[0]
            assert rec["pose"][l].tobytes() == cand.tobytes(), (name, l, rec["pose"][l], cand)
            ref = _ref_scores(c, m[0, l], D, f)
            assert np.array_equal(c.debug_recovery_scores(l), ref) and rec["best_score"][l] == ref[0], (name, l)
    D = np.array([d for _, d in odd])
    o, m, rows, rec = _pair_run(c, world, arms, D)
    sc = c.debug_recovery_scores(0)
    ref = _ref_scores(c, m[0, 0], D, f)
    assert np.array_equal(sc, ref), (sc, ref)
    _check_best(c, rec, 0, rows["score"][0], rows["n_score"][0], m[0, 0], o[0, 0], D, ref, RV.ACCEPT, 0, "odd")


# ---------------------------------------------------------------------------------------- D. settings over a context's life
def _life_call(aloam, c, W, n=3):
    """lane 0 mis-armed, lane 1 off the map, n scans from TC.START -> everything a caller can read afterwards"""
    true = W["map"][TC.START]
    _arm(c, {0: TC.mis_armed(true), 1: TC.off_map(true)})
    (o, m, rows), launches = _launches(c, lambda: MR._call(c, 2, {l: MR._entries(W["dev"], TC.START, TC.START + n) for l in range(2)}))
    out = {"o": o, "m": m, "rec": c.recovery_rows(2 * n), "T0": _T(c, 0), "T1": _T(c, 1), "launches": launches}
    out.update({"row_" + k: rows[k] for k in ROW_KEYS})
    for l in range(2):
        try:
            out["dbg%d" % l] = c.debug_recovery_scores(l)
        except aloam.AloamError as e:
            assert e.code == MR.ERR_STATE
            out["dbg%d" % l] = None
    return out


def _launches(c, fn):
    a = c.launch_count()
    out = fn()
    return out, c.launch_count() - a


def _same(a, b, what):
    for k in a:
        if k == "rec":
            for j in a[k]:
                assert np.array_equal(a[k][j], b[k][j]), (what, j)
        elif a[k] is None or b[k] is None:
            assert a[k] is None and b[k] is None, (what, k)
        else:
            assert np.array_equal(a[k], b[k], equal_nan=True), (what, k)


def test_resetting_recovery_over_a_contexts_life(aloam, world):
    """one context set to n_delta 3, 20 808, 5 and 65 536 in turn (the slices grow, then keep the larger stride): after each call
    everything equals a fresh context with that setting, and the debug scores are aloam_prior_relocalise's.  Setting recovery again
    after a triggering call makes the scores unreadable until the next call; rows turned off and on leave recovery off until it is
    set again"""
    W = world
    c = MR._localiser(aloam, W, 2)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    for name, D in RE.settings(aloam):
        c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
        got = _life_call(aloam, c, W)
        fresh = MR._localiser(aloam, W, 2)
        fresh.set_map_rows(True, TC.ISQ, TC.PTS)
        fresh.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
        ref = _life_call(aloam, fresh, W)
        assert got["rec"]["triggered"][0] and got["rec"]["triggered"][1::2].all(), name
        _same(got, ref, name)
        k = int(np.flatnonzero(got["rec"]["triggered"][0::2])[-1])   # lane 0's latest triggered row
        assert np.array_equal(got["dbg0"], _ref_scores(fresh, got["m"][k, 0], D, W["feats"][TC.START + k])), name
        assert not got["dbg1"].any() and len(got["dbg1"]) == len(D), name
        fresh.close()
        c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
        for l in range(2):
            MR._expect(aloam, MR.ERR_STATE, lambda: c.debug_recovery_scores(l))
    c.set_map_rows(False)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    off = _life_call(aloam, c, W)
    assert not off["rec"]["triggered"].any() and off["dbg0"] is None and off["dbg1"] is None
    c.set_recovery(False)
    never = _life_call(aloam, c, W)
    assert off["launches"] == never["launches"]
    _same({k: v for k, v in off.items() if k != "launches"}, {k: v for k, v in never.items() if k != "launches"}, "rows off and on")
    D = RE.settings(aloam)[0][1]
    c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
    back = _life_call(aloam, c, W)
    assert back["rec"]["triggered"][0] and back["launches"] == never["launches"] + 4 * 3
    c.close()


def _relocalise_rc(aloam, c, hyps, ls, lf, isq, mp):
    """aloam_prior_relocalise through the C ABI -> (return code, coarse scores): the scores of a call that returns
    ALOAM_ERR_CAPACITY too"""
    a, ka = aloam._view(ls)
    b, kb = aloam._view(lf)
    h = np.ascontiguousarray(hyps, np.float64)
    sc = np.zeros(len(h), np.int32)
    out = (aloam.RelocResult * 1)()
    rc = aloam.lib().aloam_prior_relocalise(c._h, a, b, aloam._dp(h), len(h), C.byref(aloam.RelocOpts(float(isq), int(mp), 1)),
                                            sc.ctypes.data_as(C.POINTER(C.c_int)), out)
    return rc, sc


def test_an_overflow_row_triggers_and_stays_readable(aloam, synth, world):
    """a localising lane armed 45 degrees and 3 m off and STARTed on the scan whose less-sharp stack filter overflows its key, at
    trigger_frac 1 (the truly armed lane scores every point of that scan): the call returns ALOAM_ERR_CAPACITY, the recovery rows
    are readable and the overflow row triggered; its candidate scores equal aloam_prior_relocalise's on the same scan (which
    reports the overflow too) and, on a subset, the oracle's on the unfiltered less-sharp stack"""
    import torch
    W = world
    raw4, _ = TE.overflow_scan(synth)
    dev = torch.from_numpy(raw4).cuda()
    D = RV.deltas(aloam)
    c = MR._localiser(aloam, W, 1)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, 1.0, RV.ACCEPT, D)
    T = TC.mis_armed(W["map"][4])
    c.lane_localise(0, T[:4], T[4:])
    ptrs, counts, ops = MR._grid(1, {0: [(dev.data_ptr(), dev.shape[0], MR.START)]})
    odom, mp = np.zeros((1, 1, 7)), np.zeros((1, 1, 7))
    st = (aloam.Stats * 1)()
    opsc = np.ascontiguousarray(ops, np.int32)
    rc = aloam.lib().aloam_scan_stream_lanes(c._h, aloam._views(ptrs, counts, 4), opsc.ctypes.data_as(C.POINTER(C.c_int)), 1, 1, 1,
                                             aloam._dp(odom), aloam._dp(mp), st)
    assert rc == MR.ERR_CAPACITY, rc
    rows = c.map_rows(1)
    rec = c.recovery_rows(1)
    assert [int(e & 1) for e in rows["err"]] == [1] and rows["kind"][0] == aloam.ROW_LOCALISED
    assert rec["triggered"][0] and RV.triggers(rows["score"][0], rows["n_score"][0], 1.0), (rows["score"], rows["n_score"])
    sc = c.debug_recovery_scores(0)
    f = c.extract_features(raw4)
    rrc, ref = _relocalise_rc(aloam, c, RE.hypotheses(mp[0, 0], D), f["less_sharp"], f["less_flat"], TC.ISQ, TC.PTS)
    assert rrc == MR.ERR_CAPACITY, rrc
    assert np.array_equal(sc, ref), np.flatnonzero(sc != ref)[:8]
    h, _ = _check_best(c, rec, 0, rows["score"][0], rows["n_score"][0], mp[0, 0], odom[0, 0], D, ref, RV.ACCEPT, 0, "overflow")
    pts = (RC.subsample(f["less_sharp"], TC.PTS), RC.scoring_points(f["less_sharp"], f["less_flat"], TC.PTS, *W["res"])[1])
    idx = sorted(set(range(0, len(D), 37)) | {h})
    got = W["scorer"].score_points(pts, RV.candidates(mp[0, 0], D[idx]), TC.ISQ, normalise=False)
    assert np.array_equal(got, sc[idx]), (got, sc[idx])
    c.close()
