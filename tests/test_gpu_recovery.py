"""GPU: recovery of localising lanes inside the mapped stream calls (aloam_set_recovery, aloam_recovery_rows,
aloam_debug_recovery_scores), on the world of tests/test_gpu_map_rows.py with the scenario of tests/recovery_cases.py.  Checked
here: with recovery off, set then off, or on but never triggering, every pose, row, registered cloud and launch count is what it
is without the feature (plus four launches per localising frame while on); the mis-armed lane triggers and adopts on the rows the
host model predicts from the device's own rows, its candidate scores equal aloam_prior_relocalise's coarse scores of the host-composed
hypotheses, the adopted T_wmap_wodom equals the host transformUpdate bit for bit, later rows follow the frozen oracle re-seated
there, and its odometry is that of the run without recovery; the off-map lane triggers on every row and never adopts; 16 lanes
equal their solo runs; at mapping_skip_frame 3 the skipped rows compose with the adopted T; refusals."""
import ctypes as C

import numpy as np
import pytest

import lane_refs as R
import recovery_cases as RV
import reloc_cases as RC
import track_cases as TC
from test_gpu_map_rows import _call, _ctx, _entries, _expect, _localiser, _world

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE = -1, -9
ROW_KEYS = ("kind", "err", "n_valid", "score", "n_score", "flags", "lm_iters", "init_cost", "final_cost")


def _set(c, D, trigger=RV.TRIGGER, accept=RV.ACCEPT):
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, trigger, accept, D)


def _arm(c, inits):
    for lane, init in inits.items():
        c.lane_localise(lane, init[:4], init[4:])


def _same_rows(a, b, what):
    for k in ROW_KEYS:
        assert np.array_equal(a[k], b[k]), (what, k)


def _launches(fn, c):
    a = c.launch_count()
    out = fn()
    return out, c.launch_count() - a


def test_recovery_off_or_never_triggering_changes_nothing(aloam, synth):
    """lanes armed true, mis-armed and off the map beside a mapping lane, and an odometry-only lane in calls of its own: recovery
    never set, set then off, and on with trigger_frac 0 give identical poses, rows, registered clouds and launches (+4 per
    localising frame while on, and no row triggers)"""
    import torch
    W = _world(aloam, synth)
    D = RV.deltas(aloam)
    true = W["map"][TC.START]
    out = []
    for mode in ("never", "off", "zero"):
        c = _localiser(aloam, W, 4)
        sink = torch.zeros((20 * W["M"], 4), dtype=torch.float32, device="cuda")
        c.set_registered_sink(sink)
        c.set_map_rows(True, TC.ISQ, TC.PTS)
        if mode == "off":
            c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
            c.set_recovery(False)
        elif mode == "zero":
            c.set_recovery(True, 0.0, RV.ACCEPT, D)
        res = []
        o, n0 = _launches(lambda: _call(c, 4, {3: _entries(W["dev"], 0, 3)}, mapped=False, rows=False), c)
        res.append(("odo", o[0], n0))
        _arm(c, {0: true, 1: TC.mis_armed(true), 2: TC.off_map(true)})
        lanes = {l: _entries(W["dev"], TC.START, TC.START + 5) for l in range(3)}
        lanes[3] = _entries(W["dev"], 0, 5)
        (o, m, rows), n1 = _launches(lambda: _call(c, 4, lanes), c)
        begin, count = c.registered_rows(o.shape[0] * 4)
        clouds = [sink[b:b + k].cpu().numpy().copy() for b, k in zip(begin, count)]
        rec = c.recovery_rows(o.shape[0] * 4)
        assert not rec["triggered"].any() and (rec["best"] == -1).all() and not rec["pose"].any(), mode
        _expect(aloam, ERR_STATE, lambda: c.debug_recovery_scores(1))
        res.append(("map", o, m, rows, clouds, n1))
        o, n2 = _launches(lambda: _call(c, 4, {3: _entries(W["dev"], 3, 6)}, mapped=False, rows=False), c)
        res.append(("odo", o[0], n2))
        out.append((mode, res, c.mapper_state(1)))
        c.close()
    base = out[0]
    for mode, res, st in out[1:]:
        assert np.array_equal(st["q_wmap_wodom"], base[2]["q_wmap_wodom"]) and np.array_equal(st["t_wmap_wodom"], base[2]["t_wmap_wodom"]), mode
        for a, b in zip(res, base[1]):
            if a[0] == "odo":
                assert np.array_equal(a[1], b[1], equal_nan=True) and a[2] == b[2], mode
                continue
            _, o, m, rows, clouds, n = a
            assert np.array_equal(o, b[1], equal_nan=True) and np.array_equal(m, b[2], equal_nan=True), mode
            _same_rows(rows, b[3], mode)
            assert len(clouds) == len(b[4]) and all(np.array_equal(x, y) for x, y in zip(clouds, b[4])), mode
            loc_frames = int((rows["kind"].reshape(-1, 4) == aloam.ROW_LOCALISED).any(axis=1).sum())
            assert n == b[5] + (4 * loc_frames if mode == "zero" else 0), (mode, n, b[5], loc_frames)


def _stepwise(aloam, W, D, recover, n=6):
    """lanes 0 (true), 1 (mis-armed), 2 (off the map) STARTed at TC.START, one stream call per step: per step (odometry, map
    poses, rows, recovery rows or None, lane 1's T_wmap_wodom, lane 1's candidate scores or None)"""
    c = _localiser(aloam, W, 3)
    if recover:
        _set(c, D)
    else:
        c.set_map_rows(True, TC.ISQ, TC.PTS)
    true = W["map"][TC.START]
    _arm(c, {0: true, 1: TC.mis_armed(true), 2: TC.off_map(true)})
    entries = _entries(W["dev"], TC.START, TC.START + n)
    steps = []
    for j in range(n):
        o, m, rows = _call(c, 3, {l: [entries[j]] for l in range(3)})
        rec = c.recovery_rows(3) if recover else None
        st = c.mapper_state(1)
        sc = c.debug_recovery_scores(1) if recover and rec["triggered"][1] else None
        steps.append((o[0], m[0], rows, rec, np.concatenate([st["q_wmap_wodom"], st["t_wmap_wodom"]]), sc))
    return c, steps


def test_the_mis_armed_lane_is_recovered_as_the_host_model_predicts(aloam, synth):
    import pyfrozen
    W = _world(aloam, synth)
    D = RV.deltas(aloam)
    base_c, base = _stepwise(aloam, W, D, False)
    base_c.close()
    c, steps = _stepwise(aloam, W, D, True)
    adopted_at = None
    oracle = None
    for j, (o, m, rows, rec, T, sc) in enumerate(steps):
        bo, bm, brows = base[j][:3]
        f = W["feats"][TC.START + j]
        # no lane's odometry restarts; the lanes that never adopt are the run without recovery
        assert np.array_equal(o, bo), j
        for lane in (0, 2):
            assert np.array_equal(m[lane], bm[lane]), (j, lane)
            for k in ROW_KEYS:
                assert rows[k][lane] == brows[k][lane], (j, lane, k)
        for lane in range(3):
            trig = RV.triggers(rows["score"][lane], rows["n_score"][lane])
            assert bool(rec["triggered"][lane]) == trig, (j, lane, rows["score"][lane], rows["n_score"][lane])
        assert not rec["triggered"][0]
        assert rec["triggered"][2] and not rec["adopted"][2] and rec["best_score"][2] == 0, (j, rec)
        if rec["triggered"][1]:
            # the device's candidate scores are aloam_prior_relocalise's coarse scores of the host-composed hypotheses
            hyps = RV.products(m[1], RC.normalised(D))
            _, ref = c.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], inlier_sq=TC.ISQ, max_score_points=TC.PTS, refine=1, scores=True)
            assert np.array_equal(sc, ref), j
            h, bs = RV.best_of(ref)
            assert (rec["best"][1], rec["best_score"][1]) == (h, bs), (j, rec["best"][1], rec["best_score"][1], h, bs)
            cand = RV.candidates(m[1], D)
            assert np.array_equal(rec["pose"][1], cand[h]), j
            assert bool(rec["adopted"][1]) == RV.accepts(bs, rows["score"][1], rows["n_score"][1]), j
            if rec["adopted"][1]:
                assert np.array_equal(T, RV.transform_update(cand[h], o[1])), (j, T)
                adopted_at = j if adopted_at is None else adopted_at
                oracle = pyfrozen.Localiser(W["frozen"], T[:4], T[4:], normalise=False)
                continue
        if oracle is not None:   # later rows: the frozen oracle re-seated at the adopted T, on the device's features and odometry
            pose, _ = oracle.step(f["less_sharp"], f["less_flat"], o[1, :4], o[1, 4:], *W["res"])
            dt, dr = R.deviation(m[1][None], pose[None])
            assert dt < 1e-6 and dr < 1e-6, (j, dt, dr)
            oracle.q, oracle.t = T[:4].copy(), T[4:].copy()
    assert adopted_at == 0, adopted_at
    k = RV.FRAMES_TO_TRACK
    m1 = np.array([s[1][1] for s in steps[k:]])
    m0 = np.array([s[1][0] for s in steps[k:]])
    dt, dr = R.deviation(m1, m0)
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    for s in steps[k:]:
        assert s[2]["score"][1] > TC.TRACK_RATIO * s[2]["n_score"][1]
    c.close()


def _lanes16(W):
    true = W["map"][TC.START]
    inits = {}
    for l in range(12):
        yaw, off = np.radians(10.0 + 5.0 * l), (0.5 * (l % 4) - 1.0, 3.0 - 0.5 * (l // 4), 0.0)
        dq = np.array([0, 0, np.sin(yaw / 2), np.cos(yaw / 2)])
        p = np.array(true, np.float64, copy=True)
        p[:4] = TC.qmul(dq, p[:4])
        p[4:] = p[4:] + np.asarray(off)
        inits[l] = p
    inits[12] = true
    inits[13] = W["map"][TC.START + 1]
    inits[14] = TC.off_map(true)
    return inits   # lane 15 maps


def test_sixteen_lanes_equal_their_solo_runs(aloam, synth):
    W = _world(aloam, synth)
    D = RV.deltas(aloam)
    inits = _lanes16(W)
    n = 5
    starts = {l: TC.START + (1 if l == 13 else 0) for l in range(16)}
    starts[15] = 0

    def run(lanes, batch):
        c = _localiser(aloam, W, batch)
        _set(c, D)
        _arm(c, {b: inits[l] for b, l in enumerate(lanes) if l in inits})
        o, m, rows = _call(c, batch, {b: _entries(W["dev"], starts[l], starts[l] + n) for b, l in enumerate(lanes)})
        rec = c.recovery_rows(n * batch)
        c.close()
        return o, m, rows, rec

    o, m, rows, rec = run(list(range(16)), 16)
    assert rec["adopted"].reshape(n, 16)[:, :12].any() and rec["triggered"].reshape(n, 16)[:, 14].all()
    assert (rows["kind"].reshape(n, 16)[:, 15] == aloam.ROW_MAPPED).all()
    for l in range(16):
        so, sm, srows, srec = run([l], 1)
        assert np.array_equal(o[:, l], so[:, 0]) and np.array_equal(m[:, l], sm[:, 0]), l
        for k in ROW_KEYS:
            assert np.array_equal(rows[k].reshape(n, 16)[:, l], srows[k]), (l, k)
        for k in srec:
            a = rec[k].reshape((n, 16) + rec[k].shape[1:])[:, l]
            assert np.array_equal(a, srec[k]), (l, k)


def test_skipped_rows_compose_with_the_adopted_t(aloam, synth):
    """mapping_skip_frame 3: the mis-armed lane adopts on its START row, a registered row; the two skipped rows after it are the
    adopted T composed with their odometry poses, bit for bit"""
    W = _world(aloam, synth)
    D = RV.deltas(aloam)
    c = _ctx(aloam, W["M"], 1, W["ns"], mapping_skip_frame=3)
    store = aloam.snapshot_store_clouds(W["blob"])
    c.prior_map_build(store["corner"], store["surf"], store["centre"])
    _set(c, D)
    true = W["map"][TC.START]
    _arm(c, {0: TC.mis_armed(true)})
    o, m, rows = _call(c, 1, {0: _entries(W["dev"], TC.START, TC.START + 4)})
    rec = c.recovery_rows(4)
    assert list(rows["kind"]) == [aloam.ROW_LOCALISED, aloam.ROW_SKIPPED, aloam.ROW_SKIPPED, aloam.ROW_LOCALISED]
    assert rec["adopted"][0] and not rec["triggered"][1:3].any()
    T = RV.transform_update(rec["pose"][0], o[0, 0])
    for j in (1, 2):
        odom = o[j, 0]
        x = np.concatenate([RV.qmul(T[:4], odom[:4]), [RV.qrot(T[:4], odom[4:])[k] + T[4 + k] for k in range(3)]])
        assert np.array_equal(m[j, 0], x), (j, m[j, 0], x)
    dt, dr = R.deviation(m[3:, 0], W["map"][TC.START + 3][None])   # the registered row after the adoption is back on the map
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    c.close()


def test_refusals_leave_the_context_as_it_was(aloam, synth):
    W = _world(aloam, synth)
    D = RV.deltas(aloam)
    lib = aloam.lib()
    c = _localiser(aloam, W, 2)
    opts = aloam.RecoveryOpts(RV.TRIGGER, RV.ACCEPT)
    d = np.ascontiguousarray(D)

    def setr(on=1, o=opts, dd=d, n=None):
        return lib.aloam_set_recovery(c._h, on, C.byref(o) if o is not None else None, aloam._dp(dd) if dd is not None else None,
                                      len(dd) if n is None and dd is not None else (n or 0))

    assert setr() == ERR_STATE                                   # no rows
    c.set_map_rows(True)
    assert setr() == ERR_STATE                                   # rows without scoring
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    bad_q = d[:3].copy(); bad_q[1, :4] = 0
    bad_v = d[:3].copy(); bad_v[2, 5] = np.nan
    for args in ({"on": 2}, {"on": -1}, {"o": None}, {"dd": None, "n": 3}, {"n": 0}, {"dd": np.zeros((65537, 7)) + [0, 0, 0, 1, 0, 0, 0]},
                 {"dd": bad_q}, {"dd": bad_v}, {"o": aloam.RecoveryOpts(float("nan"), 0.5)}, {"o": aloam.RecoveryOpts(0.5, -0.1)},
                 {"o": aloam.RecoveryOpts(1.1, 0.5)}, {"o": aloam.RecoveryOpts(0.5, float("inf"))}):
        assert setr(**args) == ERR_INVALID_ARG, args
    # nothing was turned on by the refusals: a call issues no recovery launches
    true = W["map"][TC.START]
    _arm(c, {0: TC.mis_armed(true)})
    (_, _, rows), n_off = _launches(lambda: _call(c, 2, {0: _entries(W["dev"], TC.START, TC.START + 2)}), c)
    assert not c.recovery_rows(4)["triggered"].any()
    row = (aloam.RecoveryRow * 4)()
    assert lib.aloam_recovery_rows(c._h, None, 4) == ERR_INVALID_ARG and lib.aloam_recovery_rows(c._h, row, 3) == ERR_INVALID_ARG
    # a valid setting, then refusals: the next call equals a fresh context's with the same setting
    assert setr() == 0
    for args in ({"on": 2}, {"n": 0}, {"dd": bad_q}, {"o": aloam.RecoveryOpts(0.5, 2.0)}):
        assert setr(**args) == ERR_INVALID_ARG, args
    scores = np.zeros(len(D), np.int32)
    ip = C.POINTER(C.c_int)
    assert lib.aloam_debug_recovery_scores(c._h, 0, scores.ctypes.data_as(ip), len(D)) == ERR_STATE   # before any triggered row
    _arm(c, {0: TC.mis_armed(true)})
    got = _call(c, 2, {0: _entries(W["dev"], TC.START, TC.START + 2)})
    grec = c.recovery_rows(4)
    assert grec["adopted"][0]
    assert lib.aloam_debug_recovery_scores(c._h, 0, scores.ctypes.data_as(ip), len(D) - 1) == ERR_INVALID_ARG
    assert lib.aloam_debug_recovery_scores(c._h, 2, scores.ctypes.data_as(ip), len(D)) == ERR_INVALID_ARG
    assert lib.aloam_debug_recovery_scores(c._h, 1, scores.ctypes.data_as(ip), len(D)) == ERR_STATE
    assert lib.aloam_debug_recovery_scores(c._h, 0, scores.ctypes.data_as(ip), len(D)) == 0
    f = _localiser(aloam, W, 2)
    _set(f, D)
    _arm(f, {0: TC.mis_armed(true)})
    ref = _call(f, 2, {0: _entries(W["dev"], TC.START, TC.START + 2)})
    frec = f.recovery_rows(4)
    f.close()
    assert np.array_equal(got[1], ref[1], equal_nan=True) and all(np.array_equal(grec[k], frec[k]) for k in grec)
    # turning scoring off turns recovery off: launches as without it
    c.set_map_rows(True, TC.ISQ, 0)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    _arm(c, {0: TC.mis_armed(true)})
    (_, _, rows2), n2 = _launches(lambda: _call(c, 2, {0: _entries(W["dev"], TC.START, TC.START + 2)}), c)
    assert not c.recovery_rows(4)["triggered"].any()
    c.set_recovery(False)
    _arm(c, {0: TC.mis_armed(true)})
    (_, _, rows3), n3 = _launches(lambda: _call(c, 2, {0: _entries(W["dev"], TC.START, TC.START + 2)}), c)
    assert n2 == n3 and n_off > 0
    for k in ("score", "n_score", "flags"):
        assert np.array_equal(rows2[k], rows3[k]), k
    # sharded ranks and emulating contexts refuse, and emulation turns recovery off
    assert setr() == 0
    assert lib.aloam_debug_shard_emulate(c._h, 0, 2, 0, 0) == 0
    assert setr() == ERR_STATE and setr(on=0) == ERR_STATE
    assert lib.aloam_debug_shard_emulate(c._h, 0, 0, 0, 0) == 0
    c.reset_odometry()
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    _arm(c, {0: TC.mis_armed(true)})
    _call(c, 2, {0: _entries(W["dev"], TC.START, TC.START + 1)})
    assert not c.recovery_rows(2)["triggered"].any()
    c.close()


def test_adoption_needs_a_better_score(aloam, synth):
    """trigger_frac 1, accept_frac 0 and the identity among the deltas: a tracking lane's rows that miss a point trigger, and their
    best candidate -- at best the row's own pose, normalised -- is adopted only where it scores above the row; the off-map lane's
    zero-score rows trigger and never adopt"""
    W = _world(aloam, synth)
    D = np.array([[0, 0, 0, 1.0, 0, 0, 0], [0, 0, 0, 1.0, 0.05, 0, 0], [0, 0, np.sin(0.005), np.cos(0.005), 0, 0, 0]])
    c = _localiser(aloam, W, 2)
    _set(c, D, 1.0, 0.0)
    true = W["map"][TC.START]
    _arm(c, {0: true, 1: TC.off_map(true)})
    n = 8
    o, m, rows = _call(c, 2, {l: _entries(W["dev"], TC.START, TC.START + n) for l in range(2)})
    rec = c.recovery_rows(2 * n)
    trig = [RV.triggers(s, k, 1.0) for s, k in zip(rows["score"], rows["n_score"])]
    assert list(rec["triggered"].astype(bool)) == trig and any(trig[0::2])
    for r in range(2 * n):
        if trig[r]:
            assert bool(rec["adopted"][r]) == (rec["best_score"][r] > rows["score"][r]), (r, rec["best_score"][r], rows["score"][r])
    assert rec["triggered"][1::2].all() and not rec["adopted"][1::2].any()
    assert (rec["best_score"][0::2][np.array(trig[0::2])] >= rows["score"][0::2][np.array(trig[0::2])]).all()
    c.close()
