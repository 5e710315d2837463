"""GPU parity of the lane-scheduled stream (aloam_scan_stream_lanes): trajectories of different lengths start and end
independently in the lanes of one context.  Every trajectory must be bit-identical to its solo run on a fresh context --
odometry poses, map poses, stats and the final cube store -- whatever its lane, its start step and the other lanes'
schedules; idle rows are NaN; the lockstep calls are refused until aloam_reset_odometry."""
import numpy as np
import pytest

from conftest import rot_angle

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_EMPTY_CLOUD, ERR_STATE = -1, -3, -9
IDLE, SCAN, START = 0, 1, 2
STAT_KEYS = ("n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps", "flags", "termination", "init_cost", "final_cost")


def _trajs(synth, lengths, sensor="VLP-16", seed0=100):
    return [[synth.scan(sensor, k, seed=synth.BASE_SEED + seed0 + t, n_az=900) for k in range(n)] for t, n in enumerate(lengths)]


def _refill(lengths, lanes):
    """arrival order, each trajectory to the lane that frees first; it STARTs at the step after the lane's previous one ended"""
    free_at = [0] * lanes
    placed = []
    for t, n in enumerate(lengths):
        lane = min(range(lanes), key=lambda b: (free_at[b], b))
        placed.append((t, lane, free_at[lane]))
        free_at[lane] += n
    return placed, max(free_at)


def _plan(placed, lengths, steps, lanes):
    """ops (steps, lanes) and, per entry, the trajectory and its scan index (-1 where idle)"""
    ops = np.zeros((steps, lanes), np.int32)
    who = np.full((steps, lanes), -1)
    idx = np.full((steps, lanes), -1)
    for t, lane, s in placed:
        for i in range(lengths[t]):
            ops[s + i, lane] = START if i == 0 else SCAN
            who[s + i, lane] = t
            idx[s + i, lane] = i
    return ops, who, idx


def _addresses(trajs, dev, who, idx):
    """(steps, lanes) addresses and counts of the scheduled scans (0 where idle); dev: device tensors, or None for host buffers"""
    ptrs = np.zeros(who.shape, np.uint64)
    counts = np.zeros(who.shape, np.int64)
    for (k, b), t in np.ndenumerate(who):
        if t >= 0:
            s = trajs[t][idx[k, b]]
            ptrs[k, b] = dev[t][idx[k, b]].data_ptr() if dev is not None else s.ctypes.data
            counts[k, b] = s.shape[0]
    return ptrs, counts


def _rows(poses, who, t):
    """the rows of trajectory t in step order"""
    ks, bs = np.nonzero(who == t)
    return poses[ks, bs]


def _solo_addresses(traj, dev_t):
    return np.array([d.data_ptr() for d in dev_t], np.uint64), np.array([s.shape[0] for s in traj])


def _same_state(a, b):
    return (a["centre"] == b["centre"] and a["valid"] == b["valid"] and np.array_equal(a["q_wmap_wodom"], b["q_wmap_wodom"])
            and np.array_equal(a["t_wmap_wodom"], b["t_wmap_wodom"]) and (a["total_corner"], a["total_surf"]) == (b["total_corner"], b["total_surf"]))


def _same_store(ctx_a, lane_a, ctx_b, lane_b):
    """state and every cube of the last frame's valid block, both cloud types, bit for bit"""
    sa, sb = ctx_a.mapper_state(lane_a), ctx_b.mapper_state(lane_b)
    assert _same_state(sa, sb), (lane_a, lane_b)
    for c in sa["valid"]:
        for which in (0, 1):
            a, b = ctx_a.mapper_cube(which, c, lane_a), ctx_b.mapper_cube(which, c, lane_b)
            assert a.view(np.int32).tobytes() == b.view(np.int32).tobytes(), (lane_a, c, which)
    assert sa["total_corner"] + sa["total_surf"] > 0


def _same_stats(a, b):
    return all(a[k] == b[k] for k in STAT_KEYS)


def _oracle_map_poses(orc, synth, scans, sensor, line_res, plane_res):
    ns, _, mr = synth.SENSORS[sensor][:3]
    cm = orc.CubeMap()
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    out = []
    for k, raw in enumerate(scans):
        fo = orc.Features(raw, ns, mr)
        if k > 0:
            q, t, _ = od.register(fo.sharp, fo.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
        od.set_last(fo.less_sharp, fo.less_flat)
        pose, _ = cm.step(fo.less_sharp, fo.less_flat, qw, tw, line_res, plane_res)
        out.append(pose)
    return np.array(out)


def _maxn(trajs):
    return max(s.shape[0] for tr in trajs for s in tr)


def _ctx(aloam, maxn, batch, mapped=True):
    extra = {"max_map_points": 400000} if mapped else {}
    return aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_batch=batch, max_ring_points=4096, **extra)


def _to_device(trajs):
    import torch
    return [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]


def test_refill_schedule_mapped_equals_solo_runs_and_oracle(aloam, orc, synth):
    """4 lanes, 7 trajectories; a finished lane STARTs its next trajectory at the following step (lanes restart while the others
    run), the tail is idle.  Two calls, the boundary inside four trajectories: device-resident, then from host buffers."""
    lengths = [9, 4, 6, 3, 7, 5, 2]
    lanes = 4
    trajs = _trajs(synth, lengths)
    dev = _to_device(trajs)
    placed, steps = _refill(lengths, lanes)
    ops, who, idx = _plan(placed, lengths, steps, lanes)
    dptrs, counts = _addresses(trajs, dev, who, idx)
    hptrs, _ = _addresses(trajs, None, who, idx)
    split = 5
    assert sum(1 for t, b, s in placed if s < split <= s + lengths[t] - 1) >= 3   # trajectories that span both calls
    ctx = _ctx(aloam, _maxn(trajs), lanes)
    o1, m1 = ctx.scan_stream_lanes(dptrs[:split], counts[:split], ops[:split], True)
    o2, m2 = ctx.scan_stream_lanes(hptrs[split:], counts[split:], ops[split:], False)
    odom, mapped = np.concatenate([o1, o2]), np.concatenate([m1, m2])
    assert odom.shape == mapped.shape == (steps, lanes, 7)
    assert np.isnan(odom[ops == IDLE]).all() and np.isnan(mapped[ops == IDLE]).all()
    assert np.isfinite(odom[ops != IDLE]).all() and np.isfinite(mapped[ops != IDLE]).all()
    last_of_lane = {b: t for t, b, s in placed}   # placed in start order: the lane's last trajectory wins
    for t, lane, start in placed:
        solo = _ctx(aloam, _maxn(trajs), 1)
        sp, sc = _solo_addresses(trajs[t], dev[t])
        so, sm = solo.scan_stream_mapped(sp, sc, True)
        assert np.array_equal(_rows(odom, who, t), so), "odometry of trajectory %d (lane %d, start %d)" % (t, lane, start)
        assert np.array_equal(_rows(mapped, who, t), sm), "map poses of trajectory %d (lane %d, start %d)" % (t, lane, start)
        if last_of_lane[lane] == t:
            _same_store(ctx, lane, solo, 0)
        solo.close()
    ref = _oracle_map_poses(orc, synth, trajs[0], "VLP-16", ctx.cfg.line_res, ctx.cfg.plane_res)
    m0 = _rows(mapped, who, 0)
    assert np.abs(m0[:, 4:] - ref[:, 4:]).max() < 1e-4
    assert max(rot_angle(m0[k, :4], ref[k, :4]) for k in range(lengths[0])) < 1e-4
    ctx.close()


def test_refill_schedule_odometry_only_and_stats(aloam, synth):
    lengths = [9, 4, 6, 3, 7, 5, 2]
    lanes = 4
    trajs = _trajs(synth, lengths)
    dev = _to_device(trajs)
    placed, steps = _refill(lengths, lanes)
    ops, who, idx = _plan(placed, lengths, steps, lanes)
    dptrs, counts = _addresses(trajs, dev, who, idx)
    ctx = _ctx(aloam, _maxn(trajs), lanes, mapped=False)
    odom, none = ctx.scan_stream_lanes(dptrs, counts, ops, True, mapped=False)
    assert none is None and np.isnan(odom[ops == IDLE]).all()
    stats = ctx.last_batch_stats
    last_of_lane = {b: t for t, b, s in placed}
    for t, lane, start in placed:
        solo = _ctx(aloam, _maxn(trajs), 1, mapped=False)
        sp, sc = _solo_addresses(trajs[t], dev[t])
        so, st = solo.scan_stream(sp, sc, True)
        assert np.array_equal(_rows(odom, who, t), so), "odometry of trajectory %d" % t
        if last_of_lane[lane] == t:   # the lane's last non-idle step of the call is this trajectory's last scan
            assert _same_stats(stats[lane], st.as_dict()), (lane, stats[lane], st.as_dict())
        solo.close()
    # a lane whose last step was a START only initialised; a lane idle all call has zeroed stats
    p = np.array([[dptrs[0, 0], 0, 0, 0]], np.uint64)
    c = np.array([[counts[0, 0], 0, 0, 0]])
    o, _ = ctx.scan_stream_lanes(p, c, np.array([[START, IDLE, IDLE, IDLE]], np.int32), True, mapped=False)
    st = ctx.last_batch_stats
    assert st[0]["flags"] == aloam.FLAG_INITIALISED_ONLY and st[0]["lm_iters"] == 0
    assert np.array_equal(o[0, 0], [0, 0, 0, 1, 0, 0, 0]) and np.isnan(o[0, 1:]).all()
    assert all(st[b]["flags"] == 0 and st[b]["lm_iters"] == 0 and st[b]["ms_total"] == 0 for b in (1, 2, 3))
    ctx.close()


def test_length_one_trajectories_idle_gaps_and_all_idle_steps(aloam, synth):
    """trajectories of one scan, STARTs after idle gaps (stale per-scan slots), an all-idle step inside a call, and a call of
    idle steps only: it issues no launch"""
    lengths = [1, 1, 3, 5, 2]
    trajs = _trajs(synth, lengths, seed0=200)
    dev = _to_device(trajs)
    #            0        1     2     3      4      5     6     7     8      9
    lane0 = [(0, 0), None, None, (1, 0), (2, 0), (2, 1), (2, 2), None, None, None]
    lane1 = [(3, 0), (3, 1), (3, 2), (3, 3), (3, 4), None, None, None, (4, 0), (4, 1)]
    steps = len(lane0)
    ops = np.zeros((steps, 2), np.int32)
    who = np.full((steps, 2), -1)
    idx = np.full((steps, 2), -1)
    for b, sched in enumerate((lane0, lane1)):
        for k, e in enumerate(sched):
            if e is not None:
                who[k, b], idx[k, b] = e
                ops[k, b] = START if e[1] == 0 else SCAN
    assert (ops[7] == IDLE).all()
    ptrs, counts = _addresses(trajs, dev, who, idx)
    ctx = _ctx(aloam, _maxn(trajs), 2)
    odom, mapped = ctx.scan_stream_lanes(ptrs, counts, ops, True)
    assert np.isnan(odom[ops == IDLE]).all() and np.isnan(mapped[ops == IDLE]).all()
    for t in range(len(lengths)):
        solo = _ctx(aloam, _maxn(trajs), 1)
        sp, sc = _solo_addresses(trajs[t], dev[t])
        so, sm = solo.scan_stream_mapped(sp, sc, True)
        assert np.array_equal(_rows(odom, who, t), so) and np.array_equal(_rows(mapped, who, t), sm), t
        if t in (2, 4):   # the last trajectory of lane 0 / lane 1
            _same_store(ctx, 0 if t == 2 else 1, solo, 0)
        solo.close()
    l0 = ctx.launch_count()
    o, m = ctx.scan_stream_lanes(np.zeros((3, 2), np.uint64), np.zeros((3, 2)), np.zeros((3, 2), np.int32), True)
    assert ctx.launch_count() == l0 and np.isnan(o).all() and np.isnan(m).all()
    ctx.close()


@pytest.mark.parametrize("B", [1, 2, 4])
def test_all_scan_schedule_is_the_lockstep_call(aloam, synth, B):
    """every lane STARTs at step 0 and SCANs after: the poses, the stores and the launch count of aloam_scan_stream_mapped_batch
    (B = 1: of aloam_scan_stream_mapped); a START in the middle of a call adds no launch"""
    n = 3
    trajs = _trajs(synth, [2 * n] * B, seed0=300)
    dev = _to_device(trajs)
    ptrs = np.array([[dev[b][k].data_ptr() for b in range(B)] for k in range(2 * n)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(B)] for k in range(2 * n)])
    ops = np.full((2 * n, B), SCAN, np.int32)
    ops[0] = START
    lanes_ctx, lock_ctx = _ctx(aloam, _maxn(trajs), B), _ctx(aloam, _maxn(trajs), B)
    counts_l, counts_b = [], []
    res_l, res_b = [], []
    for s in (slice(0, n), slice(n, 2 * n)):
        c0 = lanes_ctx.launch_count()
        res_l.append(lanes_ctx.scan_stream_lanes(ptrs[s], counts[s], ops[s], True))
        counts_l.append(lanes_ctx.launch_count() - c0)
        c0 = lock_ctx.launch_count()
        res_b.append(lock_ctx.scan_stream_mapped_batch(ptrs[s], counts[s], True))
        counts_b.append(lock_ctx.launch_count() - c0)
    assert counts_l == counts_b, (counts_l, counts_b)
    ol, ml = (np.concatenate([r[i] for r in res_l]) for i in (0, 1))
    ob, mb = (np.concatenate([r[i] for r in res_b]) for i in (0, 1))
    assert np.array_equal(ol, ob) and np.array_equal(ml, mb)
    for b in range(B):
        _same_store(lanes_ctx, b, lock_ctx, b)
    if B == 1:
        solo = _ctx(aloam, _maxn(trajs), 1)
        so, sm = solo.scan_stream_mapped(ptrs[:, 0], counts[:, 0], True)
        assert np.array_equal(so, ol[:, 0]) and np.array_equal(sm, ml[:, 0])
        solo.close()
    # lane 0 restarts in the middle of the next call: the same launches as the lockstep call on as many scans (with one lane,
    # the START step has no lane to register and issues fewer)
    ops2 = np.full((n, B), SCAN, np.int32)
    ops2[1, 0] = START
    c0 = lanes_ctx.launch_count()
    lanes_ctx.scan_stream_lanes(ptrs[:n], counts[:n], ops2, True)
    l_restart = lanes_ctx.launch_count() - c0
    c0 = lock_ctx.launch_count()
    lock_ctx.scan_stream_mapped_batch(ptrs[:n], counts[:n], True)
    l_lock = lock_ctx.launch_count() - c0
    assert l_restart == l_lock if B > 1 else 0 < l_restart < l_lock, (l_restart, l_lock)
    lanes_ctx.close(); lock_ctx.close()


def test_errors_and_mixing_with_lockstep_calls(aloam, synth):
    import torch
    raws = _trajs(synth, [4, 4], seed0=400)
    dev = _to_device(raws)
    maxn = _maxn(raws)
    P = np.array([[dev[b][k].data_ptr() for b in range(2)] for k in range(4)], np.uint64)
    N = np.array([[raws[b][k].shape[0] for b in range(2)] for k in range(4)])
    ops0 = np.array([[START, START], [SCAN, SCAN]], np.int32)
    ops1 = np.array([[SCAN, SCAN], [SCAN, SCAN]], np.int32)

    def expect(code, fn):
        with pytest.raises(aloam.AloamError) as e:
            fn()
        assert e.value.code == code

    ctx = _ctx(aloam, maxn, 2)
    fresh = _ctx(aloam, maxn, 2)
    # rejected before any state changes, on a fresh context ...
    expect(ERR_STATE, lambda: ctx.scan_stream_lanes(P[:1], N[:1], [[SCAN, START]], True))
    expect(ERR_INVALID_ARG, lambda: ctx.scan_stream_lanes(P[:1], N[:1], [[START, 3]], True))
    expect(ERR_INVALID_ARG, lambda: ctx.scan_stream_lanes(np.tile(P[:1, :1], (1, 3)), np.tile(N[:1, :1], (1, 3)), [[START] * 3], True))
    no_map = _ctx(aloam, maxn, 2, mapped=False)
    expect(ERR_INVALID_ARG, lambda: no_map.scan_stream_lanes(P[:2], N[:2], ops0, True))
    # ... so the lockstep calls still work there
    ctx.scan_stream_batch(P[:1], N[:1], True)
    ctx.reset_odometry()
    a = ctx.scan_stream_lanes(P[:2], N[:2], ops0, True)
    b = fresh.scan_stream_lanes(P[:2], N[:2], ops0, True)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    # ... and in the middle of running trajectories: the lanes go on as if the calls had not been made
    expect(ERR_INVALID_ARG, lambda: ctx.scan_stream_lanes(P[2:], N[2:], [[SCAN, SCAN], [SCAN, 3]], True))
    expect(ERR_STATE, lambda: ctx.scan_stream_lanes(P[2:], N[2:], [[SCAN, IDLE], [SCAN, SCAN]], True))
    expect(ERR_STATE, lambda: ctx.scan_stream_lanes(P[2:], N[2:], ops1, True, mapped=False))   # started mapped
    a = ctx.scan_stream_lanes(P[2:], N[2:], ops1, True)
    b = fresh.scan_stream_lanes(P[2:], N[2:], ops1, True)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    # the lockstep calls are refused after a lanes call, until aloam_reset_odometry
    expect(ERR_STATE, lambda: ctx.scan_stream_mapped_batch(P[:1], N[:1], True))
    expect(ERR_STATE, lambda: ctx.scan_stream_batch(P[:1], N[:1], True))
    expect(ERR_STATE, lambda: ctx.scan_stream_mapped(P[:1, 0], N[:1, 0], True))
    expect(ERR_STATE, lambda: ctx.scan_stream(P[:1, 0], N[:1, 0], True))
    expect(ERR_STATE, lambda: ctx.scan_to_pose(raws[0][0]))
    expect(ERR_STATE, lambda: ctx.scan_to_pose_device(int(P[0, 0]), int(N[0, 0])))
    # an empty cloud in one lane fails the run and leaves no lane running
    far = raws[1][0].copy(); far[:, :3] *= 1e-3   # everything closer than minimum_range: nothing survives (scanRegistration.cpp:137)
    dfar = torch.from_numpy(far).cuda()
    expect(ERR_EMPTY_CLOUD, lambda: ctx.scan_stream_lanes(np.array([[P[0, 0], dfar.data_ptr()]], np.uint64), N[:1], [[START, START]], True))
    expect(ERR_STATE, lambda: ctx.scan_stream_lanes(P[:1], N[:1], [[SCAN, IDLE]], True))
    expect(ERR_STATE, lambda: ctx.scan_stream_lanes(P[:1], N[:1], [[IDLE, SCAN]], True))
    o, m = ctx.scan_stream_lanes(P[:2], N[:2], ops0, True)   # a START works again
    assert np.isfinite(o).all() and np.isfinite(m).all()
    ctx.reset_odometry()
    o = ctx.scan_stream_batch(P[:2], N[:2], True)
    ob = no_map.scan_stream_batch(P[:2], N[:2], True)
    assert np.array_equal(o, ob)
    ctx.close(); fresh.close(); no_map.close()
