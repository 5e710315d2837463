"""Every lane of wide, odd-width, mixed-size and de-skewed batches.  Each kernel takes its work from a by-value Batch of up to
16 records picked by blockIdx.y / .z, and the grid-stride launches split 8 * SMs (2 * SMs, the cooperative sort's grid)
CTAs by integer division over the lanes.  So every lane of a run is compared with two references: the same trajectory
alone on a fresh context (bit for bit: poses, stats, mapper state and every cube of the valid block) and the CPU oracle
chain (1e-4 m / 1e-4 rad), which catches an error on the code path a solo run shares with the batch."""
import ctypes as C

import numpy as np
import pytest

import edge_scenes as es
import lane_refs as R

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_RING_TOO_LARGE, ERR_STATE = -1, -7, -9
IDLE, SCAN, START = 0, 1, 2


def _grid(trajs, dev=None):
    """(n_scans, lanes) addresses (device tensors, or the host arrays when dev is None) and point counts"""
    n, B = len(trajs[0]), len(trajs)
    ptrs = np.array([[dev[b][k].data_ptr() if dev is not None else trajs[b][k].ctypes.data for b in range(B)] for k in range(n)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(B)] for k in range(n)])
    return ptrs, counts


def _mapped_ctx(aloam, trajs, batch, distortion=0, max_ring=4096):
    return aloam.Aloam(n_scans=16, max_points=R.maxn(trajs) + 1024, max_map_points=400000, max_batch=batch,
                       max_ring_points=max_ring, distortion=distortion)


def _mapped_batch_two_calls(ctx, trajs, dev, split):
    """device-resident scans up to `split`, host buffers after it"""
    dptrs, counts = _grid(trajs, dev)
    hptrs, _ = _grid(trajs)
    o1, m1 = ctx.scan_stream_mapped_batch(dptrs[:split], counts[:split], True)
    o2, m2 = ctx.scan_stream_mapped_batch(hptrs[split:], counts[split:], False)
    return np.concatenate([o1, o2]), np.concatenate([m1, m2])


def _check_mapped_lane(aloam, orc, synth, what, scans, key, odom, mapped, store, sizes=None, distortion=0, with_oracle=True):
    """one trajectory's rows of a mapped run against its solo aloam_scan_stream_mapped run (in calls of `sizes`) and the
    oracle chain; `what` names the lane in the messages"""
    what = "%s (trajectory %s)" % (what, key)
    s = R.solo(aloam, scans, key, True, distortion, sizes)
    assert np.array_equal(odom, s["odom"]), "odometry of %s differs from its solo run" % what
    assert np.array_equal(mapped, s["map"]), "map poses of %s differ from its solo run" % what
    if store is not None:
        R.same_store(store, s["store"], "store of " + what)
    if with_oracle:
        o, m = R.oracle(orc, synth, scans, key, True, distortion)
        R.assert_near(odom, o, "odometry of " + what)
        R.assert_near(mapped, m, "map poses of " + what)


def test_full_width_odometry_batch_at_bench_shape(aloam, orc, synth):
    """HDL-32 32 x 2200, 2304-point rings, 16 lanes, 5 scans in two calls (bench configs[4])"""
    B, n, sizes = 16, 5, (3, 2)
    keys = [("HDL-32", t, None) for t in range(B)]
    trajs = [R.traj(synth, t, n, "HDL-32", None) for t in range(B)]
    dev = [R.to_device(tr) for tr in trajs]
    ptrs, counts = _grid(trajs, dev)
    ctx = aloam.Aloam(n_scans=32, max_points=R.maxn(trajs) + 1024, max_batch=B, max_ring_points=2304)
    poses = np.concatenate([ctx.scan_stream_batch(ptrs[s], counts[s], True) for s in R.splits_of(n, sizes)])
    stats = ctx.last_batch_stats
    ctx.close()
    assert poses.shape == (n, B, 7)
    for b in range(B):
        s = R.solo(aloam, trajs[b], keys[b], False, sizes=sizes, ns=32, max_ring=2304)
        assert np.array_equal(poses[:, b], s["odom"]), "lane %d differs from its solo run" % b
        assert R.same_stats(stats[b], s["stats"]), (b, stats[b], s["stats"])
        o, _ = R.oracle(orc, synth, trajs[b], keys[b], False, sensor="HDL-32")
        R.assert_near(poses[:, b], o, "lane %d" % b)
    assert all(st["lm_iters"] > 0 for st in stats)


def test_full_width_mapped_batch(aloam, orc, synth):
    """VLP-16 (900 azimuths), 16 lanes, 6 scans: 4 device-resident, then 2 from host buffers"""
    B, n = 16, 6
    keys = [("VLP-16", t, 900) for t in range(B)]
    trajs = [R.traj(synth, t, n) for t in range(B)]
    dev = [R.to_device(tr) for tr in trajs]
    ctx = _mapped_ctx(aloam, trajs, B)
    odom, mapped = _mapped_batch_two_calls(ctx, trajs, dev, 4)
    stores = [R.snapshot(ctx, b) for b in range(B)]
    ctx.close()
    for b in range(B):
        _check_mapped_lane(aloam, orc, synth, "lane %d" % b, trajs[b], keys[b], odom[:, b], mapped[:, b], stores[b], (4, 2))


def test_odd_widths_on_one_context(aloam, synth):
    """5, 7 and 13 lanes of one max_batch = 16 context (every per-lane CTA count is non-integral), reset in between; lane b
    runs trajectory width - 1 - b"""
    n = 6
    trajs = [R.traj(synth, t, n) for t in range(16)]
    dev = [R.to_device(tr) for tr in trajs]
    ctx = _mapped_ctx(aloam, trajs, 16)
    results = {}
    for B in (5, 7, 13):
        order = [B - 1 - b for b in range(B)]
        ctx.reset_odometry()
        ctx.mapper_reset()
        odom, mapped = _mapped_batch_two_calls(ctx, [trajs[t] for t in order], [dev[t] for t in order], 4)
        assert odom.shape == (n, B, 7)
        results[B] = (order, odom, mapped, [R.snapshot(ctx, b) for b in range(B)])
    ctx.close()
    for B, (order, odom, mapped, stores) in results.items():
        for b, t in enumerate(order):
            _check_mapped_lane(aloam, None, synth, "lane %d of %d" % (b, B), trajs[t], ("VLP-16", t, 900), odom[:, b], mapped[:, b],
                               stores[b], (4, 2), with_oracle=False)


def _ring_sizes(raw):
    """returns per VLP-16 ring (scanRegistration.cpp:150-158), from the points' elevation"""
    ang = np.degrees(np.arctan(raw[:, 2] / np.sqrt(raw[:, 0] ** 2 + raw[:, 1] ** 2)))
    return np.bincount((((ang + 15) / 2) + 0.5).astype(int), minlength=16)


def _mostly_too_close(raw):
    """all but every 8th return shrunk 1000-fold, inside minimum_range (0.3 m): a tiny scan that is not empty"""
    out = raw.copy()
    out[np.arange(len(out)) % 8 != 0, :3] *= 1e-3
    return out


MIXED_AZ = [int(a) for a in np.linspace(300, 4094, 16)]
TINY_LANE = 6


def test_mixed_sizes_in_one_step_and_a_ring_over_capacity(aloam, synth):
    """16 lanes of one sensor from 300 to 4094 azimuths (rings up to 4094 of 4096 points) and one lane whose returns are
    mostly inside minimum_range, mapped; then a 4097-point ring in lane 11 fails the call and the next call is the one of a
    fresh context"""
    import torch
    B, n = 16, 3
    trajs, keys = [], []
    for b in range(B):
        tr = R.traj(synth, 60 + b, n, n_az=MIXED_AZ[b] if b != TINY_LANE else 900)
        keys.append(("VLP-16", 60 + b, MIXED_AZ[b]) if b != TINY_LANE else ("VLP-16-too-close", 60 + b, 900))
        trajs.append([_mostly_too_close(s) for s in tr] if b == TINY_LANE else tr)
    assert max(_ring_sizes(s).max() for s in trajs[-1]) >= 4090
    assert all(0 < (np.linalg.norm(s[:, :3], axis=1) >= 0.3).sum() < 2000 for s in trajs[TINY_LANE])
    dev = [R.to_device(tr) for tr in trajs]
    ptrs, counts = _grid(trajs, dev)
    ctx = _mapped_ctx(aloam, trajs, B)
    odom, mapped = ctx.scan_stream_mapped_batch(ptrs, counts, True)
    stores = [R.snapshot(ctx, b) for b in range(B)]
    ctx.close()
    for b in range(B):
        _check_mapped_lane(aloam, None, synth, "lane %d" % b, trajs[b], keys[b], odom[:, b], mapped[:, b], stores[b], with_oracle=False)
    rings = [600] * 16; rings[3] = 4097
    over = torch.from_numpy(es.room_scan(rings)).cuda()
    bad_p, bad_c = ptrs[:1].copy(), counts[:1].copy()
    bad_p[0, 11], bad_c[0, 11] = over.data_ptr(), over.shape[0]
    kw = dict(n_scans=16, max_points=R.maxn(trajs) + 1024, max_batch=B, max_ring_points=4096)
    ctx, fresh = aloam.Aloam(**kw), aloam.Aloam(**kw)
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_batch(bad_p, bad_c, True)
    assert e.value.code == ERR_RING_TOO_LARGE
    after = ctx.scan_stream_batch(ptrs, counts, True)
    st_after = ctx.last_batch_stats
    ref = fresh.scan_stream_batch(ptrs, counts, True)
    assert np.array_equal(after, ref) and all(R.same_stats(a, b) for a, b in zip(st_after, fresh.last_batch_stats))
    assert np.array_equal(after, odom)
    ctx.close(); fresh.close()


def _plan(placed, steps, lanes):
    """placed: (trajectory, lane, start step, length) -> ops, and per entry the trajectory and scan index (-1: idle)"""
    ops = np.zeros((steps, lanes), np.int32)
    who = np.full((steps, lanes), -1)
    idx = np.full((steps, lanes), -1)
    for t, lane, s, ln in placed:
        assert (who[s:s + ln, lane] == -1).all()
        for i in range(ln):
            ops[s + i, lane] = START if i == 0 else SCAN
            who[s + i, lane], idx[s + i, lane] = t, i
    return ops, who, idx


def _run_lanes(ctx, trajs, placed, steps, lanes, split):
    """the schedule in two calls, device-resident up to `split`, host buffers after it -> odom, map poses, who"""
    ops, who, idx = _plan(placed, steps, lanes)
    dev = {t: R.to_device(trajs[t]) for t in trajs}
    dptrs = np.zeros((steps, lanes), np.uint64)
    hptrs = np.zeros((steps, lanes), np.uint64)
    counts = np.zeros((steps, lanes), np.int64)
    for (k, b), t in np.ndenumerate(who):
        if t >= 0:
            dptrs[k, b] = dev[t][idx[k, b]].data_ptr()
            hptrs[k, b] = trajs[t][idx[k, b]].ctypes.data
            counts[k, b] = trajs[t][idx[k, b]].shape[0]
    o1, m1 = ctx.scan_stream_lanes(dptrs[:split], counts[:split], ops[:split], True)
    o2, m2 = ctx.scan_stream_lanes(hptrs[split:], counts[split:], ops[split:], False)
    odom, mapped = np.concatenate([o1, o2]), np.concatenate([m1, m2])
    assert np.isnan(odom[ops == IDLE]).all() and np.isfinite(odom[ops != IDLE]).all() and np.isfinite(mapped[ops != IDLE]).all()
    return odom, mapped, who


def _rows(poses, who, t):
    ks, bs = np.nonzero(who == t)
    return poses[ks, bs]


def _check_schedule(aloam, orc, synth, ctx, trajs, placed, odom, mapped, who, distortion=0, with_oracle=False):
    last_of_lane = {lane: t for t, lane, s, ln in placed}   # placed in start order per lane
    stores = {lane: R.snapshot(ctx, lane) for lane in last_of_lane}
    for t, lane, start, ln in placed:
        _check_mapped_lane(aloam, orc, synth, "lane %d from step %d" % (lane, start), trajs[t], ("VLP-16", t, 900), _rows(odom, who, t),
                           _rows(mapped, who, t), stores[lane] if last_of_lane[lane] == t else None, distortion=distortion,
                           with_oracle=with_oracle)


def _schedule16(steps=12):
    """lane 9 alone (steps 0-1), lanes 9 and 15 alone (2-3), all 16 lanes (4), then lanes 1, 5, 9, 13, 15 refill with
    trajectories of 1 to 4 scans up to the last step while the others go idle"""
    placed, t = [], 100
    for lane in range(16):
        start, ln = {9: (0, 9), 15: (2, 6)}.get(lane, (4, 2 + lane % 5))
        placed.append((t, lane, start, ln)); t += 1
        end, i = start + ln, 0
        while (lane % 4 == 1 or lane == 15) and end < steps:
            ln = min((3, 1, 4, 2)[(lane + i) % 4], steps - end)
            placed.append((t, lane, end, ln)); t += 1
            end, i = end + ln, i + 1
    return sorted(placed, key=lambda p: p[2]), steps


def test_lane_schedule_at_width_16_mapped(aloam, synth):
    placed, steps = _schedule16()
    trajs = {t: R.traj(synth, t, ln) for t, lane, s, ln in placed}
    ctx = _mapped_ctx(aloam, list(trajs.values()), 16)
    odom, mapped, who = _run_lanes(ctx, trajs, placed, steps, 16, 5)
    assert (who[:2, :9] == -1).all() and (who[:2, 10:] == -1).all() and (who[2:4] >= 0).sum(1).tolist() == [2, 2]
    assert (who[4] >= 0).all() and who[-1, 9] >= 0
    _check_schedule(aloam, None, synth, ctx, trajs, placed, odom, mapped, who)
    # a 5-lane call: lanes 5 .. 15 are idle in it, so they stop running and a SCAN on lane 9 is refused
    t0 = trajs[placed[0][0]]
    p = np.array([[t0[0].ctypes.data] * 5], np.uint64)
    c = np.array([[t0[0].shape[0]] * 5])
    o, m = ctx.scan_stream_lanes(p, c, np.full((1, 5), START, np.int32), False)
    assert np.array_equal(o[0], np.tile([0, 0, 0, 1.0, 0, 0, 0], (5, 1)))
    ops = np.zeros((1, 16), np.int32); ops[0, 9] = SCAN
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_lanes(np.tile(p[:, :1], (1, 16)), np.tile(c[:, :1], (1, 16)), ops, False)
    assert e.value.code == ERR_STATE
    ctx.close()


def test_deskew_stream_equals_per_scan_calls(aloam, orc, synth):
    """distortion = 1: aloam_scan_stream (two calls) == aloam_scan_to_pose scan by scan, and within 1e-4 of the oracle
    (relTime can differ by one ulp from the CPU's atan2, test_gpu_deskew.py)"""
    n = 6
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    kw = dict(n_scans=16, max_points=R.maxn([scans]) + 1024, max_ring_points=4096, distortion=1)
    a, b = aloam.Aloam(**kw), aloam.Aloam(**kw)
    ptrs = np.array([d.data_ptr() for d in dev], np.uint64)
    counts = np.array([s.shape[0] for s in scans])
    poses = np.concatenate([a.scan_stream(ptrs[s], counts[s], True)[0] for s in R.splits_of(n, (4, 2))])
    for k in range(n):
        q, t, _ = b.scan_to_pose(scans[k])
        assert np.array_equal(np.concatenate([q, t]), poses[k]), k
    a.close(); b.close()
    o, _ = R.oracle(orc, synth, scans, ("VLP-16", 0, 900), False, distortion=1)
    R.assert_near(poses, o, "de-skewed stream")


@pytest.mark.parametrize("B", [4, 16])
def test_deskew_odometry_batch(aloam, orc, synth, B):
    n, sizes = 5, (3, 2)
    trajs = [R.traj(synth, t, n) for t in range(B)]
    dev = [R.to_device(tr) for tr in trajs]
    ptrs, counts = _grid(trajs, dev)
    ctx = aloam.Aloam(n_scans=16, max_points=R.maxn(trajs) + 1024, max_batch=B, max_ring_points=4096, distortion=1)
    poses = np.concatenate([ctx.scan_stream_batch(ptrs[s], counts[s], True) for s in R.splits_of(n, sizes)])
    stats = ctx.last_batch_stats
    ctx.close()
    for b in range(B):
        key = ("VLP-16", b, 900)
        s = R.solo(aloam, trajs[b], key, False, 1, sizes)
        assert np.array_equal(poses[:, b], s["odom"]), "lane %d differs from its solo run" % b
        assert R.same_stats(stats[b], s["stats"]), (b, stats[b], s["stats"])
        o, _ = R.oracle(orc, synth, trajs[b], key, False, distortion=1)
        R.assert_near(poses[:, b], o, "de-skewed lane %d of %d" % (b, B))


def test_deskew_mapped_batch_and_lane_schedule(aloam, orc, synth):
    """distortion = 1: 13 lockstep mapped lanes, then (after a reset) a 7-lane refill schedule on the same context"""
    B, n = 13, 6
    trajs = [R.traj(synth, t, n) for t in range(B)]
    dev = [R.to_device(tr) for tr in trajs]
    lengths = [5, 3, 6, 2, 4, 5, 3, 4, 2]
    free_at, placed = [0] * 7, []
    for i, ln in enumerate(lengths):
        lane = min(range(7), key=lambda l: (free_at[l], l))
        placed.append((200 + i, lane, free_at[lane], ln))
        free_at[lane] += ln
    placed.sort(key=lambda p: p[2])
    strajs = {t: R.traj(synth, t, ln) for t, lane, s, ln in placed}
    ctx = _mapped_ctx(aloam, trajs + list(strajs.values()), 16, distortion=1)
    odom, mapped = _mapped_batch_two_calls(ctx, trajs, dev, 4)
    for b in range(B):
        _check_mapped_lane(aloam, orc, synth, "de-skewed lane %d" % b, trajs[b], ("VLP-16", b, 900), odom[:, b], mapped[:, b],
                           R.snapshot(ctx, b), (4, 2), distortion=1)
    ctx.reset_odometry()
    odom, mapped, who = _run_lanes(ctx, strajs, placed, max(free_at), 7, 3)
    _check_schedule(aloam, orc, synth, ctx, strajs, placed, odom, mapped, who, distortion=1, with_oracle=True)
    ctx.close()


def _pad8(raw, rng):
    """32-byte points: x, y, z, intensity, then four pad floats that must never be read"""
    out = np.empty((len(raw), 8), np.float32)
    out[:, :4] = raw
    out[:, 4:] = rng.choice(np.array([np.nan, 1e30, -7.0, 3.5], np.float32), (len(raw), 4))
    return out


def test_stride8_streams_from_host_buffers(aloam, synth):
    import torch
    B, n = 5, 4
    rng = np.random.default_rng(8)
    trajs = [R.traj(synth, t, n) for t in range(B)]
    wide = [[_pad8(s, rng) for s in tr] for tr in trajs]
    p4, counts = _grid(trajs)
    p8, _ = _grid(wide)
    ctx = _mapped_ctx(aloam, trajs, B)
    o4, m4 = ctx.scan_stream_mapped_batch(p4, counts, False)
    s4 = [R.snapshot(ctx, b) for b in range(B)]
    ctx.reset_odometry()
    ctx.mapper_reset()
    o8, m8 = ctx.scan_stream_mapped_batch(p8, counts, False, stride=8)
    assert np.array_equal(o4, o8) and np.array_equal(m4, m8)
    for b in range(B):
        R.same_store(R.snapshot(ctx, b), s4[b], "stride-8 lane %d" % b)
    ctx.reset_odometry()
    assert np.array_equal(ctx.scan_stream_batch(p8, counts, False, stride=8), o4)
    # one step that mixes strides (the second step, lane 3) is refused, by the lockstep and the lane-scheduled calls
    views = aloam._views(p4[:2], counts[:2], 4)
    views[B + 3] = aloam.CloudView(C.cast(C.c_void_p(int(p8[1, 3])), C.POINTER(C.c_float)), int(counts[1, 3]), 8)
    poses, maps = np.zeros((2, B, 7)), np.zeros((2, B, 7))
    L = aloam.lib()
    assert L.aloam_scan_stream_batch(ctx._h, views, 2, B, 0, aloam._dp(poses), (aloam.Stats * B)()) == ERR_INVALID_ARG
    assert L.aloam_scan_stream_mapped_batch(ctx._h, views, 2, B, 0, aloam._dp(poses), aloam._dp(maps), (aloam.Stats * B)()) == ERR_INVALID_ARG
    ops = np.full((2, B), SCAN, np.int32); ops[0] = START
    assert L.aloam_scan_stream_lanes(ctx._h, views, ops.ctypes.data_as(C.POINTER(C.c_int)), 2, B, 0, aloam._dp(poses), aloam._dp(maps),
                                     (aloam.Stats * B)()) == ERR_INVALID_ARG
    # a device-resident stride-8 view is refused
    d8 = [[torch.from_numpy(s).cuda() for s in tr] for tr in wide]
    dp8, _ = _grid(wide, d8)
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_batch(dp8[:1], counts[:1], True, stride=8)
    assert e.value.code == ERR_INVALID_ARG
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_lanes(dp8[:1], counts[:1], np.full((1, B), START, np.int32), True, stride=8)
    assert e.value.code == ERR_INVALID_ARG
    # none of the refused calls changed the context: the odometry goes on from the stride-8 batch
    ctx.reset_odometry()
    assert np.array_equal(ctx.scan_stream_batch(p4, counts, False), o4)
    ctx.close()
