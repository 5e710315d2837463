"""GPU: mapping_skip_frame in the mapped stream calls.  Scan j of a trajectory (0 at its START) goes to the mapper when
j % mapping_skip_frame == 0; every other scan gets the high-frequency pose T_wmap_wodom * odometry pose, with the T_wmap_wodom
of the lane's latest mapped scan (laserMapping.cpp:197-229), and leaves the cube store alone.  Pinned here: the odometry does
not change; mapped rows and stores equal aloam_mapper_step run on exactly the mapped scans; skipped rows equal the host
composition bit for bit; call boundaries, batches, lane schedules and emulated shards change nothing; the mapper is really
skipped (launch count); and the skip-aware oracle chain (tests/skip_refs.py) is within 1e-4."""
import math

import numpy as np
import pytest

import lane_refs as R
import skip_refs as S

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
N = 24
KEY = ("VLP-16", 0, 900)
_RUNS = {}


# 0.5 / 1.0 m leaves: at the VLP-16's 0.2 m corner leaf the cube ahead of the sensor outgrows its slab after about 17 scans of
# this scene and the store drops points the oracle keeps (see tests/test_gpu_long_streams.py)
LEAVES = (0.5, 1.0)


def _kw(scans_list, **extra):
    return dict(n_scans=16, max_points=R.maxn(scans_list) + 1024, max_map_points=400000, max_ring_points=4096, line_res=LEAVES[0],
                plane_res=LEAVES[1], **extra)


def _solo_skip(aloam, scans, key, skip, sizes=None):
    """the trajectory alone on a fresh context through aloam_scan_stream_mapped with mapping_skip_frame = skip, in calls of
    `sizes` (default one call; device-resident and host buffers in turn) -> (odom, map, store snapshot); cached"""
    sizes = tuple(sizes or (len(scans),))
    ck = (key, len(scans), skip, sizes)
    if ck not in _RUNS:
        dev = R.to_device(scans)
        counts = np.array([s.shape[0] for s in scans])
        c = aloam.Aloam(**_kw([scans], mapping_skip_frame=skip))
        odom, mp = [], []
        for i, s in enumerate(R.splits_of(len(scans), sizes)):
            on_device = i % 2 == 0
            ptrs = [dev[k].data_ptr() if on_device else scans[k].ctypes.data for k in range(s.start, s.stop)]
            o, m = c.scan_stream_mapped(ptrs, counts[s], on_device)
            odom.append(o); mp.append(m)
        _RUNS[ck] = (np.concatenate(odom), np.concatenate(mp), R.snapshot(c, 0))
        c.close()
    return _RUNS[ck]


def _per_scan_reference(aloam, orc, c, scans, skip, odom):
    """on context c (fresh or emulating a rank): aloam_scan_to_pose per scan; aloam_extract_features -> aloam_mapper_step on
    the mapped scans only; the host composition with aloam_mapper_debug_state's T_wmap_wodom on the others -> map rows"""
    c.mapper_reset()
    rows = []
    for j, raw in enumerate(scans):
        q, t, _ = c.scan_to_pose(raw)
        assert np.array_equal(np.concatenate([q, t]), odom[j]), "odometry of scan %d" % j
        if S.mapped(j, skip):
            f = c.extract_features(raw)
            mq, mt, _ = c.mapper_step(f["less_sharp"], f["less_flat"], q, t)
            rows.append(np.concatenate([mq, mt]))
        else:
            st = c.mapper_state()
            rows.append(orc.transform_associate_to_map(st["q_wmap_wodom"], st["t_wmap_wodom"], q, t))
    return np.array(rows)


def _same_rows(got, ref, what):
    bad = [j for j in range(len(ref)) if not np.array_equal(got[j], ref[j])]
    assert not bad, (what, "rows differ", bad)


@pytest.mark.parametrize("skip", [1, 2, 3, 5])
def test_single_trajectory_bit_identity(aloam, orc, synth, skip):
    scans = R.traj(synth, 0, N)
    odom, mapped, store = _solo_skip(aloam, scans, KEY, skip)
    odom1, mapped1, store1 = _solo_skip(aloam, scans, KEY, 1)
    assert np.array_equal(odom, odom1), "the odometry does not depend on mapping_skip_frame"
    c = aloam.Aloam(**_kw([scans]))
    ref = _per_scan_reference(aloam, orc, c, scans, skip, odom)
    _same_rows(mapped, ref, "skip %d vs aloam_mapper_step on the mapped scans + host composition" % skip)
    R.same_store(store, R.snapshot(c, 0), "store after %d scans, skip %d" % (N, skip))
    c.close()
    o_ref, m_ref = S.oracle_chain(orc, synth, scans, skip, KEY, leaves=LEAVES)
    R.assert_near(odom, o_ref, "odometry, skip %d" % skip)
    R.assert_near(mapped, m_ref, "map poses, skip %d" % skip)
    if skip > 1:   # the skipped rows are not the refined ones of a skip = 1 run
        assert any(not np.array_equal(mapped[j], mapped1[j]) for j in range(N) if not S.mapped(j, skip))
    else:          # today's results (every scan through aloam_mapper_step, above), also for a config whose field is left 0
        z = aloam.Aloam(**_kw([scans], mapping_skip_frame=0))
        assert z.cfg.mapping_skip_frame == 0
        dev = R.to_device(scans)
        oz, mz = z.scan_stream_mapped([d.data_ptr() for d in dev], [s.shape[0] for s in scans], True)
        assert np.array_equal(oz, odom) and np.array_equal(mz, mapped)
        R.same_store(R.snapshot(z, 0), store, "field left 0")
        z.close()


# call boundaries on every residue mod 2, 3, 4 and 5
SIZES = [1, 1, 1, 2, 4, 6, 5, 4]


@pytest.mark.parametrize("skip", [2, 3, 5])
def test_call_boundaries_on_every_residue(aloam, synth, skip):
    assert sum(SIZES) == N and max(SIZES) <= 7
    inner = np.cumsum(SIZES)[:-1]
    assert all(set(inner % m) == set(range(m)) for m in (2, 3, 4, 5))
    scans = R.traj(synth, 0, N)
    one = _solo_skip(aloam, scans, KEY, skip)
    many = _solo_skip(aloam, scans, KEY, skip, SIZES)
    assert np.array_equal(many[0], one[0]) and np.array_equal(many[1], one[1])
    R.same_store(many[2], one[2], "calls of %s, skip %d" % (SIZES, skip))


def test_sixteen_lane_batch_with_skip_3(aloam, synth):
    import torch
    B, n, skip = 16, 7, 3
    trajs = [R.traj(synth, t, n) for t in range(B)]
    dev = [R.to_device(tr) for tr in trajs]
    ptrs = np.array([[dev[b][k].data_ptr() for b in range(B)] for k in range(n)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(B)] for k in range(n)])
    ctx = aloam.Aloam(**_kw(trajs, max_batch=B, mapping_skip_frame=skip))
    odom, mapped = ctx.scan_stream_mapped_batch(ptrs[:4], counts[:4], True)      # two calls: 4 + 3 steps
    o2, m2 = ctx.scan_stream_mapped_batch(ptrs[4:], counts[4:], True)
    odom, mapped = np.concatenate([odom, o2]), np.concatenate([mapped, m2])
    torch.cuda.synchronize()
    for b in range(B):
        so, sm, sst = _solo_skip(aloam, trajs[b], ("VLP-16", b, 900), skip)
        assert np.array_equal(odom[:, b], so) and np.array_equal(mapped[:, b], sm), "lane %d" % b
        R.same_store(R.snapshot(ctx, b), sst, "lane %d" % b)
    ctx.close()


I, Sc, St = 0, 1, 2   # LANE_IDLE, LANE_SCAN, LANE_START
# the staggered schedule: lane -> list of (start step, trajectory id, length) over 12 steps
PLAN = {0: [(0, 10, 12)], 1: [(0, 11, 5), (7, 12, 5)], 2: [(0, 13, 3), (5, 14, 7)], 3: [(0, 15, 4), (4, 16, 8)]}


def _staggered(synth, n=12):
    """PLAN as (n, lanes) arrays of ops, device addresses and counts, with the trajectories' scans by id"""
    B = len(PLAN)
    ops = np.full((n, B), I, np.int32)
    scans = {tid: R.traj(synth, tid, ln) for runs in PLAN.values() for (_, tid, ln) in runs}
    dev = {tid: R.to_device(sc) for tid, sc in scans.items()}
    ptrs = np.zeros((n, B), np.uint64)
    counts = np.zeros((n, B), np.int64)
    for lane, runs in PLAN.items():
        for s0, tid, ln in runs:
            for j in range(ln):
                ops[s0 + j, lane] = St if j == 0 else Sc
                ptrs[s0 + j, lane] = dev[tid][j].data_ptr()
                counts[s0 + j, lane] = scans[tid][j].shape[0]
    return ops, ptrs, counts, scans, dev


def _mapped_rows(ops, skip):
    """(n, lanes) booleans: the row's scan goes to the mapper, its lane's scan index counted from its START"""
    idx, m = {}, np.zeros(ops.shape, bool)
    for k in range(ops.shape[0]):
        for lane in range(ops.shape[1]):
            if ops[k, lane] != I:
                idx[lane] = 0 if ops[k, lane] == St else idx[lane] + 1
                m[k, lane] = S.mapped(idx[lane], skip)
    return m


def test_lane_schedule_with_staggered_starts_restarts_and_idle_lanes(aloam, synth):
    """4 lanes, 12 steps in two calls, skip 3.  Step 0 maps every lane, steps 1, 2 none, others a subset; lane 3 restarts at
    step 4 (its scan index starts again at 0), lanes 1 and 2 are idle for two steps between trajectories"""
    skip, n = 3, 12
    B = len(PLAN)
    ops, ptrs, counts, scans, dev = _staggered(synth, n)
    # the schedule covers the cases it is meant to
    maps = [[bool(m) for m, op in zip(row, ops[k]) if op != I] for k, row in enumerate(_mapped_rows(ops, skip))]
    assert all(maps[0]) and len(maps[0]) == B and not any(maps[1]) and not any(maps[2])
    assert any(any(m) and not all(m) for m in maps)
    assert ops[4, 3] == St and ops[3, 3] == Sc
    ctx = aloam.Aloam(**_kw(list(scans.values()), max_batch=B, mapping_skip_frame=skip))
    o1, m1 = ctx.scan_stream_lanes(ptrs[:6], counts[:6], ops[:6], True)
    o2, m2 = ctx.scan_stream_lanes(ptrs[6:], counts[6:], ops[6:], True)
    odom, mapped = np.concatenate([o1, o2]), np.concatenate([m1, m2])
    assert np.isnan(odom[ops == I]).all() and np.isnan(mapped[ops == I]).all()
    for lane, runs in PLAN.items():
        for s0, tid, ln in runs:
            so, sm, sst = _solo_skip(aloam, scans[tid], ("VLP-16", tid, 900), skip)
            rows = slice(s0, s0 + ln)
            assert np.array_equal(odom[rows, lane], so) and np.array_equal(mapped[rows, lane], sm), (lane, tid)
        R.same_store(R.snapshot(ctx, lane), sst, "lane %d, last trajectory" % lane)
    ctx.close()


def test_refused_lanes_calls_leave_the_skip_phase_alone(aloam, synth):
    """the staggered schedule in two calls with a registered sink, skip 3, refused calls between them: an op of 3, a SCAN on an
    idle lane after a step that advances the other lanes, an unmapped call on mapped lanes, and a call whose registered rows
    exceed the sink by one point.  The second call equals the uninterrupted run and the solo runs bit for bit."""
    import torch
    skip, n, cut = 3, 12, 6
    ops, ptrs, counts, scans, dev = _staggered(synth, n)
    B = ops.shape[1]
    second = int(counts[cut:][_mapped_rows(ops, skip)[cut:]].sum())   # points the second call registers
    assert second > 0

    def run(refusals):
        ctx = aloam.Aloam(**_kw(list(scans.values()), max_batch=B, mapping_skip_frame=skip))
        sink = torch.zeros((int(counts.sum()), 4), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        ctx.set_registered_sink(sink)
        ctx.scan_stream_lanes(ptrs[:cut], counts[:cut], ops[:cut], True)
        if refusals:
            p2, c2 = ptrs[cut:], counts[cut:]
            bad = ops[cut:].copy(); bad[2, 1] = 3
            with pytest.raises(aloam.AloamError) as e:
                ctx.scan_stream_lanes(p2, c2, bad, True)
            assert e.value.code == ERR_INVALID_ARG
            bad = ops[cut:].copy()
            assert bad[0, 1] == I and bad[1, 1] == St
            bad[1, 1] = Sc   # lane 1 has been idle since step 5
            with pytest.raises(aloam.AloamError) as e:
                ctx.scan_stream_lanes(p2, c2, bad, True)
            assert e.value.code == ERR_STATE
            with pytest.raises(aloam.AloamError) as e:
                ctx.scan_stream_lanes(p2, c2, ops[cut:], True, mapped=False)
            assert e.value.code == ERR_STATE
            ctx.set_registered_sink(sink[:second - 1])
            with pytest.raises(aloam.AloamError) as e:
                ctx.scan_stream_lanes(p2, c2, ops[cut:], True)
            assert e.value.code == ERR_CAPACITY
            ctx.set_registered_sink(sink[:second])
        o, m = ctx.scan_stream_lanes(ptrs[cut:], counts[cut:], ops[cut:], True)
        begin, count = ctx.registered_rows((n - cut) * B)
        assert count.sum() == second
        torch.cuda.synchronize()
        out = (o, m, begin, count, sink[:second].cpu().numpy().copy(), [R.snapshot(ctx, l) for l in range(B)])
        ctx.close()
        return out

    got, ref = run(True), run(False)
    for a, b, what in zip(got[:5], ref[:5], ("odometry", "map poses", "row begins", "row counts", "registered clouds")):
        assert np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), what
    for lane in range(B):
        R.same_store(got[5][lane], ref[5][lane], "lane %d against the uninterrupted run" % lane)
    for lane, runs in PLAN.items():
        for s0, tid, ln in runs:
            if s0 + ln <= cut:
                continue
            so, sm, sst = _solo_skip(aloam, scans[tid], ("VLP-16", tid, 900), skip)
            k0 = max(s0, cut)
            rows = slice(k0 - cut, s0 + ln - cut)
            assert np.array_equal(got[0][rows, lane], so[k0 - s0:]) and np.array_equal(got[1][rows, lane], sm[k0 - s0:]), (lane, tid)
        R.same_store(got[5][lane], sst, "lane %d, last trajectory" % lane)


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("exchange", [0, 1, 2])
def test_sharded_emulated_with_skip_2(aloam, orc, synth, world, exchange):
    skip, n, rank = 2, 8, world - 1
    scans = R.traj(synth, 0, n)
    ptrs, counts = [s.ctypes.data for s in scans], [s.shape[0] for s in scans]
    ctx = aloam.Aloam(**_kw([scans], mapping_skip_frame=skip))
    ctx.debug_shard_emulate(rank, world, exchange)
    odom, mapped = ctx.scan_stream_mapped(ptrs, counts, False)
    ctx.close()
    ref_ctx = aloam.Aloam(**_kw([scans], mapping_skip_frame=skip))
    ref_ctx.debug_shard_emulate(rank, world, exchange)
    ref = _per_scan_reference(aloam, orc, ref_ctx, scans, skip, odom)
    ref_ctx.close()
    _same_rows(mapped, ref, "rank %d of %d, exchange %d" % (rank, world, exchange))
    assert np.abs(mapped[::skip, 4:] - odom[::skip, 4:]).max() > 0   # the refinement ran


@pytest.mark.parametrize("skip", [2, 3])
def test_launch_count_shows_the_mapper_is_skipped(aloam, synth, skip):
    """launches of a mapped call minus those of the odometry-only call over the same scans = launches of one mapper frame x
    ceil(n / k) + one k_mapper_high_freq per step with a skipped scan"""
    n = 10
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    ptrs, counts = [d.data_ptr() for d in dev], [s.shape[0] for s in scans]

    def extra(k):
        mapped = aloam.Aloam(**_kw([scans], mapping_skip_frame=k))
        odo = aloam.Aloam(**_kw([scans]))
        mapped.scan_stream_mapped(ptrs, counts, True)    # creates the lanes and the map buffers
        odo.scan_stream(ptrs, counts, True)
        mapped.reset_odometry(); odo.reset_odometry()     # the scan index starts again at 0
        l0, l1 = mapped.launch_count(), odo.launch_count()
        mapped.scan_stream_mapped(ptrs, counts, True)
        odo.scan_stream(ptrs, counts, True)
        e = (mapped.launch_count() - l0) - (odo.launch_count() - l1)
        mapped.close(); odo.close()
        return e

    per_frame, rem = divmod(extra(1), n)
    assert rem == 0 and per_frame > 1
    n_mapped = math.ceil(n / skip)
    assert extra(skip) == per_frame * n_mapped + (n - n_mapped)


def test_negative_skip_is_refused(aloam):
    with pytest.raises(aloam.AloamError) as e:
        aloam.Aloam(n_scans=16, max_points=20000, max_map_points=1000, mapping_skip_frame=-1)
    assert e.value.code == ERR_INVALID_ARG
