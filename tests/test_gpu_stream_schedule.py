"""GPU checks of what every scan stream call shares: one driver runs a lane schedule, and the lockstep calls are the schedule
where every lane STARTs at the context's first step and SCANs at every later one.  Pinned here: the stats of a lockstep call
(initialise-only exactly when a lane's last step was its first, the others as aloam_scan_to_pose / the solo stream report
them), and the lane state of aloam_scan_stream_lanes when a mapper frame fails with a key overflow (the lanes go on)."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_cubemap import _overflow_box

pytestmark = pytest.mark.gpu

ERR_CAPACITY = -4
STAT_KEYS = ("n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps", "flags", "termination", "init_cost", "final_cost")


def _same_stats(a, b):
    return all(a[k] == b[k] for k in STAT_KEYS)


def _trajs(synth, n_traj, n_scans, seed0):
    return [[synth.scan("VLP-16", k, seed=synth.BASE_SEED + seed0 + t, n_az=900) for k in range(n_scans)] for t in range(n_traj)]


def _maxn(trajs):
    return max(s.shape[0] for tr in trajs for s in tr)


def test_lockstep_stats_first_scan_initialises_then_as_scan_to_pose(aloam, synth):
    """a one-scan aloam_scan_stream on a fresh context only initialises; the next call reports what aloam_scan_to_pose
    reports for the same scan, with the same pose"""
    raws = _trajs(synth, 1, 2, seed0=500)[0]
    kw = dict(n_scans=16, max_points=_maxn([raws]) + 1024, max_ring_points=4096)
    stream, single = aloam.Aloam(**kw), aloam.Aloam(**kw)
    p0, st0 = stream.scan_stream([raws[0].ctypes.data], [raws[0].shape[0]], False)
    assert st0.flags == aloam.FLAG_INITIALISED_ONLY and st0.lm_iters == 0
    assert np.array_equal(p0[0], [0, 0, 0, 1, 0, 0, 0])
    _, _, s0 = single.scan_to_pose(raws[0])
    assert s0["flags"] == aloam.FLAG_INITIALISED_ONLY
    p1, st1 = stream.scan_stream([raws[1].ctypes.data], [raws[1].shape[0]], False)
    q, t, s1 = single.scan_to_pose(raws[1])
    assert np.array_equal(p1[0], np.concatenate([q, t]))
    assert not st1.flags & aloam.FLAG_INITIALISED_ONLY and st1.lm_iters > 0
    assert _same_stats(st1.as_dict(), s1), (st1.as_dict(), s1)
    stream.close(); single.close()


def test_batch_stats_per_lane_equal_solo_stream(aloam, synth):
    """aloam_scan_stream_batch over two calls (one step, then three): every lane's stats are those of its trajectory run
    alone through aloam_scan_stream with the same calls"""
    B, n = 3, 4
    trajs = _trajs(synth, B, n, seed0=510)
    ptrs = np.array([[trajs[b][k].ctypes.data for b in range(B)] for k in range(n)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(B)] for k in range(n)])
    kw = dict(n_scans=16, max_points=_maxn(trajs) + 1024, max_ring_points=4096)
    ctx = aloam.Aloam(max_batch=B, **kw)
    batch_stats = []
    for s in (slice(0, 1), slice(1, n)):
        ctx.scan_stream_batch(ptrs[s], counts[s], False)
        batch_stats.append(ctx.last_batch_stats)
    assert all(st["flags"] == aloam.FLAG_INITIALISED_ONLY for st in batch_stats[0])
    for b in range(B):
        solo = aloam.Aloam(**kw)
        for call, s in enumerate((slice(0, 1), slice(1, n))):
            _, st = solo.scan_stream(ptrs[s, b], counts[s, b], False)
            assert _same_stats(batch_stats[call][b], st.as_dict()), (call, b, batch_stats[call][b], st.as_dict())
        solo.close()
    assert batch_stats[1][0]["lm_iters"] > 0
    ctx.close()


def test_lanes_key_overflow_fills_the_poses_and_the_lanes_go_on(aloam, synth):
    """a mapped aloam_scan_stream_lanes call whose frame re-filters a cube beyond the key width returns ALOAM_ERR_CAPACITY
    with every pose row filled; the lanes keep running (a following SCAN is accepted) and their odometry is the lockstep
    batch's"""
    import torch
    B, n = 2, 3
    trajs = _trajs(synth, B, n, seed0=520)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    ptrs = np.array([[dev[b][k].data_ptr() for b in range(B)] for k in range(n)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(B)] for k in range(n)])
    maxn = _maxn(trajs)
    ctx = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, max_batch=B, max_ring_points=4096,
                      line_res=0.02, plane_res=0.02)
    odom0, map0 = ctx.scan_stream_lanes(ptrs[:1], counts[:1], np.full((1, B), aloam.LANE_START, np.int32), True)
    # lane 0's store (the one the host API maps into) gets a cube whose index range needs more than 31 key bits, in the
    # valid block of the next scans
    rng = np.random.default_rng(59)
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    with pytest.raises(aloam.AloamError) as e:
        ctx.mapper_step(empty, _overflow_box(rng, (87.113, 87.113, 37.113)), ident, np.zeros(3))
    assert e.value.code == ERR_CAPACITY
    scan_ops = np.full((1, B), aloam.LANE_SCAN, np.int32)
    odom, mapped, rcs = [odom0], [map0], []
    for k in (1, 2):   # through the C ABI: the wrapper raises on the error and drops the poses
        views = (aloam.CloudView * B)(*[aloam.CloudView(C.cast(C.c_void_p(int(ptrs[k, b])), C.POINTER(C.c_float)), int(counts[k, b]), 4)
                                        for b in range(B)])
        o, m = np.zeros((1, B, 7)), np.zeros((1, B, 7))
        rcs.append(aloam.lib().aloam_scan_stream_lanes(ctx._h, views, scan_ops.ctypes.data_as(C.POINTER(C.c_int)), 1, B, 1,
                                                       aloam._dp(o), aloam._dp(m), (aloam.Stats * B)()))
        odom.append(o); mapped.append(m)
    assert rcs[0] == ERR_CAPACITY and rcs[1] in (0, ERR_CAPACITY), rcs
    odom, mapped = np.concatenate(odom), np.concatenate(mapped)
    assert np.isfinite(odom).all() and np.isfinite(mapped).all()
    ref = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_batch=B, max_ring_points=4096)
    assert np.array_equal(ref.scan_stream_batch(ptrs, counts, True), odom)
    ref.close(); ctx.close()
