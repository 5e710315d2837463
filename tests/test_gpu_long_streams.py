"""Long pipelined streams and the call-size limit.  The stream driver cycles 4 feature slots, 3 ScanScalars slots and 2
raw / ring-major buffers, and its mapping stage may lag the odometry by up to 4 frames; a call holds at most 4096
(scan, lane) entries.  Calls of 1, 2, 3, ... scans put the call boundaries on every residue of the frame counter mod 4,
3 and 2, and a call of exactly 4096 entries uses both ends of every per-entry buffer."""
import numpy as np
import pytest

import lane_refs as R

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG = -1
KEY = ("VLP-16", 0, 900)


def _call_sizes(n, longest):
    """1, 2, ..., longest, 1, 2, ... cut to add up to n"""
    sizes, k = [], 0
    while sum(sizes) < n:
        sizes.append(min(k % longest + 1, n - sum(sizes)))
        k += 1
    return sizes


def _boundaries_cover_every_residue(sizes):
    inner = np.cumsum(sizes)[:-1]
    return all(set(inner % m) == set(range(m)) for m in (4, 3, 2))


def test_long_mapped_stream_equals_per_scan_calls_and_oracle(aloam, orc, synth):
    """64 scans through aloam_scan_stream_mapped in calls of 1 .. 7 scans, device-resident and host buffers in turn ==
    aloam_scan_to_pose, then aloam_extract_features -> aloam_mapper_step, scan by scan, and within 1e-4 of the oracle.
    The map filters with 0.5 / 1.0 m leaves: at the VLP-16's 0.2 m corner leaf the cube ahead of the sensor outgrows its
    slab (min(16384, max_points) points) after about 17 scans of this scene, and from then on the store drops points the
    reference keeps (ALOAM_FLAG_CUBE_OVERFLOW); at 0.5 m the largest cube stays below 12 000 points for all 64 scans."""
    n = 64
    sizes = _call_sizes(n, 7)
    assert _boundaries_cover_every_residue(sizes), sizes
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    counts = np.array([s.shape[0] for s in scans])
    leaves = (0.5, 1.0)
    kw = dict(n_scans=16, max_points=R.maxn([scans]) + 1024, max_map_points=400000, max_ring_points=4096, line_res=leaves[0],
              plane_res=leaves[1])
    c = aloam.Aloam(**kw)
    odom, mapped = [], []
    for i, s in enumerate(R.splits_of(n, sizes)):
        on_device = i % 2 == 0
        ptrs = [dev[k].data_ptr() if on_device else scans[k].ctypes.data for k in range(s.start, s.stop)]
        o, m = c.scan_stream_mapped(ptrs, counts[s], on_device)
        odom.append(o); mapped.append(m)
    odom, mapped = np.concatenate(odom), np.concatenate(mapped)
    store = R.snapshot(c, 0)
    c.close()
    c = aloam.Aloam(**kw)
    c.mapper_reset()
    for k, raw in enumerate(scans):
        q, t, _ = c.scan_to_pose(raw)
        assert np.array_equal(np.concatenate([q, t]), odom[k]), "odometry of scan %d" % k
        f = c.extract_features(raw)
        mq, mt, st = c.mapper_step(f["less_sharp"], f["less_flat"], q, t)
        assert np.array_equal(np.concatenate([mq, mt]), mapped[k]), "map pose of scan %d" % k
        assert not st["flags"] & aloam.FLAG_CUBE_OVERFLOW, k
    R.same_store(store, R.snapshot(c, 0), "store after 64 scans")
    c.close()
    o, m = R.oracle(orc, synth, scans, KEY, True, leaves=leaves)
    R.assert_near(odom, o, "odometry over 64 scans")
    R.assert_near(mapped, m, "map poses over 64 scans")


def test_long_batch_in_calls_of_every_length(aloam, synth):
    """16 lanes, 24 steps of aloam_scan_stream_batch in calls of 1, 2, 3, 4, 6, 7, 1 steps, device-resident and host
    buffers in turn: every lane equals its solo aloam_scan_stream run in one call"""
    B, n, sizes = 16, 24, [1, 2, 3, 4, 6, 7, 1]
    assert _boundaries_cover_every_residue(sizes)
    trajs = [R.traj(synth, t, n) for t in range(B)]
    dev = [R.to_device(tr) for tr in trajs]
    counts = np.array([[trajs[b][k].shape[0] for b in range(B)] for k in range(n)])
    ctx = aloam.Aloam(n_scans=16, max_points=R.maxn(trajs) + 1024, max_batch=B, max_ring_points=4096)
    poses = []
    for i, s in enumerate(R.splits_of(n, sizes)):
        on_device = i % 2 == 0
        ptrs = np.array([[dev[b][k].data_ptr() if on_device else trajs[b][k].ctypes.data for b in range(B)] for k in range(s.start, s.stop)],
                        np.uint64)
        poses.append(ctx.scan_stream_batch(ptrs, counts[s], on_device))
    stats = ctx.last_batch_stats
    ctx.close()
    poses = np.concatenate(poses)
    for b in range(B):
        so = R.solo(aloam, trajs[b], ("VLP-16", b, 900), False)
        assert np.array_equal(poses[:, b], so["odom"]), "lane %d differs from its solo run" % b
        assert R.same_stats(stats[b], so["stats"]), (b, stats[b], so["stats"])


def test_calls_of_4096_entries(aloam, synth):
    """16 lanes share one 256-scan trajectory: 256 steps are exactly 4096 entries, accepted (odometry and mapped); every
    lane equals lane 0, lane 0 its solo run.  4097 entries are refused and leave the context as it was"""
    B, n = 16, 256
    scans = R.traj(synth, 7, n)
    key = ("VLP-16", 7, 900)
    dev = R.to_device(scans)
    ptrs = np.array([[d.data_ptr()] * B for d in dev], np.uint64)
    counts = np.array([[s.shape[0]] * B for s in scans])
    maxpts = R.maxn([scans]) + 1024
    over_p, over_c = np.concatenate([ptrs, ptrs[:1]]), np.concatenate([counts, counts[:1]])   # 257 x 16 entries
    # odometry: one lane, 4097 scans, refused; then the same context runs the trajectory as a fresh one does
    one = aloam.Aloam(n_scans=16, max_points=maxpts, max_ring_points=4096)
    with pytest.raises(aloam.AloamError) as e:
        one.scan_stream(np.resize(ptrs[:, 0], 4097), np.resize(counts[:, 0], 4097), True)
    assert e.value.code == ERR_INVALID_ARG
    p1, _ = one.scan_stream(ptrs[:, 0], counts[:, 0], True)
    one.close()
    solo = R.solo(aloam, scans, key, False)
    assert np.array_equal(p1, solo["odom"])
    ctx = aloam.Aloam(n_scans=16, max_points=maxpts, max_batch=B, max_ring_points=4096)
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_batch(over_p, over_c, True)
    assert e.value.code == ERR_INVALID_ARG
    poses = ctx.scan_stream_batch(ptrs, counts, True)
    ctx.close()
    assert poses.shape == (n, B, 7) and np.array_equal(poses[:, 0], solo["odom"])
    for b in range(1, B):
        assert np.array_equal(poses[:, b], poses[:, 0]), "odometry of lane %d" % b
    # mapped
    ctx = aloam.Aloam(n_scans=16, max_points=maxpts, max_map_points=400000, max_batch=B, max_ring_points=4096)
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_mapped_batch(over_p, over_c, True)
    assert e.value.code == ERR_INVALID_ARG
    odom, mapped = ctx.scan_stream_mapped_batch(ptrs, counts, True)
    stores = [R.snapshot(ctx, b) for b in range(B)]
    ctx.close()
    solo = R.solo(aloam, scans, key, True)
    assert np.array_equal(odom[:, 0], solo["odom"]) and np.array_equal(mapped[:, 0], solo["map"])
    R.same_store(stores[0], solo["store"], "store of lane 0")
    for b in range(1, B):
        assert np.array_equal(odom[:, b], odom[:, 0]) and np.array_equal(mapped[:, b], mapped[:, 0]), "lane %d" % b
        R.same_store(stores[b], stores[0], "store of lane %d" % b)
