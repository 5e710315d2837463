"""GPU parity of the batched mapped stream (aloam_scan_stream_mapped_batch): several trajectories advance in lockstep
through odometry and scan-to-map in one context.  Every lane must be bit-identical to its solo run through
aloam_scan_stream_mapped on a fresh context -- poses, mapper state and every cube of its store -- its odometry must equal
aloam_scan_stream_batch, and lane 0 must follow the oracle's ascanRegistration | alaserOdometry | alaserMapping chain."""
import numpy as np
import pytest

from conftest import rot_angle

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_EMPTY_CLOUD, ERR_STATE = -1, -3, -9


def _trajectories(synth, sensor, n_traj, n_scans, n_az=None):
    return [[synth.scan(sensor, k, seed=synth.BASE_SEED + 50 + b, n_az=n_az) for k in range(n_scans)] for b in range(n_traj)]


def _addresses(trajs, n_scans, device):
    """(n_scans, lanes) addresses and counts; device: torch tensors on cuda:0 (kept alive by the caller)"""
    n_traj = len(trajs)
    src = [[device[b][k].data_ptr() for b in range(n_traj)] for k in range(n_scans)] if device is not None else \
        [[trajs[b][k].ctypes.data for b in range(n_traj)] for k in range(n_scans)]
    counts = np.array([[trajs[b][k].shape[0] for b in range(n_traj)] for k in range(n_scans)])
    return np.array(src, np.uint64), counts


def _same_state(a, b):
    return (a["centre"] == b["centre"] and a["valid"] == b["valid"] and np.array_equal(a["q_wmap_wodom"], b["q_wmap_wodom"])
            and np.array_equal(a["t_wmap_wodom"], b["t_wmap_wodom"]) and (a["total_corner"], a["total_surf"]) == (b["total_corner"], b["total_surf"]))


def _same_store(ctx_a, lane_a, ctx_b, lane_b):
    """state and every cube of the last frame's valid block, both cloud types, bit for bit"""
    sa, sb = ctx_a.mapper_state(lane_a), ctx_b.mapper_state(lane_b)
    assert _same_state(sa, sb), (lane_a, lane_b)
    for idx in sa["valid"]:
        for which in (0, 1):
            a, b = ctx_a.mapper_cube(which, idx, lane_a), ctx_b.mapper_cube(which, idx, lane_b)
            assert a.view(np.int32).tobytes() == b.view(np.int32).tobytes(), (lane_a, idx, which)
    assert sa["total_corner"] + sa["total_surf"] > 0


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


def _ctx(aloam, ns, maxn, max_ring, batch):
    return aloam.Aloam(n_scans=ns, max_points=maxn + 1024, max_map_points=400000, max_batch=batch, max_ring_points=max_ring)


@pytest.mark.parametrize("sensor,n_traj,max_ring", [("HDL-32", 4, 2304), ("HDL-64", 3, 2048), ("VLP-16", 16, 4096)])
def test_mapped_batch_equals_solo_and_oracle(aloam, orc, synth, sensor, n_traj, max_ring):
    import torch
    n_scans = 6
    ns = synth.SENSORS[sensor][0]
    trajs = _trajectories(synth, sensor, n_traj, n_scans, n_az=900 if sensor == "VLP-16" else None)
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    dptrs, counts = _addresses(trajs, n_scans, dev)
    hptrs, _ = _addresses(trajs, n_scans, None)
    ctx = _ctx(aloam, ns, maxn, max_ring, n_traj)
    # two calls, 4 scans device-resident then 2 from host buffers: the state of every lane carries over
    o1, m1 = ctx.scan_stream_mapped_batch(dptrs[:4], counts[:4], True)
    o2, m2 = ctx.scan_stream_mapped_batch(hptrs[4:], counts[4:], False)
    odom, mapped = np.concatenate([o1, o2]), np.concatenate([m1, m2])
    assert odom.shape == mapped.shape == (n_scans, n_traj, 7)
    # the odometry is aloam_scan_stream_batch's
    ob = aloam.Aloam(n_scans=ns, max_points=maxn + 1024, max_batch=n_traj, max_ring_points=max_ring)
    assert np.array_equal(ob.scan_stream_batch(dptrs, counts, True), odom)
    ob.close()
    for b in range(min(n_traj, 4)):
        solo = _ctx(aloam, ns, maxn, max_ring, 1)
        so1, sm1 = solo.scan_stream_mapped(dptrs[:4, b], counts[:4, b], True)
        so2, sm2 = solo.scan_stream_mapped(hptrs[4:, b], counts[4:, b], False)
        assert np.array_equal(np.concatenate([so1, so2]), odom[:, b]), "odometry of lane %d differs from its solo run" % b
        assert np.array_equal(np.concatenate([sm1, sm2]), mapped[:, b]), "map poses of lane %d differ from its solo run" % b
        _same_store(ctx, b, solo, 0)
        solo.close()
    ref = _oracle_map_poses(orc, synth, trajs[0], sensor, ctx.cfg.line_res, ctx.cfg.plane_res)   # the sensor's default leaves
    assert np.abs(mapped[:, 0, 4:] - ref[:, 4:]).max() < 1e-4
    assert max(rot_angle(mapped[k, 0, :4], ref[k, :4]) for k in range(n_scans)) < 1e-4
    ctx.close()


def test_host_path_equals_device_path_after_reset(aloam, synth):
    import torch
    n_scans, n_traj = 4, 3
    trajs = _trajectories(synth, "VLP-16", n_traj, n_scans, n_az=900)
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    dptrs, counts = _addresses(trajs, n_scans, dev)
    hptrs, _ = _addresses(trajs, n_scans, None)
    ctx = _ctx(aloam, 16, maxn, 4096, n_traj)
    od, md = ctx.scan_stream_mapped_batch(dptrs, counts, True)
    ctx.reset_odometry()
    ctx.mapper_reset()   # every lane back to a fresh store
    oh, mh = ctx.scan_stream_mapped_batch(hptrs, counts, False)
    assert np.array_equal(od, oh) and np.array_equal(md, mh)
    ctx.close()


def test_lanes_do_not_interfere(aloam, synth):
    """the same trajectory in every lane: identical poses and identical stores everywhere"""
    import torch
    n_scans, n_traj = 5, 4
    raws = _trajectories(synth, "VLP-16", 1, n_scans, n_az=900)[0]
    maxn = max(r.shape[0] for r in raws)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    ptrs = np.array([[d.data_ptr()] * n_traj for d in dev], np.uint64)
    counts = np.array([[r.shape[0]] * n_traj for r in raws])
    ctx = _ctx(aloam, 16, maxn, 4096, n_traj)
    odom, mapped = ctx.scan_stream_mapped_batch(ptrs, counts, True)
    for b in range(1, n_traj):
        assert np.array_equal(odom[:, b], odom[:, 0]) and np.array_equal(mapped[:, b], mapped[:, 0]), b
        _same_store(ctx, b, ctx, 0)
    ctx.close()


def test_batch_of_one_is_the_solo_call(aloam, synth):
    import torch
    n_scans = 5
    raws = _trajectories(synth, "HDL-32", 1, n_scans)[0]
    maxn = max(r.shape[0] for r in raws)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    ptrs = np.array([[d.data_ptr()] for d in dev], np.uint64)
    counts = np.array([[r.shape[0]] for r in raws])
    a = _ctx(aloam, 32, maxn, 2304, 1)
    ob, mb = a.scan_stream_mapped_batch(ptrs, counts, True)
    b = _ctx(aloam, 32, maxn, 2304, 1)
    os_, ms = b.scan_stream_mapped(ptrs[:, 0], counts[:, 0], True)
    assert np.array_equal(ob[:, 0], os_) and np.array_equal(mb[:, 0], ms)
    _same_store(a, 0, b, 0)
    a.close(); b.close()


def test_mapper_launches_are_shared_by_all_lanes(aloam, synth):
    """the mapper stage (mapped stream minus odometry-only stream, same scans) issues the same launches for 1, 2 and 4 lanes:
    every launch of the frame, both segmented filters included, covers all lanes"""
    import torch
    n_scans = 3
    trajs = _trajectories(synth, "VLP-16", 4, n_scans, n_az=900)
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    ptrs, counts = _addresses(trajs, n_scans, dev)
    extra = []
    for B in (1, 2, 4):
        mapped = _ctx(aloam, 16, maxn, 4096, B)
        odo = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_batch=B, max_ring_points=4096)
        # a first call creates the lanes (and, for B = 1, the context's map buffers that lane 0 shares): count the second
        mapped.scan_stream_mapped_batch(ptrs[:, :B], counts[:, :B], True)
        odo.scan_stream_batch(ptrs[:, :B], counts[:, :B], True)
        l0 = mapped.launch_count()
        mapped.scan_stream_mapped_batch(ptrs[:, :B], counts[:, :B], True)
        l1 = odo.launch_count()
        odo.scan_stream_batch(ptrs[:, :B], counts[:, :B], True)
        extra.append((mapped.launch_count() - l0) - (odo.launch_count() - l1))
        mapped.close(); odo.close()
    assert extra[0] > 0 and extra == [extra[0]] * 3, extra


def test_lanes_are_created_lazily_and_keep_their_state(aloam, synth):
    """a max_batch = 4 context driven with 2 lanes has no store for lanes 2-3; a later 4-lane call creates them fresh while
    lanes 0-1 go on with their cube stores (the odometry is reset in between, so lanes 2-3 start their trajectory too)"""
    import torch
    n_traj = 4
    trajs = _trajectories(synth, "VLP-16", n_traj, 5, n_az=900)
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    ptrs, counts = _addresses(trajs, 5, dev)
    ctx = _ctx(aloam, 16, maxn, 4096, n_traj)
    o1, m1 = ctx.scan_stream_mapped_batch(ptrs[:3, :2], counts[:3, :2], True)
    for lane in (2, 3):
        with pytest.raises(aloam.AloamError) as e:
            ctx.mapper_state(lane)
        assert e.value.code == ERR_STATE
        with pytest.raises(aloam.AloamError) as e:
            ctx.mapper_cube(1, 0, lane)
        assert e.value.code == ERR_STATE
    with pytest.raises(aloam.AloamError) as e:
        ctx.mapper_state(16)   # beyond ALOAM_MAX_BATCH
    assert e.value.code == ERR_INVALID_ARG
    ctx.reset_odometry()
    o2, m2 = ctx.scan_stream_mapped_batch(ptrs[3:], counts[3:], True)
    for b in range(n_traj):
        solo = _ctx(aloam, 16, maxn, 4096, 1)
        if b < 2:   # the same call sequence: 3 scans, odometry reset, 2 scans into the same cube store
            so1, sm1 = solo.scan_stream_mapped(ptrs[:3, b], counts[:3, b], True)
            assert np.array_equal(o1[:, b], so1) and np.array_equal(m1[:, b], sm1), b
            solo.reset_odometry()
        so2, sm2 = solo.scan_stream_mapped(ptrs[3:, b], counts[3:, b], True)
        assert np.array_equal(o2[:, b], so2) and np.array_equal(m2[:, b], sm2), b
        _same_store(ctx, b, solo, 0)
        solo.close()
    ctx.close()


def test_mapped_batch_argument_checks(aloam, synth):
    import torch
    raw = synth.scan("VLP-16", 0, n_az=900)
    d = torch.from_numpy(raw).cuda()
    n = raw.shape[0]
    ctx = aloam.Aloam(n_scans=16, max_points=n + 1024, max_map_points=400000, max_batch=2)
    with pytest.raises(aloam.AloamError) as e:   # more trajectories than the context was created for
        ctx.scan_stream_mapped_batch(np.full((1, 3), d.data_ptr(), np.uint64), np.full((1, 3), n), True)
    assert e.value.code == ERR_INVALID_ARG
    import ctypes as C
    views = (aloam.CloudView * 2)(*[aloam.CloudView(C.cast(C.c_void_p(d.data_ptr()), C.POINTER(C.c_float)), n, 4)] * 2)
    odom = np.zeros((1, 2, 7))
    rc = aloam.lib().aloam_scan_stream_mapped_batch(ctx._h, views, 1, 2, 1, aloam._dp(odom), None, None)   # map_poses NULL
    assert rc == ERR_INVALID_ARG
    no_map = aloam.Aloam(n_scans=16, max_points=n + 1024, max_batch=2)   # max_map_points = 0
    with pytest.raises(aloam.AloamError) as e:
        no_map.scan_stream_mapped_batch(np.full((1, 2), d.data_ptr(), np.uint64), np.full((1, 2), n), True)
    assert e.value.code == ERR_INVALID_ARG
    no_map.close()
    far = raw.copy(); far[:, :3] *= 1e-3    # everything closer than minimum_range: nothing survives (scanRegistration.cpp:137)
    dfar = torch.from_numpy(far).cuda()
    with pytest.raises(aloam.AloamError) as e:
        ctx.scan_stream_mapped_batch(np.array([[d.data_ptr(), dfar.data_ptr()]], np.uint64), np.full((1, 2), n), True)
    assert e.value.code == ERR_EMPTY_CLOUD
    # the context is usable afterwards (the odometry was reset, the mappers go on)
    o, m = ctx.scan_stream_mapped_batch(np.full((2, 2), d.data_ptr(), np.uint64), np.full((2, 2), n), True)
    assert np.isfinite(o).all() and np.isfinite(m).all()
    ctx.close()
