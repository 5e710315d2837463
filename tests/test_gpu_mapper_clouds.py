"""GPU: the clouds the reference mapper publishes (laserMapping.cpp:806-848) -- the cube-store export (aloam_mapper_export:
/laser_cloud_surround and /laser_cloud_map) and the registered full-resolution scans of the mapped streams
(aloam_set_registered_sink / aloam_registered_rows: /velodyne_cloud_registered), bit for bit against the store's cubes, the
oracle and solo runs."""
import numpy as np
import pytest

import pyclouds

pytestmark = pytest.mark.gpu

W, H, D = 21, 21, 11
NCUBE = W * H * D
ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32).tobytes()


def _concat(clouds):
    clouds = [c for c in clouds if len(c)]
    return np.concatenate(clouds) if clouds else np.zeros((0, 4), np.float32)


def _device_cube_order(ctx, what, lane=0):
    """the reference's order through the one-cube test hook: corner then surf cube of every valid cube / of every cube"""
    idx = ctx.mapper_state(lane)["valid"] if what == 0 else range(NCUBE)
    return _concat([ctx.mapper_cube(ty, i, lane) for i in idx for ty in (0, 1)])


def _oracle_order(cm, what):
    idx = cm.state()["valid"] if what == 0 else range(NCUBE)
    return _concat([cm.cube(ty, i) for i in idx for ty in (0, 1)])


def _export_both(ctx, what, lane=0):
    """host (pageable) and device destinations must give the same bytes"""
    import torch
    host = ctx.mapper_export(what, lane)
    dev = torch.full((len(host) + 3, 4), -7.0, dtype=torch.float32, device="cuda")
    got = ctx.mapper_export(what, lane, out=dev)
    assert _bits(got.cpu().numpy()) == _bits(host)
    assert bool((dev[len(host):] == -7.0).all())   # nothing past the export
    return host


def test_export_equals_cubes_and_oracle_along_a_scrolling_path(aloam, orc):
    """the thin-cloud path of the cube-store tests (pose = odometry pose, cubes bit-exact with the oracle): after every frame the
    surround and the whole map equal the concatenation of the store's cubes in the reference's order, and the oracle's"""
    rng = np.random.default_rng(11)
    c = aloam.Aloam(n_scans=16, max_points=20000, max_map_points=200000, line_res=0.4, plane_res=0.8)
    c.mapper_reset()
    cm = orc.CubeMap()
    ident = np.array([0, 0, 0, 1.0])
    path = [(0, 0, 0), (60, -35, 12), (130, -80, 30), (260, -170, 75), (420, -290, 140), (-90, 40, -30), (-700, 600, -260), (200, -420, 200)]
    for k, t in enumerate(path):
        corner = (rng.normal(size=(6, 4)) * [8, 8, 2, 0]).astype(np.float32)
        surf = (rng.normal(size=(300, 4)) * [30, 30, 3, 0]).astype(np.float32)
        cm.step(corner, surf, ident, np.array(t, float), 0.4, 0.8)
        c.mapper_step(corner, surf, ident, np.array(t, float))
        sur = _export_both(c, aloam.EXPORT_SURROUND)
        assert _bits(sur) == _bits(_oracle_order(cm, 0)) and len(sur) > 0, k
        assert _bits(sur) == _bits(_device_cube_order(c, 0)), k
        mp = _export_both(c, aloam.EXPORT_MAP)
        assert _bits(mp) == _bits(_oracle_order(cm, 1)), k
        assert c.mapper_export_size(aloam.EXPORT_MAP) == len(mp) and len(mp) >= len(sur)
    c.close()


def test_export_of_mapped_batch_lanes(aloam, synth, scans):
    """every lane of a mapped batch: both exports equal the lane's cubes in the reference's order"""
    raws = [[scans("VLP-16", k + 2 * b, n_az=900) for k in range(5)] for b in range(3)]
    maxn = max(r.shape[0] for t in raws for r in t)
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, max_batch=3)
    ptrs = np.array([[raws[b][k].ctypes.data for b in range(3)] for k in range(5)], np.uint64)
    counts = np.array([[raws[b][k].shape[0] for b in range(3)] for k in range(5)])
    c.scan_stream_mapped_batch(ptrs, counts, False)
    for lane in range(3):
        for what in (aloam.EXPORT_SURROUND, aloam.EXPORT_MAP):
            got = _export_both(c, what, lane)
            assert len(got) > 0 and _bits(got) == _bits(_device_cube_order(c, what, lane)), (lane, what)
    c.close()


def test_export_arguments_and_capacity(aloam, scans):
    import torch
    raws = [scans("VLP-16", k, n_az=900) for k in range(3)]
    c = aloam.Aloam(n_scans=16, max_points=max(r.shape[0] for r in raws) + 1024, max_map_points=400000, max_batch=2)
    lib, h = aloam.lib(), c._h
    n = aloam.C.c_longlong(-1)
    assert lib.aloam_mapper_export(h, 0, 0, None, 0, aloam.C.byref(n)) == ERR_STATE      # no store yet
    c.mapper_reset()                                                                        # the empty store
    assert c.mapper_export_size(aloam.EXPORT_SURROUND) == 0 and c.mapper_export_size(aloam.EXPORT_MAP) == 0
    assert c.mapper_export(aloam.EXPORT_MAP).shape == (0, 4)
    c.scan_stream_mapped([r.ctypes.data for r in raws], [r.shape[0] for r in raws], False)
    total = c.mapper_export_size(aloam.EXPORT_MAP)
    assert total > 0
    assert lib.aloam_mapper_export(h, 1, 0, None, 0, aloam.C.byref(n)) == ERR_STATE      # lane 1 was never used
    assert lib.aloam_mapper_export(h, 16, 0, None, 0, aloam.C.byref(n)) == ERR_INVALID_ARG
    assert lib.aloam_mapper_export(h, -1, 0, None, 0, aloam.C.byref(n)) == ERR_INVALID_ARG
    assert lib.aloam_mapper_export(h, 0, 2, None, 0, aloam.C.byref(n)) == ERR_INVALID_ARG
    assert lib.aloam_mapper_export(h, 0, -1, None, 0, aloam.C.byref(n)) == ERR_INVALID_ARG
    for dev in (False, True):   # one point short: ALOAM_ERR_CAPACITY, the size reported, nothing written
        buf = torch.full((total - 1, 4), 3.5, dtype=torch.float32, device="cuda" if dev else "cpu")
        n.value = -1
        assert lib.aloam_mapper_export(h, 0, 1, aloam.C.c_void_p(buf.data_ptr()), total - 1, aloam.C.byref(n)) == ERR_CAPACITY
        assert n.value == total and bool((buf == 3.5).all())
    pinned = torch.zeros((total, 4), dtype=torch.float32).pin_memory()
    assert _bits(c.mapper_export(aloam.EXPORT_MAP, out=pinned).numpy()) == _bits(c.mapper_export(aloam.EXPORT_MAP))
    c.close()


# ---------------------------------------------------------------------------------------------------------------- registered scans


def _full(aloam, raw):
    """the ring-major full cloud of a scan (aloam_extract_features' `full`) from a context of its own"""
    e = aloam.Aloam(n_scans=16, max_points=raw.shape[0] + 1024)
    f = e.extract_features(raw)["full"]
    e.close()
    return f


def _sink(rows_total):
    import torch
    return torch.full((rows_total + 16, 4), np.nan, dtype=torch.float32, device="cuda")


def _check_rows(aloam, orc, sink, begin, count, raws_rows, map_rows, mapped_rows, fulls=None):
    """every mapped row is pointAssociateToMap(map pose of the row, full cloud); others have count 0; begin follows the raw sizes"""
    s = sink.cpu().numpy() if hasattr(sink, "cpu") else sink
    off = 0
    for r, raw in enumerate(raws_rows):
        assert begin[r] == off, r
        if raw is None or not mapped_rows[r]:
            assert count[r] == 0, r
            continue
        full = fulls[r] if fulls is not None else _full(aloam, raw)
        assert count[r] == len(full), r
        assert _bits(s[begin[r]:begin[r] + count[r]]) == _bits(pyclouds.associate_to_map(map_rows[r], full)), r
        off += raw.shape[0]


@pytest.mark.parametrize("skip", [1, 3])
def test_registered_rows_of_the_mapped_stream(aloam, orc, scans, skip):
    raws = [scans("VLP-16", k, n_az=900) for k in range(7)]
    maxn = max(r.shape[0] for r in raws)
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, mapping_skip_frame=skip)
    sink = _sink(sum(r.shape[0] for r in raws))
    c.set_registered_sink(sink)
    # two calls: the rows of each start at offset 0, the scan numbering carries over
    o1, m1 = c.scan_stream_mapped([r.ctypes.data for r in raws[:4]], [r.shape[0] for r in raws[:4]], False)
    b1, n1 = c.registered_rows(4)
    _check_rows(aloam, orc, sink, b1, n1, raws[:4], m1, [j % skip == 0 for j in range(4)])
    o2, m2 = c.scan_stream_mapped([r.ctypes.data for r in raws[4:]], [r.shape[0] for r in raws[4:]], False)
    b2, n2 = c.registered_rows(3)
    _check_rows(aloam, orc, sink, b2, n2, raws[4:], m2, [j % skip == 0 for j in range(4, 7)])
    with pytest.raises(aloam.AloamError) as e:
        c.registered_rows(4)
    assert e.value.code == ERR_INVALID_ARG
    # the same poses as a context that never set a sink
    ref = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, mapping_skip_frame=skip)
    r1 = ref.scan_stream_mapped([r.ctypes.data for r in raws[:4]], [r.shape[0] for r in raws[:4]], False)
    r2 = ref.scan_stream_mapped([r.ctypes.data for r in raws[4:]], [r.shape[0] for r in raws[4:]], False)
    assert np.array_equal(np.concatenate([m1, m2]), np.concatenate([r1[1], r2[1]]))
    assert np.array_equal(np.concatenate([o1, o2]), np.concatenate([r1[0], r2[0]]))
    c.close(); ref.close()


def test_registered_rows_of_a_16_lane_batch_equal_solo_runs(aloam, scans):
    """16 lanes over 4 distinct trajectories, mapping_skip_frame 2: every lane's rows equal its solo run's bytes; device and
    pinned sinks give the same bytes"""
    import torch
    n_scans, B, T = 5, 16, 4
    trajs = [[scans("VLP-16", k + 3 * t, n_az=900) for k in range(n_scans)] for t in range(T)]
    maxn = max(r.shape[0] for t in trajs for r in t)
    lanes = [trajs[b % T] for b in range(B)]
    solo = []
    for t in range(T):
        s = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, mapping_skip_frame=2)
        sk = _sink(sum(r.shape[0] for r in trajs[t]))
        s.set_registered_sink(sk)
        _, mp = s.scan_stream_mapped([r.ctypes.data for r in trajs[t]], [r.shape[0] for r in trajs[t]], False)
        b, n = s.registered_rows(n_scans)
        solo.append((mp, [sk[b[k]:b[k] + n[k]].cpu().numpy() for k in range(n_scans)]))
        s.close()
    total = sum(r.shape[0] for t in lanes for r in t)
    ptrs = np.array([[lanes[b][k].ctypes.data for b in range(B)] for k in range(n_scans)], np.uint64)
    counts = np.array([[lanes[b][k].shape[0] for b in range(B)] for k in range(n_scans)])
    got = []
    for pinned in (False, True):
        c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, max_batch=B, mapping_skip_frame=2)
        sink = torch.zeros((total, 4), dtype=torch.float32).pin_memory() if pinned else _sink(total)
        c.set_registered_sink(sink)
        _, mp = c.scan_stream_mapped_batch(ptrs, counts, False)
        begin, count = c.registered_rows(n_scans * B)
        s = sink.cpu().numpy()
        rows = []
        off = 0
        for k in range(n_scans):
            for b in range(B):
                r = k * B + b
                assert begin[r] == off
                smp, srows = solo[b % T]
                assert np.array_equal(mp[k, b], smp[k])
                assert _bits(s[begin[r]:begin[r] + count[r]]) == _bits(srows[k]), (k, b)
                assert (count[r] > 0) == (k % 2 == 0)
                off += counts[k, b] if k % 2 == 0 else 0
                rows.append(_bits(s[begin[r]:begin[r] + count[r]]))
        got.append(rows)
        c.close()
    assert got[0] == got[1]


def test_registered_rows_of_staggered_lanes_equal_solo_runs(aloam, scans):
    """aloam_scan_stream_lanes: trajectories that start at different steps, one ending early; every row equals the solo run of its
    trajectory, idle rows have count 0"""
    L = aloam
    n_steps, B = 6, 3
    trajs = {0: [scans("VLP-16", k, n_az=900) for k in range(6)], 1: [scans("VLP-16", 10 + k, n_az=900) for k in range(4)],
             2: [scans("VLP-16", 20 + k, n_az=900) for k in range(3)]}
    start = {0: 0, 1: 2, 2: 1}
    maxn = max(r.shape[0] for t in trajs.values() for r in t)
    solo = {}
    for t, tr in trajs.items():
        s = L.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
        sk = _sink(sum(r.shape[0] for r in tr))
        s.set_registered_sink(sk)
        s.scan_stream_mapped([r.ctypes.data for r in tr], [r.shape[0] for r in tr], False)
        b, n = s.registered_rows(len(tr))
        solo[t] = [sk[b[k]:b[k] + n[k]].cpu().numpy() for k in range(len(tr))]
        s.close()
    ops = np.zeros((n_steps, B), np.int32); ptrs = np.zeros((n_steps, B), np.uint64); counts = np.zeros((n_steps, B), np.int64)
    for b in range(B):
        for j, raw in enumerate(trajs[b]):
            k = start[b] + j
            if k < n_steps:
                ops[k, b] = L.LANE_START if j == 0 else L.LANE_SCAN
                ptrs[k, b] = raw.ctypes.data; counts[k, b] = raw.shape[0]
    c = L.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, max_batch=B)
    sink = _sink(int(counts.sum()))
    c.set_registered_sink(sink)
    c.scan_stream_lanes(ptrs, counts, ops, False)
    begin, count = c.registered_rows(n_steps * B)
    s = sink.cpu().numpy()
    off = 0
    for k in range(n_steps):
        for b in range(B):
            r = k * B + b
            assert begin[r] == off
            if ops[k, b] == L.LANE_IDLE:
                assert count[r] == 0
                continue
            assert _bits(s[begin[r]:begin[r] + count[r]]) == _bits(solo[b][k - start[b]]), (k, b)
            off += counts[k, b]
    c.close()


def test_registered_sink_checks_and_a_refused_call_changes_nothing(aloam, scans):
    import torch
    raws = [scans("VLP-16", k, n_az=900) for k in range(6)]
    maxn = max(r.shape[0] for r in raws)
    ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    lib = aloam.lib()
    pageable = torch.zeros((1000, 4), dtype=torch.float32)
    assert lib.aloam_set_registered_sink(c._h, aloam.C.c_void_p(pageable.data_ptr()), 1000) == ERR_INVALID_ARG
    assert lib.aloam_set_registered_sink(c._h, None, -1) == ERR_INVALID_ARG
    with pytest.raises(aloam.AloamError) as e:
        c.registered_rows(0)
    assert e.value.code == ERR_STATE                                       # no mapped stream call yet
    c.scan_stream_mapped(ptrs[:2], counts[:2], False)
    small = _sink(sum(counts[2:4]) - 1 - 16)                               # one point short for scans 2 and 3
    c.set_registered_sink(small)
    with pytest.raises(aloam.AloamError) as e:
        c.scan_stream_mapped(ptrs[2:4], counts[2:4], False)
    assert e.value.code == ERR_CAPACITY and bool(torch.isnan(small).all())
    big = _sink(sum(counts))
    c.set_registered_sink(big)
    _, m = c.scan_stream_mapped(ptrs[2:], counts[2:], False)
    ref = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    ref.scan_stream_mapped(ptrs[:2], counts[:2], False)
    _, mr = ref.scan_stream_mapped(ptrs[2:], counts[2:], False)
    assert np.array_equal(m, mr)
    c.close(); ref.close()


def test_no_sink_issues_what_it_issued_before(aloam, scans):
    """a mapped call with no sink, or after clearing it, launches exactly what a context that never set one launches"""
    raws = [scans("VLP-16", k, n_az=900) for k in range(4)]
    maxn = max(r.shape[0] for r in raws)
    ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
    a = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    b = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    b.set_registered_sink(_sink(sum(counts)))
    b.set_registered_sink(None)
    la, lb = a.launch_count(), b.launch_count()
    oa, ma = a.scan_stream_mapped(ptrs, counts, False)
    ob, mb = b.scan_stream_mapped(ptrs, counts, False)
    assert a.launch_count() - la == b.launch_count() - lb
    assert np.array_equal(ma, mb) and np.array_equal(oa, ob)
    _, cnt = b.registered_rows(4)
    assert not cnt.any()
    a.close(); b.close()


def test_registered_rows_on_an_emulated_rank(aloam, orc, scans):
    """the sharded frame (a context emulating rank 0 of 1 and of 2): every mapped row is its own map pose applied to the full cloud,
    and rank 0 of 1 gives the single-GPU rows"""
    raws = [scans("VLP-16", k, n_az=900) for k in range(4)]
    maxn = max(r.shape[0] for r in raws)
    ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
    fulls = [_full(aloam, r) for r in raws]
    out = {}
    for world in (None, 1, 2):
        c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
        if world:
            c.debug_shard_emulate(0, world)
        sink = _sink(sum(counts))
        c.set_registered_sink(sink)
        _, m = c.scan_stream_mapped(ptrs, counts, False)
        b, n = c.registered_rows(4)
        _check_rows(aloam, orc, sink, b, n, raws, m, [True] * 4, fulls)
        out[world] = (m, sink.cpu().numpy())
        c.close()
    if np.array_equal(out[None][0], out[1][0]):
        assert _bits(out[None][1][:sum(counts)]) == _bits(out[1][1][:sum(counts)])
