"""GPU parity: the device-resident map cube store (cubemap.cu) vs the oracle restatement (oracle/cubemap.cc) of
laserMapping.cpp:309-550,736-801 -- shift, gather, stack filters, insertion, per-cube VoxelGrid, and the whole mapping
loop over a short trajectory."""
import numpy as np
import pytest

from conftest import rot_angle

pytestmark = pytest.mark.gpu

W, H = 21, 21


def test_cube_store_bit_exact_when_the_pose_is_the_odometry_pose(aloam, orc):
    """thin clouds (< 10 corner points in reach) => no optimisation, pose = odometry pose: every cube of the block must
    then equal the oracle's bit for bit along a path that scrolls the ring buffer in all six directions"""
    rng = np.random.default_rng(11)
    c = aloam.Aloam(n_scans=16, max_points=20000, max_map_points=200000, line_res=0.4, plane_res=0.8)
    c.mapper_reset()
    cm = orc.CubeMap()
    ident = np.array([0, 0, 0, 1.0])
    path = [(0, 0, 0), (60, -35, 12), (130, -80, 30), (260, -170, 75), (420, -290, 140), (300, -100, 60), (-90, 40, -30),
            (-400, 380, -160), (-700, 600, -260), (-640, 610, -250), (-300, -200, 100), (200, -420, 200)]   # the last two: the shift towards +j
    for t in path:
        t = np.array(t, float)
        corner = (rng.normal(size=(6, 4)) * [8, 8, 2, 0]).astype(np.float32)
        surf = (rng.normal(size=(300, 4)) * [30, 30, 3, 0]).astype(np.float32)
        pose, info = cm.step(corner, surf, ident, t, 0.4, 0.8)
        q, tt, st = c.mapper_step(corner, surf, ident, t)
        assert np.array_equal(np.concatenate([q, tt]), pose) and st["flags"] & aloam.FLAG_MAP_TOO_THIN
        so, sg = cm.state(), c.mapper_state()
        assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
        assert (sg["total_corner"], sg["total_surf"]) == (so["total_corner"], so["total_surf"])
        for idx in so["valid"]:
            for which in (0, 1):
                assert np.array_equal(c.mapper_cube(which, idx), cm.cube(which, idx)), (t, idx, which)
    c.close()


def test_mapping_loop_over_a_trajectory(aloam, orc, synth, scans):
    """odometry poses from the oracle, map refinement on the device: refined poses within the north-star tolerance of
    the oracle's mapping loop, same optimisation decisions, submaps of (nearly) the same size"""
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    c = aloam.Aloam(n_scans=16, max_points=40000, max_map_points=400000)      # VLP-16 launch file: 0.2 / 0.4
    c.mapper_reset()
    cm = orc.CubeMap()
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3)
    qw = np.array([0, 0, 0, 1.0]); tw = np.zeros(3)
    for k in range(6):
        f = orc.Features(scans("VLP-16", k, n_az=900), ns, mr)
        if k > 0:
            q, t, _ = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
        od.set_last(f.less_sharp, f.less_flat)
        pose, info = cm.step(f.less_sharp, f.less_flat, qw, tw, 0.2, 0.4)
        gq, gt, st = c.mapper_step(f.less_sharp, f.less_flat, qw, tw)
        assert bool(info["optimised"]) == (not (st["flags"] & aloam.FLAG_MAP_TOO_THIN))
        assert np.abs(gt - pose[4:]).max() < 1e-4 and rot_angle(gq, pose[:4]) < 1e-4, (k, gt - pose[4:])
        so, sg = cm.state(), c.mapper_state()
        assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
        # the poses agree to ~1e-8, so a transformed point can land on the other side of a voxel boundary: sizes may
        # differ by a handful of points, not more
        assert abs(sg["total_corner"] - so["total_corner"]) <= 5 and abs(sg["total_surf"] - so["total_surf"]) <= 20
        # cube CONTENTS after the optimisation: same voxels in the same order, centroids equal to float rounding of a 1e-8 pose
        # difference (a cube whose size differs had a point cross a voxel / cube boundary and is skipped)
        same = differ = 0
        for idx in so["valid"]:
            for which in (0, 1):
                a, b = c.mapper_cube(which, idx), cm.cube(which, idx)
                if a.shape != b.shape:
                    differ += 1
                    continue
                same += 1
                if len(a):
                    assert np.abs(a[:, :3] - b[:, :3]).max() < 2e-5 and np.abs(a[:, 3] - b[:, 3]).max() < 1e-4, (k, idx, which)
        assert same >= 1 and differ <= 4
    c.close()


def test_stream_with_mapping_equals_per_scan_calls_and_oracle(aloam, orc, synth, scans):
    """aloam_scan_stream_mapped (odometry -> scan-to-map hand-off on the device, SURVEY 8 f-2) == aloam_scan_to_pose +
    aloam_mapper_step per scan, and both follow the oracle's ascanRegistration | alaserOdometry | alaserMapping chain"""
    import torch
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    raws = [scans("VLP-16", k, n_az=900) for k in range(6)]
    maxn = max(r.shape[0] for r in raws)
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    # split in two calls: the mapper state carries over
    o1, m1 = c.scan_stream_mapped([d.data_ptr() for d in dev[:4]], [r.shape[0] for r in raws[:4]], True)
    o2, m2 = c.scan_stream_mapped([r.ctypes.data for r in raws[4:]], [r.shape[0] for r in raws[4:]], False)
    odom, mapped = np.concatenate([o1, o2]), np.concatenate([m1, m2])
    c.close()
    # per-scan calls
    c2 = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    c2.mapper_reset()
    cm = orc.CubeMap()
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    for k, raw in enumerate(raws):
        gq, gt, _ = c2.scan_to_pose(raw)
        assert np.array_equal(np.concatenate([gq, gt]), odom[k])
        f = c2.extract_features(raw)
        mq, mt, _ = c2.mapper_step(f["less_sharp"], f["less_flat"], gq, gt)
        assert np.array_equal(np.concatenate([mq, mt]), mapped[k]), k
        fo = orc.Features(raw, ns, mr)
        if k > 0:
            q, t, _ = od.register(fo.sharp, fo.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
        od.set_last(fo.less_sharp, fo.less_flat)
        pose, info = cm.step(fo.less_sharp, fo.less_flat, qw, tw, 0.2, 0.4)
        assert np.abs(mapped[k, 4:] - pose[4:]).max() < 1e-4 and rot_angle(mapped[k, :4], pose[:4]) < 1e-4
    c2.close()


def test_slab_overflow_is_flagged_not_fatal(aloam):
    """a cube that receives more points than a slab holds keeps running: the overflow is dropped and flagged (the
    reference's cubes grow without bound between re-filters; ADVICE r1)"""
    rng = np.random.default_rng(3)
    c = aloam.Aloam(n_scans=16, max_points=3000, max_map_points=20000, line_res=0.01, plane_res=0.01)   # slab capacity = 3000
    c.mapper_reset()
    ident = np.array([0, 0, 0, 1.0])
    flags = 0
    for k in range(3):
        corner = (rng.uniform(-10, 10, size=(5, 4))).astype(np.float32)
        surf = (rng.uniform(-20, 20, size=(2500, 4)) * [1, 1, 0.2, 0]).astype(np.float32)     # all inside the centre cube
        q, t, st = c.mapper_step(corner, surf, ident, np.zeros(3))
        flags |= st["flags"]
    assert flags & aloam.FLAG_CUBE_OVERFLOW
    assert c.mapper_state()["total_surf"] == 3000
    c.close()


# ---- bit-exact frames at the store's size limits.  One cloud type is left empty, so the submap is too thin and the pose
# is the odometry pose on both sides: every frame must then agree bit for bit, rotation arithmetic included.
D = 11
INT_MAX = 2**31 - 1


def _quat(axis, angle):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return np.concatenate([a * np.sin(angle / 2), [np.cos(angle / 2)]])


def _index_range(cloud, leaf):
    f = np.float32
    inv = f(1) / f(leaf)
    mn, mx = cloud[:, :3].min(0), cloud[:, :3].max(0)
    d = [int((f(mx[a]) - f(mn[a])) * inv) + 1 for a in range(3)]
    div = [int(np.floor(f(mx[a]) * inv)) - int(np.floor(f(mn[a]) * inv)) + 1 for a in range(3)]
    return d[0] * d[1] * d[2], div[0] * div[1] * div[2]


def _box(rng, n, lo, hi):
    out = np.zeros((n, 4), np.float32)
    out[:, :3] = rng.uniform(lo, hi, size=(n, 3))
    out[:, 3] = rng.uniform(0, 16, n)
    return out


def _dense(rng, n):
    """body-frame cloud: most points within +-100 m, a sixth out to +-150 m (cubes outside the 5 x 5 x 3 block, which are
    never re-filtered and so keep the raw insertion order)"""
    near = _box(rng, n - n // 6, [-100, -100, -20], [100, 100, 20])
    far = _box(rng, n // 6, [-150, -150, -60], [150, 150, 60])
    return np.concatenate([near, far])[rng.permutation(n)]


def _same_store(c, cm, exact_totals=True):
    so, sg = cm.state(), c.mapper_state()
    assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
    assert np.array_equal(sg["q_wmap_wodom"], so["q_wmap_wodom"]) and np.array_equal(sg["t_wmap_wodom"], so["t_wmap_wodom"])
    if exact_totals:
        assert (sg["total_corner"], sg["total_surf"]) == (so["total_corner"], so["total_surf"])
    held = 0
    for idx in range(W * H * D):
        for which in (0, 1):
            ref = cm.cube(which, idx)
            if len(ref):
                held += 1
                assert np.array_equal(c.mapper_cube(which, idx), ref), (idx, which)
    return held


@pytest.mark.parametrize("leaves", [(0.2, 0.4), (0.4, 0.8), (0.1, 0.2)])
@pytest.mark.parametrize("dense", ["surf", "corner"])
def test_dense_rotated_frames_bit_exact(aloam, orc, leaves, dense):
    """~60 k points per frame of one type under non-identity odometry rotations, along a path that scrolls the ring buffer
    and comes back (freed slabs are reused): pose, map-to-odometry transform, centre, valid list, totals and EVERY cube
    the oracle holds are bit-identical.  (0.1, 0.2) gives 27 index bits and 5 segment windows in the re-filter."""
    rng = np.random.default_rng(int(leaves[0] * 100) + (7 if dense == "surf" else 0))
    c = aloam.Aloam(n_scans=16, max_points=65536, max_map_points=1000000, line_res=leaves[0], plane_res=leaves[1])
    c.mapper_reset()
    cm = orc.CubeMap()
    path = [(0, 0, 0), (180, -120, 40), (430, -300, 140), (260, -100, 60), (-150, 90, -40), (-420, 330, -150), (-60, 20, -10), (5, -3, 2)]
    empty = np.zeros((0, 4), np.float32)
    held = 0
    for k, t in enumerate(path):
        q = _quat([1.0, -0.5 + 0.2 * k, 0.3], 0.35 + 0.4 * k)
        cloud = _dense(rng, 60000)
        corner, surf = (empty, cloud) if dense == "surf" else (cloud, empty)
        pose, info = cm.step(corner, surf, q, np.array(t, float), *leaves)
        gq, gt, st = c.mapper_step(corner, surf, q, np.array(t, float))
        assert np.array_equal(np.concatenate([gq, gt]), pose), k
        assert st["flags"] & aloam.FLAG_MAP_TOO_THIN and not st["flags"] & aloam.FLAG_CUBE_OVERFLOW, (k, st["flags"])
        held = max(held, _same_store(c, cm))
    assert held > 40
    c.close()


def test_refilter_beyond_the_submap_capacity(aloam, orc):
    """max_points 3000, max_map_points 5000: the valid cubes hold up to 18 000 points, more than 2 x max(max_map_points,
    max_points) = 10 000 (the sort buffers were once sized by that).  The re-filter stays exact, and a frame whose submap
    gather is truncated at max_map_points raises FLAG_CUBE_OVERFLOW -- that frame only"""
    rng = np.random.default_rng(41)
    c = aloam.Aloam(n_scans=16, max_points=3000, max_map_points=5000, line_res=0.05, plane_res=0.05)
    c.mapper_reset()
    cm = orc.CubeMap()
    empty = np.zeros((0, 4), np.float32)
    flagged = []
    for k in range(7):
        q = _quat([0.2, 0.1, 1.0], 0.1 * k)
        t = np.array([3.0 * k, -2.0 * k, 0.5 * k])
        surf = _box(rng, 3000, [-100, -100, -5], [100, 100, 5])
        pose, info = cm.step(empty, surf, q, t, 0.05, 0.05)
        gq, gt, st = c.mapper_step(empty, surf, q, t)
        assert np.array_equal(np.concatenate([gq, gt]), pose), k
        truncated = info["surf_from_map"] > 5000
        assert bool(st["flags"] & aloam.FLAG_CUBE_OVERFLOW) == truncated, (k, info, st["flags"])
        flagged.append(truncated)
        _same_store(c, cm)
        so = cm.state()
        assert max(len(cm.cube(1, i)) for i in so["valid"]) <= 3000        # no slab overflow: only the gather is short
    assert cm.state()["total_surf"] > 10000 and flagged[0] is False and any(flagged)
    c.close()


def test_overflow_flags_are_per_frame(aloam, orc):
    """slab overflow: the flag is set on the frame whose insertion overflows, clear on a later frame that does not; the
    overflowing cube (outside the valid block, never re-filtered) holds the oracle's first `cap` points in order"""
    rng = np.random.default_rng(43)
    c = aloam.Aloam(n_scans=16, max_points=3000, max_map_points=20000, line_res=0.05, plane_res=0.05)   # slab capacity 3000
    c.mapper_reset()
    cm = orc.CubeMap()
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    far = 14 + W * 10 + W * H * 5                                          # cube x in [175, 225): outside i = 8..12
    frames = [_box(rng, 2500, [180, -20, -20], [220, 20, 20]), _box(rng, 2500, [180, -20, -20], [220, 20, 20]),
              _box(rng, 500, [-20, -20, -5], [20, 20, 5])]
    for k, surf in enumerate(frames):
        pose, info = cm.step(empty, surf, ident, np.zeros(3), 0.05, 0.05)
        q, t, st = c.mapper_step(empty, surf, ident, np.zeros(3))
        assert np.array_equal(np.concatenate([q, t]), pose)
        assert bool(st["flags"] & aloam.FLAG_CUBE_OVERFLOW) == (k == 1), (k, st["flags"])
        assert far not in cm.state()["valid"]
        ref = cm.cube(1, far)
        assert np.array_equal(c.mapper_cube(1, far), ref[:3000])
    assert len(cm.cube(1, far)) == 5000 and c.mapper_state()["total_surf"] == cm.state()["total_surf"] - 2000
    c.close()


def test_pool_exhaustion_is_flagged(aloam, orc):
    """one frame with points in 1323 cubes: 1024 slabs are handed out, the rest dropped and flagged; every stored cube
    equals the oracle's"""
    rng = np.random.default_rng(47)
    c = aloam.Aloam(n_scans=16, max_points=3000, max_map_points=20000)
    c.mapper_reset()
    cm = orc.CubeMap()
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    ii, jj, kk = np.meshgrid(np.arange(W), np.arange(H), np.arange(3), indexing="ij")
    surf = np.zeros((ii.size, 4), np.float32)
    surf[:, 0] = (ii.ravel() - 10) * 50.0 + rng.uniform(-10, 10, ii.size)
    surf[:, 1] = (jj.ravel() - 10) * 50.0 + rng.uniform(-10, 10, ii.size)
    surf[:, 2] = (kk.ravel() - 5) * 50.0 + rng.uniform(-10, 10, ii.size)
    surf[:, 3] = rng.uniform(0, 16, ii.size)
    surf = surf[rng.permutation(len(surf))]
    pose, info = cm.step(empty, surf, ident, np.zeros(3), 0.2, 0.4)
    q, t, st = c.mapper_step(empty, surf, ident, np.zeros(3))
    assert np.array_equal(np.concatenate([q, t]), pose)
    assert st["flags"] & aloam.FLAG_CUBE_OVERFLOW
    assert cm.state()["total_surf"] == 1323 and c.mapper_state()["total_surf"] == 1024
    stored = 0
    for idx in range(W * H * D):
        ref = cm.cube(1, idx)
        if len(ref):
            got = c.mapper_cube(1, idx)
            if len(got):
                stored += 1
                assert np.array_equal(got, ref), idx
    assert stored == 1024
    c.close()


def _overflow_box(rng, lo, n=2000):
    """a 25.79 m box at leaf 0.02 off the voxel lattice: dxyz product 1290^3 <= INT_MAX (PCL filters it), but 1291^3 > 2^31
    cells do not fit the 31 index bits of the sort key"""
    lo = np.float32(lo)
    box = np.zeros((n, 4), np.float32)
    box[:, :3] = rng.uniform(0, 25.79, size=(n, 3)) + lo
    box[0, :3] = lo
    box[1, :3] = np.float32(lo + np.float32(25.79))
    box[:, 3] = rng.uniform(0, 16, n)
    dprod, cells = _index_range(box, 0.02)
    assert dprod <= INT_MAX and cells > 2**31
    return box


def test_key_overflow_fails_that_frame_only(aloam):
    """a cube whose index range needs more than 31 key bits: that frame returns ALOAM_ERR_CAPACITY, the next one (the cube
    no longer in the valid block) returns 0"""
    rng = np.random.default_rng(53)
    c = aloam.Aloam(n_scans=16, max_points=3000, max_map_points=20000, line_res=0.02, plane_res=0.02)
    c.mapper_reset()
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    with pytest.raises(aloam.AloamError) as e:
        c.mapper_step(empty, _overflow_box(rng, -12.887), ident, np.zeros(3))
    assert e.value.code == -4
    q, t, st = c.mapper_step(empty, _box(rng, 500, [-5, -5, -2], [5, 5, 2]), ident, np.array([150.0, 0, 0]))
    assert 10 + W * 10 + W * H * 5 not in c.mapper_state()["valid"]
    assert not st["flags"] & aloam.FLAG_CUBE_OVERFLOW
    c.close()


def test_stream_with_mapping_reports_key_overflow(aloam, scans):
    """aloam_scan_stream_mapped returns ALOAM_ERR_CAPACITY when a frame's re-filter meets a cube beyond the key width, as
    aloam_mapper_step does; the same scans without that cube return normally"""
    rng = np.random.default_rng(59)
    raws = [scans("VLP-16", k, n_az=900) for k in range(3)]
    maxn = max(r.shape[0] for r in raws)
    box = _overflow_box(rng, (87.113, 87.113, 37.113))       # cube (12, 12, 6): in the valid block of the first scans
    box_cube = 12 + W * 12 + W * H * 6
    ident, empty = np.array([0, 0, 0, 1.0]), np.zeros((0, 4), np.float32)
    for inject in (False, True):
        c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000, line_res=0.02, plane_res=0.02)
        c.mapper_reset()
        if inject:
            with pytest.raises(aloam.AloamError) as e:
                c.mapper_step(empty, box, ident, np.zeros(3))
            assert e.value.code == -4
        ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
        if inject:
            with pytest.raises(aloam.AloamError) as e:
                c.scan_stream_mapped(ptrs, counts, False)
            assert e.value.code == -4
            assert box_cube in c.mapper_state()["valid"]
            assert np.array_equal(c.mapper_cube(1, box_cube), box)   # no scan point reached it: the cube alone overflows
        else:
            c.scan_stream_mapped(ptrs, counts, False)
        c.close()
