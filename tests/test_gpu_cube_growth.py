"""GPU: cube growth (aloam_set_cube_growth).  With growth on a cube whose slab fills moves to a larger aligned run of slabs of the
same pool, up to ALOAM_MAX_CUBE_POINTS points, so dense trajectories that overflow one slab follow the oracle mapper (which has no
limit) frame after frame; with growth off, and on scenes where no cube passes a slab, nothing changes."""
import numpy as np
import pytest

import lane_refs as R
from conftest import rot_angle

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY = -1, -4
IDLE, SCAN, START = 0, 1, 2
IDENT_Q = np.array([0.0, 0.0, 0.0, 1.0])
EMPTY = np.zeros((0, 4), np.float32)


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, e.value.code


def _near(mq, mt, pose, what):
    assert np.abs(mt - pose[4:]).max() < R.BAR and rot_angle(mq, pose[:4]) < R.BAR, (what, mt - pose[4:])


def _mapping_loop(aloam, orc, ctx, raws, leaves, every_cube=False):
    """scan_to_pose + extract_features + mapper_step on ctx, the oracle CubeMap fed the same clouds and odometry poses: every frame
    within the bar of the oracle, centre and valid list equal, every valid cube byte for byte.  Returns (map poses, the largest
    corner cube seen)"""
    cm = orc.CubeMap()
    poses, biggest = [], 0
    for k, raw in enumerate(raws):
        gq, gt, _ = ctx.scan_to_pose(raw)
        f = ctx.extract_features(raw)
        mq, mt, st = ctx.mapper_step(f["less_sharp"], f["less_flat"], gq, gt)
        assert not st["flags"] & aloam.FLAG_CUBE_OVERFLOW, k
        pose, _ = cm.step(f["less_sharp"], f["less_flat"], gq, gt, *leaves)
        _near(mq, mt, pose, k)
        poses.append(np.concatenate([mq, mt]))
        so, sg = cm.state(), ctx.mapper_state()
        assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"], k
        for idx in so["valid"]:
            a = ctx.mapper_cube(0, idx)
            biggest = max(biggest, len(a))
            assert a.tobytes() == cm.cube(0, idx).tobytes(), (k, 0, idx)
            assert ctx.mapper_cube(1, idx).tobytes() == cm.cube(1, idx).tobytes(), (k, 1, idx)
    if every_cube:
        for idx in range(4851):
            for w in (0, 1):
                assert ctx.mapper_cube(w, idx).tobytes() == cm.cube(w, idx).tobytes(), (w, idx)
    return np.array(poses), biggest


# ------------------------------------------------------------------------------------------------ dense trajectories against the oracle
def test_vlp16_default_leaves(aloam, orc, synth):
    """the 64-scan VLP-16 trajectory of test_gpu_long_streams.py at the default 0.2 / 0.4 m leaves with growth on: the stream equals
    scan_to_pose + mapper_step bit for bit, no row overflows, a corner cube ends above one slab (16384 points), every map pose is
    within 1e-4 of the oracle and every cube of the final store equals the oracle's byte for byte"""
    n = 64
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    kw = dict(n_scans=16, max_points=R.maxn([scans]) + 1024, max_map_points=400000, max_ring_points=4096)
    c = aloam.Aloam(**kw)
    c.set_cube_growth(1)
    c.set_map_rows(True)
    odom, mapped = c.scan_stream_mapped([d.data_ptr() for d in dev], [s.shape[0] for s in scans], True)
    rows = c.map_rows(n)
    assert not (rows["flags"] & aloam.FLAG_CUBE_OVERFLOW).any() and not rows["err"].any()
    c.close()
    c = aloam.Aloam(**kw)
    c.set_cube_growth(1)
    c.mapper_reset()
    poses, biggest = _mapping_loop(aloam, orc, c, scans, (0.2, 0.4), every_cube=True)
    c.close()
    assert np.array_equal(poses, mapped)
    assert biggest > 16384, biggest
    _, m = R.oracle(orc, synth, scans, ("VLP-16", 0, 900), True)
    R.assert_near(mapped, m, "map poses over 64 scans")


def test_os64_every_frame(aloam, orc, synth):
    """the OS64 field-mode trajectory of test_gpu_ring_field.py, 20 frames with growth on: every frame against the oracle mapper,
    none skipped for overflow"""
    frames = 20
    ns = len(synth.RING_SENSORS["OS64"][0])
    raws = [synth.scan_rings("OS64", k) for k in range(frames)]
    c = aloam.Aloam(n_scans=ns, max_points=max(len(r) for r in raws) + 1024, ring_source=aloam.RING_FIELD, minimum_range=0.3,
                    line_res=0.2, plane_res=0.4, max_map_points=400000)
    c.set_cube_growth(1)
    c.mapper_reset()
    _, biggest = _mapping_loop(aloam, orc, c, raws, (0.2, 0.4))
    c.close()
    assert biggest > 16384, biggest


# ------------------------------------------------------------------------------------------------ growth off == on without growth
def test_off_and_on_agree_without_growth(aloam, synth):
    """a trajectory on which no cube passes a slab: the VLP-16 trajectory of test_gpu_long_streams.py at its 0.5 / 1.0 m leaves,
    whose largest cube stays below 12 000 points (a known non-growing scene, in place of a batched HDL-32 one).  Lane 0 started
    before set_cube_growth(1), lane 1 after, in one context -- the same map poses, rows, export and snapshot bytes apart from
    header byte 220"""
    n = 16
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    c = aloam.Aloam(n_scans=16, max_points=R.maxn([scans]) + 1024, max_map_points=400000, max_batch=2, line_res=0.5, plane_res=1.0)
    c.set_map_rows(True)
    ptrs = np.array([[d.data_ptr(), d.data_ptr()] for d in dev], np.uint64)
    counts = np.array([[s.shape[0]] * 2 for s in scans])
    out = []
    for lane in (0, 1):
        if lane == 1:
            c.set_cube_growth(1)
        ops = np.full((n, 2), IDLE, np.int32)
        ops[:, lane] = SCAN
        ops[0, lane] = START
        _, m = c.scan_stream_lanes(ptrs, counts, ops, True)
        rows = c.map_rows(2 * n)
        blob = c.lane_save(lane)
        out.append((m[:, lane], {k: v.reshape(n, 2, *v.shape[1:])[:, lane] for k, v in rows.items()}, c.mapper_export(aloam.EXPORT_MAP, lane), blob))
    c.close()
    (m0, r0, e0, b0), (m1, r1, e1, b1) = out
    assert np.array_equal(m0, m1)
    for k in r0:
        assert np.array_equal(r0[k], r1[k]), k
    assert e0.tobytes() == e1.tobytes()
    g0, g1 = (np.frombuffer(b[220:224].tobytes(), np.int32)[0] for b in (b0, b1))
    assert (g0, g1) == (0, 1)
    assert b0[:220].tobytes() == b1[:220].tobytes() and b0[224:].tobytes() == b1[224:].tobytes()


# ------------------------------------------------------------------------------------------------ lanes and snapshots
def test_sixteen_lanes_equal_solo(aloam, synth):
    """16 lanes of 4 VLP-16 trajectories at the default leaves, 32 steps with growth on: every lane equals its solo run bit for bit
    (map poses and store), and the lanes grow cubes past one slab"""
    B, n = 16, 32
    trajs = [R.traj(synth, t, n) for t in range(4)]
    dev = [R.to_device(tr) for tr in trajs]
    maxpts = R.maxn(trajs) + 1024
    ctx = aloam.Aloam(n_scans=16, max_points=maxpts, max_map_points=400000, max_batch=B)
    ctx.set_cube_growth(1)
    ptrs = np.array([[dev[b % 4][k].data_ptr() for b in range(B)] for k in range(n)], np.uint64)
    counts = np.array([[trajs[b % 4][k].shape[0] for b in range(B)] for k in range(n)])
    _, mapped = ctx.scan_stream_mapped_batch(ptrs, counts, True)
    stores = [R.snapshot(ctx, b) for b in range(B)]
    biggest = max(len(ctx.mapper_cube(0, i, b)) for b in range(4) for i in stores[b][0]["valid"])
    ctx.close()
    assert biggest > 16384, biggest
    for t in range(4):
        c = aloam.Aloam(n_scans=16, max_points=maxpts, max_map_points=400000)
        c.set_cube_growth(1)
        _, m = c.scan_stream_mapped([d.data_ptr() for d in dev[t]], counts[:, t], True)
        solo = R.snapshot(c, 0)
        c.close()
        for b in range(t, B, 4):
            assert np.array_equal(mapped[:, b], m), "lane %d" % b
            R.same_store(stores[b], solo, "store of lane %d" % b)


def test_snapshot_resume_with_grown_cubes(aloam, synth):
    """a growth-on lane saved mid-trajectory with grown cubes, restored into another lane and into another context whose growth is
    off, and continued: bit-identical to the uninterrupted run (the restored lane keeps the snapshot's growth)"""
    n, cut = 40, 24
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    kw = dict(n_scans=16, max_points=R.maxn([scans]) + 1024, max_map_points=400000, max_batch=2)
    ptrs = np.array([[d.data_ptr()] * 2 for d in dev], np.uint64)
    counts = np.array([[s.shape[0]] * 2 for s in scans])

    def ops(rows, lane, first):
        o = np.full((rows, 2), IDLE, np.int32)
        o[:, lane] = SCAN
        o[0, lane] = first
        return o

    c = aloam.Aloam(**kw)
    c.set_cube_growth(1)
    _, whole = c.scan_stream_lanes(ptrs, counts, ops(n, 0, START), True)
    ref = c.mapper_export(aloam.EXPORT_MAP, 0)
    _, a = c.scan_stream_lanes(ptrs[:cut], counts[:cut], ops(cut, 0, START), True)
    blob = c.lane_save(0)
    assert np.frombuffer(blob[220:224].tobytes(), np.int32)[0] == 1
    c.lane_restore(1, blob)
    _, b = c.scan_stream_lanes(ptrs[cut:], counts[cut:], ops(n - cut, 1, SCAN), True)
    assert np.array_equal(a[:, 0], whole[:cut, 0]) and np.array_equal(b[:, 1], whole[cut:, 0])
    assert c.mapper_export(aloam.EXPORT_MAP, 1).tobytes() == ref.tobytes()
    big = max(len(c.mapper_cube(0, i, 1)) for i in c.mapper_state(1)["valid"])
    c.close()
    assert big > 16384, big
    d = aloam.Aloam(**kw)   # growth off
    d.lane_restore(0, blob)
    _, e = d.scan_stream_lanes(ptrs[cut:], counts[cut:], ops(n - cut, 0, SCAN), True)
    assert np.array_equal(e[:, 0], whole[cut:, 0])
    assert d.mapper_export(aloam.EXPORT_MAP, 0).tobytes() == ref.tobytes()
    assert np.frombuffer(d.lane_save(0)[220:224].tobytes(), np.int32)[0] == 1
    d.close()


# ------------------------------------------------------------------------------------------------ boundaries on crafted scenes
def _fill(rng, n, lo, hi, x_lo=None, x_hi=None):
    """n points uniform in [lo, hi)^3 (x in [x_lo, x_hi) when given), random intensity"""
    p = np.zeros((n, 4), np.float32)
    p[:, :3] = rng.uniform(lo, hi, (n, 3))
    if x_lo is not None:
        p[:, 0] = rng.uniform(x_lo, x_hi, n)
    p[:, 3] = rng.uniform(0, 16, n)
    return p


def test_counts_at_every_run_boundary(aloam, orc):
    """surf points into the centre cube, max_points = 2048 (slab capacity 2048, runs up to 128 slabs = ALOAM_MAX_CUBE_POINTS), leaves
    so fine that every filter passes its points through: the cube equals the oracle's at cap, cap + 1, 2 cap, 2 cap + 1 and the
    ceiling with no flag; one point more is dropped (the last one in stack order) and flags the frame"""
    cap, ceiling = 2048, 262144
    rng = np.random.default_rng(5)
    c = aloam.Aloam(n_scans=16, max_points=cap, max_map_points=400000, line_res=1e-4, plane_res=1e-4)
    c.set_cube_growth(1)
    c.mapper_reset()
    cm = orc.CubeMap()
    idx = 10 + 21 * 10 + 441 * 5
    sizes = [cap, 1, cap - 1, 1] + [cap] * ((ceiling - 2 * cap - 1) // cap) + [(ceiling - 2 * cap - 1) % cap, 1]
    total, checks = 0, {cap, cap + 1, 2 * cap, 2 * cap + 1, ceiling}
    for j, m in enumerate(sizes):
        if m == 0:
            continue
        surf = _fill(rng, m, -20.0, 20.0)
        cm.step(EMPTY, surf, IDENT_Q, np.zeros(3), 1e-4, 1e-4)
        _, _, st = c.mapper_step(EMPTY, surf, IDENT_Q, np.zeros(3))
        total += m
        if total <= ceiling:
            assert not st["flags"] & aloam.FLAG_CUBE_OVERFLOW, (j, total)
            if total in checks:
                assert c.mapper_cube(1, idx).tobytes() == cm.cube(1, idx).tobytes(), total
        else:
            assert st["flags"] & aloam.FLAG_CUBE_OVERFLOW
            got, want = c.mapper_cube(1, idx), cm.cube(1, idx)
            assert len(got) == ceiling and got.tobytes() == want[:ceiling].tobytes()
    assert total == ceiling + 1
    c.close()


def test_refilter_budget(aloam, orc):
    """max_points = 1024: the re-filter sorts at most 75 x 2048 = 153600 points.  Cube A (centre) grows to 100352 points, then cube
    B (one cube up in i) takes points: the frames stay unflagged until A + B passes the budget, then B is left unfiltered and the
    frame raises ALOAM_FLAG_CUBE_OVERFLOW; with pass-through leaves the cubes still equal the oracle's"""
    cap, budget = 1024, 75 * 2048
    rng = np.random.default_rng(9)
    c = aloam.Aloam(n_scans=16, max_points=cap, max_map_points=400000, line_res=1e-4, plane_res=1e-4)
    c.set_cube_growth(1)
    c.mapper_reset()
    cm = orc.CubeMap()
    a, b = 10 + 21 * 10 + 441 * 5, 11 + 21 * 10 + 441 * 5
    na = nb = 0
    while na < 98 * cap:
        surf = _fill(rng, cap, -20.0, 20.0)
        cm.step(EMPTY, surf, IDENT_Q, np.zeros(3), 1e-4, 1e-4)
        _, _, st = c.mapper_step(EMPTY, surf, IDENT_Q, np.zeros(3))
        assert not st["flags"] & aloam.FLAG_CUBE_OVERFLOW
        na += cap
    flagged = 0
    while na + nb <= budget + cap:
        surf = _fill(rng, cap, -20.0, 20.0, 30.0, 70.0)
        cm.step(EMPTY, surf, IDENT_Q, np.zeros(3), 1e-4, 1e-4)
        _, _, st = c.mapper_step(EMPTY, surf, IDENT_Q, np.zeros(3))
        nb += cap
        over = bool(st["flags"] & aloam.FLAG_CUBE_OVERFLOW)
        assert over == (na + nb > budget), (na, nb)
        flagged += over
    assert flagged >= 1
    assert c.mapper_cube(1, a).tobytes() == cm.cube(1, a).tobytes() and c.mapper_cube(1, b).tobytes() == cm.cube(1, b).tobytes()
    c.close()


# ------------------------------------------------------------------------------------------------ prior maps
def test_map_on_prior_dense_cubes(aloam):
    """a built prior map with one corner cube of 16385 points, then one of 65537 (the build refuses it while growth is off):
    lane_map_on_prior seeds them with growth on and refuses them with growth off; the seeded lane's snapshot holds the cube"""
    rng = np.random.default_rng(3)
    for n in (16385, 65537):
        corner = _fill(rng, n, -20.0, 20.0)
        surf = _fill(rng, 200, -20.0, 20.0)
        c = aloam.Aloam(n_scans=16, max_points=70000, max_map_points=400000, line_res=1e-4, plane_res=1e-4)
        if n > 65536:
            _expect(aloam, ERR_CAPACITY, lambda: c.prior_map_build(corner, surf))
        c.set_cube_growth(1)
        c.prior_map_build(corner, surf)
        assert c.mapper_export_size(aloam.EXPORT_MAP, aloam.PRIOR_MAP) == n + 200
        c.lane_map_on_prior(0, IDENT_Q, np.zeros(3))
        c.set_cube_growth(0)
        _expect(aloam, ERR_CAPACITY, lambda: c.lane_map_on_prior(0, IDENT_Q, np.zeros(3)))
        _expect(aloam, ERR_INVALID_ARG, lambda: c.set_cube_growth(2))
        c.set_cube_growth(1)
        c.lane_map_on_prior(0, IDENT_Q, np.zeros(3))
        prior = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP)
        raw = _fill(rng, 3000, -20.0, 20.0)   # a scan with few features: the START's frame sees the seeded store
        import torch
        d = torch.from_numpy(raw).cuda()
        c.scan_stream_lanes(np.array([[d.data_ptr()]], np.uint64), np.array([[len(raw)]]), np.array([[START]], np.int32), True)
        blob = c.lane_save(0)
        assert np.frombuffer(blob[220:224].tobytes(), np.int32)[0] == 1
        # the seeded store holds the prior map's cube in its order (pass-through leaves); the START frame may only append to it
        got = c.mapper_cube(0, 10 + 21 * 10 + 441 * 5)
        assert len(got) >= n and got[:n].tobytes() == prior[:n].tobytes()
        c.close()
