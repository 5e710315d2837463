"""GPU: the mapper's ring buffer at its decisions (cubemap.cu cube_coord, mapper_begin_body, rotate_line, cube_ids_body).
aloam_mapper_step on the crafted paths of tests/cube_edge_cases.py -- poses on every decision of the cube rule, points on every
face under rotations, long jumps along each axis and the diagonal -- against the host model, the oracle's CubeMap and the
reference's compiled laserMapping.cpp, bit for bit (thin frames: the pose is the hand-off pose); the slab pool after full and
partial wraps; stores relabelled by whole cubes inside the mapped lane streams, whose first or later frames must shift, against
the unrelabelled run; a shifted store moved to another context; and restores of out-of-range snapshots refused."""
import numpy as np
import pytest

import cube_edge_cases as E

pytestmark = pytest.mark.gpu

EMPTY = np.zeros((0, 4), np.float32)


def _frames(name):
    return E.decision_paths().get(name) or E.jump_paths()[name]


def _ctx(aloam, **kw):
    cfg = dict(n_scans=16, max_points=20000, max_map_points=200000, line_res=E.LEAVES[0], plane_res=E.LEAVES[1])
    cfg.update(kw)
    return aloam.Aloam(**cfg)


def _ref(orc, tag):
    """the reference's mapping node, or None where oracle/_ref is not usable (only its comparisons are left out then)"""
    import refsource
    try:
        return refsource.RefMapping(refsource.private_copy("libref_mapping.so", tag), *E.LEAVES, orc.SORT_CANONICAL)
    except (OSError, AssertionError, pytest.skip.Exception):
        return None


def _run_path(aloam, orc, c, frames, ref=None):
    """the frames through aloam_mapper_step on c, the host model, the oracle and (if given) the reference, compared after every
    frame: pose = the model's, centre, valid list and T = the oracle's and the reference's, and every cube the model holds = the
    oracle's bit for bit, with the same totals (no point stored anywhere else).  Returns the model"""
    c.mapper_reset()
    m, cm = E.Model(), orc.CubeMap()
    for j, (q, t, surf) in enumerate(frames):
        pose, st = m.frame(EMPTY, surf, q, t)
        cm.step(EMPTY, surf, q, t, *E.LEAVES)
        gq, gt, gs = c.mapper_step(EMPTY, surf, q, t)
        assert np.array_equal(np.concatenate([gq, gt]), pose), j
        assert gs["flags"] & aloam.FLAG_MAP_TOO_THIN and not gs["flags"] & aloam.FLAG_CUBE_OVERFLOW, (j, gs["flags"])
        so, sg = cm.state(), c.mapper_state()
        assert sg["centre"] == so["centre"] == st["centre"] and sg["valid"] == so["valid"] == st["valid"], j
        assert np.array_equal(sg["q_wmap_wodom"], so["q_wmap_wodom"]) and np.array_equal(sg["t_wmap_wodom"], so["t_wmap_wodom"]), j
        assert (sg["total_corner"], sg["total_surf"]) == (so["total_corner"], so["total_surf"]), j
        if ref is not None:
            r = ref.process(EMPTY, surf, surf, q, t, stamp=0.1 * (j + 1))
            assert np.array_equal(r["pose"], pose) and sg["centre"] == r["centre"], j
            assert np.array_equal(sg["q_wmap_wodom"], r["q_wmap_wodom"]) and np.array_equal(sg["t_wmap_wodom"], r["t_wmap_wodom"]), j
            assert (sg["total_corner"], sg["total_surf"]) == (0, int(ref.sizes(1).sum())), j
        for ty, i in m.held():
            assert c.mapper_cube(ty, i).tobytes() == cm.cube(ty, i).tobytes(), (j, ty, i)
    return m


@pytest.mark.parametrize("name", E.DECISION_PATHS + E.JUMP_PATHS)
def test_crafted_paths_bit_exact(aloam, orc, name):
    """every frame of a crafted path against the model, the oracle and the reference's laserMapping.cpp (_run_path)"""
    frames = _frames(name)
    ref = _ref(orc, "gpu_cube_" + name)
    c = _ctx(aloam)
    try:
        _run_path(aloam, orc, c, frames, ref)
    finally:
        c.close()


@pytest.mark.parametrize("axis", range(3))
def test_a_store_of_face_points_rebuilds_into_the_same_cubes(aloam, orc, axis):
    """the store a decision path leaves -- points on the faces of the axis near where the path ends, -25 among them, and on the
    float either side -- exported and rebuilt with aloam_prior_map_build at the store's centre: no point is dropped and every cube holds
    the same points (build_cube_coord bins them as cube_coord did; the rebuild's per-cube filter keeps each point, as no two share
    a voxel, in voxel order)"""
    frames = _frames("decisions_%d" % axis)
    c, b = _ctx(aloam), _ctx(aloam)
    try:
        m = _run_path(aloam, orc, c, frames)
        store = c.mapper_export(aloam.EXPORT_MAP)
        for f in (-75.0, -25.0, 25.0) if axis < 2 else (-25.0, 25.0):   # (the k path's points on -75 have scrolled out by its end)
            assert (store[:, axis] == np.float32(f)).any(), f
        assert b.prior_map_build(EMPTY, store, c.mapper_state()["centre"]) == (0, 0)
        prior = b.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP)
        assert prior.shape == store.shape
        o = 0
        for ty, i in m.held():                       # sorted by (type, index): surf cubes only, in the export's order
            n = m.count(ty, i)
            assert np.array_equal(E.as_set(prior[o:o + n]), E.as_set(store[o:o + n])), i
            assert np.array_equal(E.as_set(store[o:o + n]), E.as_set(m.cube(ty, i))), i
            o += n
        assert o == store.shape[0]
    finally:
        c.close()
        b.close()


def _grid_cloud(rng, cen, t, kk):
    """one surf point near the middle of every cube (i, j, k) of the buffer with k in kk, under centre offsets cen, in the body
    frame of a pose with identity rotation and translation t"""
    ii, jj, ks = np.meshgrid(np.arange(E.CW), np.arange(E.CH), np.asarray(kk), indexing="ij")
    n = ii.size
    out = np.zeros((n, 4), np.float32)
    for a, idx in enumerate((ii, jj, ks)):
        out[:, a] = (idx.ravel() - cen[a]) * 50.0 + rng.uniform(-10, 10, n) - t[a]
    out[:, 3] = rng.uniform(0, 16, n)
    return out[rng.permutation(n)]


@pytest.mark.parametrize("growth", [0, 1])
@pytest.mark.parametrize("jump,fill_k", [(40, (4, 5, 6)), (12, (5,)), (-40, (4, 5, 6)), (-12, (5,))])
def test_slab_pool_after_wraps(aloam, orc, jump, fill_k, growth):
    """frame 0 puts a point in every cube of layers fill_k (1323 or 441 cubes); frame 1 jumps `jump` cubes along i, wrapping every
    cube (+-40) or five i-planes (+-12: the lowest ones on the shifts towards low indices, the highest ones on the shifts towards
    high indices); frame 2 puts a point in all 1323 cubes of layers 4-6 around the new centre.  The
    wrapped cubes' slabs are back in the pool: the store holds exactly the model's cubes -- those kept plus as many new ones as
    the 1024 slabs allow -- and every cube it holds equals the oracle's.  With growth on (one point per cube, so every run is one
    slab) the result is the same"""
    rng = np.random.default_rng(abs(jump) + (jump < 0))
    c = aloam.Aloam(n_scans=16, max_points=3000, max_map_points=20000)
    try:
        c.set_cube_growth(growth)
        c.mapper_reset()
        m, cm = E.Model(), orc.CubeMap()
        ident = np.array(E.IDENT_Q)
        far = np.array([50.0 * jump, 0.0, 0.0])
        frames = [(np.zeros(3), lambda: _grid_cloud(rng, E.CEN0, np.zeros(3), fill_k)), (far, lambda: EMPTY),
                  (far, lambda: _grid_cloud(rng, m.cen, far, (4, 5, 6)))]
        for j, (t, make) in enumerate(frames):
            kept = len(m.held())
            surf = make()
            pose, _ = m.frame(EMPTY, surf, ident, t)
            cm.step(EMPTY, surf, ident, t, 0.2, 0.4)
            gq, gt, st = c.mapper_step(EMPTY, surf, ident, t)
            assert np.array_equal(np.concatenate([gq, gt]), pose), j
            assert c.mapper_state()["centre"] == cm.state()["centre"], j
        new = len(m.held()) - kept
        assert kept == (0 if abs(jump) == 40 else 16 * E.CH) and new > 1024 - kept
        stored = 0
        for ty, i in m.held():
            got = c.mapper_cube(ty, i)
            if len(got):
                stored += 1
                assert got.tobytes() == cm.cube(ty, i).tobytes(), i
        assert stored == 1024 and c.mapper_state()["total_surf"] == sum(len(c.mapper_cube(1, i)) for _, i in m.held())
        assert st["flags"] & aloam.FLAG_CUBE_OVERFLOW
    finally:
        c.close()


# ---- relabelled stores inside the mapped lane streams

def _scans(synth, n):
    return [synth.scan("VLP-16", k, seed=synth.BASE_SEED + 91, n_az=900, max_range=40.0) for k in range(n)]


def _entries(dev, lanes):
    ptrs = np.array([[d.data_ptr()] * lanes for d in dev], np.uint64)
    counts = np.array([[d.shape[0]] * lanes for d in dev], np.int64)
    return ptrs, counts


def _source(aloam, synth, skip, n0):
    """a mapped lane run over scans 0 .. n0 - 1 and saved: (blob, the centre cube of its last map pose)"""
    import torch
    scans = _scans(synth, n0)
    dev = [torch.from_numpy(s).cuda() for s in scans]
    c = _ctx(aloam, max_batch=1, mapping_skip_frame=skip)
    try:
        ptrs, counts = _entries(dev, 1)
        ops = np.full((n0, 1), aloam.LANE_SCAN, np.int32); ops[0, 0] = aloam.LANE_START
        _, mp = c.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
        blob = np.asarray(c.lane_save(0)).copy()
    finally:
        c.close()
    cen = E.store_centre(blob)
    return blob, tuple(E.cube_coord(mp[-1, 0, 4 + a], cen[a]) for a in range(3))


def _continue(aloam, ctx, blobs, dev, sink):
    """restores blobs[l] into lane l and continues every lane over the scans of dev in one call: (odom, map poses, per lane the
    records of its rows (aloam_map_rows), the registered cloud of every row, EXPORT_SURROUND and EXPORT_MAP bytes)"""
    n, b = len(dev), len(blobs)
    for l, blob in enumerate(blobs):
        ctx.lane_restore(l, blob)
    ctx.set_registered_sink(sink)
    ctx.set_map_rows(True)
    ptrs, counts = _entries(dev, b)
    od, mp = ctx.scan_stream_lanes(ptrs, counts, np.full((n, b), aloam.LANE_SCAN, np.int32), True, mapped=True)
    rows = ctx.map_rows(n * b)
    stats = [{k: v[l::b] for k, v in rows.items()} for l in range(b)]   # per lane: its rows' kind, flags, stats and sizes
    begin, count = ctx.registered_rows(n * b)
    reg = [[sink[begin[r * b + l]:begin[r * b + l] + count[r * b + l]].cpu().numpy().tobytes() for r in range(n)] for l in range(b)]
    ex = [(ctx.mapper_export(aloam.EXPORT_SURROUND, l).tobytes(), ctx.mapper_export(aloam.EXPORT_MAP, l).tobytes()) for l in range(b)]
    return od, mp, stats, reg, ex


def _same_lane(run, l, ref, k, what):
    od, mp, stats, reg, ex = run
    rod, rmp, rstats, rreg, rex = ref
    assert np.array_equal(od[:, l], rod[:, k]) and np.array_equal(mp[:, l], rmp[:, k]), what
    assert all(np.array_equal(stats[l][key], rstats[k][key]) for key in rstats[k]), what
    assert reg[l] == rreg[k], what
    assert ex[l] == rex[k], what


def test_relabelled_stores_shift_first_and_later_and_run_identically(aloam, synth):
    """lanes restored from one saved store relabelled by d: d puts the centre cube at 2 or 18 in i and j and at 2 or 8 in k, so
    the first frame shifts, or 17 in i, so an optimised frame shifts later, as the vehicle crosses x = 25 m.  Every lane's poses,
    registered clouds and exports equal the unrelabelled lane's bit for bit"""
    import torch
    n0, n1 = 6, 30
    blob, ctr = _source(aloam, synth, 1, n0)
    ds = [(0, 0, 0)]
    for a, lo, hi in ((0, 2, 18), (1, 2, 18), (2, 2, 8)):
        for want in (lo, hi):
            d = [0, 0, 0]; d[a] = want - ctr[a]; ds.append(tuple(d))
    ds.append((17 - ctr[0], 0, 0))
    blobs = [E.relabel(blob, d) if any(d) else blob for d in ds]
    dev = [torch.from_numpy(s).cuda() for s in _scans(synth, n0 + n1)[n0:]]
    c = _ctx(aloam, max_batch=len(ds))
    sink = torch.zeros((len(ds) * n1 * 20000, 4), dtype=torch.float32, device="cuda")
    try:
        run = _continue(aloam, c, blobs, dev, sink)
        for l, d in enumerate(ds):
            _same_lane(run, l, run, 0, d)
            cen = c.mapper_state(l)["centre"]
            start = tuple(E.store_centre(blob)[a] + d[a] for a in range(3))
            assert (cen != start) == (l > 0), (d, cen, start)   # every relabelled lane shifted, the plain one never did
        assert not (run[2][len(ds) - 1]["flags"] & aloam.FLAG_MAP_TOO_THIN).any()   # the later shift is on optimised frames
    finally:
        c.close()


def test_sixteen_relabelled_lanes_at_skip_three_equal_their_solo_run(aloam, synth):
    """a 16-lane mapped call at mapping_skip_frame 3 in which each lane runs the same saved store under its own relabelling
    (first-frame shifts both ways on every axis, diagonal ones, none): every lane equals the solo run of the plain store"""
    import torch
    n0, n1 = 7, 12
    blob, ctr = _source(aloam, synth, 3, n0)
    counts = E.store_counts(blob)
    rng = np.random.default_rng(3)
    ds = [(0, 0, 0), (2 - ctr[0], 0, 0), (18 - ctr[0], 0, 0), (0, 2 - ctr[1], 0), (0, 18 - ctr[1], 0), (0, 0, 2 - ctr[2]),
          (0, 0, 8 - ctr[2]), (2 - ctr[0], 18 - ctr[1], 8 - ctr[2]), (18 - ctr[0], 2 - ctr[1], 2 - ctr[2])]
    while len(ds) < 16:
        d = tuple(int(v) for v in rng.integers([-7, -7, -2], [8, 8, 3]))
        if E.relabel_fits(counts, [], d):
            ds.append(d)
    blobs = [E.relabel(blob, d) if any(d) else blob for d in ds]
    dev = [torch.from_numpy(s).cuda() for s in _scans(synth, n0 + n1)[n0:]]
    solo = _ctx(aloam, max_batch=1, mapping_skip_frame=3)
    many = _ctx(aloam, max_batch=16, mapping_skip_frame=3)
    try:
        ref = _continue(aloam, solo, [blob], dev, torch.zeros((n1 * 20000, 4), dtype=torch.float32, device="cuda"))
        run = _continue(aloam, many, blobs, dev, torch.zeros((16 * n1 * 20000, 4), dtype=torch.float32, device="cuda"))
        for l, d in enumerate(ds):
            _same_lane(run, l, ref, 0, d)
        assert sum(many.mapper_state(l)["centre"] != tuple(E.store_centre(blob)[a] + d[a] for a in range(3)) for l, d in enumerate(ds)) >= 8
    finally:
        solo.close()
        many.close()


def test_a_shifted_store_moves_to_another_context(aloam, synth):
    """a store that has just shifted, saved and restored into lane 3 of another context, continues bit-identically"""
    import torch
    n0 = 6
    blob, ctr = _source(aloam, synth, 1, n0)
    shifted_blob = E.relabel(blob, (2 - ctr[0], 18 - ctr[1], 0))
    scans = _scans(synth, n0 + 8)
    dev = [torch.from_numpy(s).cuda() for s in scans[n0:]]
    a, b = _ctx(aloam, max_batch=1), _ctx(aloam, max_batch=4)
    try:
        _continue(aloam, a, [shifted_blob], dev[:3], torch.zeros((3 * 20000, 4), dtype=torch.float32, device="cuda"))
        assert a.mapper_state(0)["centre"] != E.store_centre(shifted_blob)
        saved = np.asarray(a.lane_save(0)).copy()
        sink = torch.zeros((5 * 20000, 4), dtype=torch.float32, device="cuda")
        ref = _continue(aloam, a, [saved], dev[3:], sink)
        b.lane_restore(3, saved)
        b.set_registered_sink(sink)
        n = len(dev) - 3
        ptrs, counts = _entries(dev[3:], 4)
        ops = np.full((n, 4), aloam.LANE_IDLE, np.int32); ops[:, 3] = aloam.LANE_SCAN
        od, mp = b.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
        assert np.array_equal(od[:, 3], ref[0][:, 0]) and np.array_equal(mp[:, 3], ref[1][:, 0])
        assert (b.mapper_export(aloam.EXPORT_SURROUND, 3).tobytes(), b.mapper_export(aloam.EXPORT_MAP, 3).tobytes()) == ref[4][0]
    finally:
        a.close()
        b.close()


def test_restore_refuses_out_of_range_centres_and_poses(aloam, synth):
    """aloam_lane_restore refuses, on the host, a saved store whose centre offset is beyond +-2^20, whose T_wmap_wodom is
    infinite or ~1e12 m away, or whose map position lies 17 cubes outside the buffer; the lane is left not running and a good
    snapshot still restores"""
    blob, ctr = _source(aloam, synth, 1, 3)
    cen = E.store_centre(blob)
    b, s = E.store_section(blob)
    import struct
    t = struct.unpack_from("<3d", b, s + 568)
    bad = [E.with_store_fields(blob, cen=(2 ** 20 + 1, cen[1], cen[2])), E.with_store_fields(blob, cen=(cen[0], 2 ** 31 - 1, cen[2])),
           E.with_store_fields(blob, t_wmap=(np.inf, t[1], t[2])), E.with_store_fields(blob, t_wmap=(t[0], 1e12, t[2])),
           E.with_store_fields(blob, t_wmap=(t[0], t[1], t[2] + 50.0 * (E.CD + 17 - ctr[2]))),
           E.with_store_fields(blob, q_wmap=(0.0, np.nan, 0.0, 1.0))]
    c = _ctx(aloam, max_batch=2)
    try:
        for k, blob_bad in enumerate(bad):
            with pytest.raises(aloam.AloamError) as e:
                c.lane_restore(1, blob_bad)
            assert e.value.code == aloam.ERR_SNAPSHOT, k
            with pytest.raises(aloam.AloamError):
                c.lane_save(1)                       # not running
        c.lane_restore(1, blob)
        assert np.asarray(c.lane_save(1)).tobytes() == np.asarray(blob).tobytes()
    finally:
        c.close()
