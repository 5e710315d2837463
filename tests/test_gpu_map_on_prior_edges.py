"""GPU: edge cases of mapping trajectories that start on a copy of the prior map (aloam_lane_map_on_prior; tests/
map_on_prior_edge_cases.py).  A START frame on a seeded store that leaves its submap thin has the map pose T_wmap_wodom exactly, so
the seeded oracle (an independent restatement of the store, fed the device's features: their intensities may differ from the
oracle's own in the last bit) fixes the pose, the centre, the valid list and every cube bit for bit, whatever the seed's table walk
and copy do.  Checked here: crafted layouts (chunk boundaries of the table walk,
cube kinds, centre offsets other than the default; loaded and built priors), then the restored-snapshot path bit for bit and the
oracle at 1e-4; the fit bounds run (a full slab pool, capacity-exact cubes, refusals that keep an earlier arming); both sides of the
slack bound on every axis; seeded records at every lane position against solo runs; seeded STARTs on lanes with stale state; the
arming across failed loads, lockstep calls and later loads; count-0 cubes."""
import numpy as np
import pytest

import cube_edge_cases as E
import lane_refs as R
import map_on_prior_edge_cases as M
from conftest import load_pkg

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY = -1, -4
IDLE, SCAN, START = 0, 1, 2
N_SCANS = 8
REG = 20000   # room per row in a registered sink


def _ctx(aloam, batch=1, maxpts=20000):
    return aloam.Aloam(n_scans=16, max_points=maxpts, max_batch=batch, max_ring_points=4096, max_map_points=400000)


_CACHE = {}


def _scans(synth):
    if "scans" not in _CACHE:
        scans = M.edge_scans(synth, N_SCANS)
        _CACHE["scans"] = (scans, R.to_device(scans))
    return _CACHE["scans"]


def _features(aloam):
    """the device's (less_sharp, less_flat) of every scan (extract_features: the stream calls' features bit for bit)"""
    if "feats" not in _CACHE:
        c = _ctx(aloam)
        _CACHE["feats"] = [(f["less_sharp"], f["less_flat"]) for f in (c.extract_features(s) for s in _CACHE["scans"][0])]
        c.close()
    return _CACHE["feats"]


def _base(aloam, synth, maxpts=20000):
    """a mapped snapshot of a context of this configuration (one mapped scan): what the crafted stores are written into"""
    if ("base", maxpts) not in _CACHE:
        c = _ctx(aloam, 1, maxpts)
        c.set_map_rows(True)
        _run(c, 1, {0: [(0, START)]})
        _CACHE["base", maxpts] = np.asarray(c.lane_save(0)).copy()
        c.close()
    return _CACHE["base", maxpts]


def _run(c, batch, plan, sink=True):
    """one mapped aloam_scan_stream_lanes call; plan = {lane: [(scan index or None for idle, op), ...]} -> {lane: (odometry rows,
    map rows, row records, registered clouds (bytes per row), (EXPORT_SURROUND, EXPORT_MAP) bytes after the call)}"""
    import torch
    A = load_pkg()
    dev = _CACHE["scans"][1]
    steps = max(len(p) for p in plan.values())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for l, p in plan.items():
        for k, (s, op) in enumerate(p):
            if op != IDLE:
                ptrs[k, l], counts[k, l], ops[k, l] = dev[s].data_ptr(), dev[s].shape[0], op
    buf = torch.zeros((steps * batch * REG, 4), dtype=torch.float32, device="cuda") if sink else None
    c.set_registered_sink(buf)
    c.set_map_rows(True)
    o, m = c.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
    rows = c.map_rows(steps * batch)
    begin, count = c.registered_rows(steps * batch) if sink else (None, None)
    out = {}
    for l, p in plan.items():
        live = [k for k, (_, op) in enumerate(p) if op != IDLE]
        rec = {k: v[l::batch][live] for k, v in rows.items()}
        reg = [buf[begin[k * batch + l]:begin[k * batch + l] + count[k * batch + l]].cpu().numpy().tobytes() for k in live] if sink else None
        try:
            ex = (c.mapper_export(A.EXPORT_SURROUND, l).tobytes(), c.mapper_export(A.EXPORT_MAP, l).tobytes())
        except A.AloamError:   # a localising lane has no store
            ex = None
        out[l] = (o[live, l], m[live, l], rec, reg, ex)
    c.set_registered_sink(None)
    return out


@pytest.fixture(autouse=True)
def _scans_on_device(synth):
    _scans(synth)


def _same(a, b, what, rows=None):
    """two results of _run for one lane, bit for bit: poses, row records, registered clouds and, unless only rows `rows` of a
    are compared, both exports"""
    s = slice(None) if rows is None else rows
    assert np.array_equal(a[0][s], b[0]) and np.array_equal(a[1][s], b[1]), what
    for k in b[2]:
        assert np.array_equal(a[2][k][s], b[2][k]), (what, k)
    assert a[3][s] == b[3], what
    if rows is None:
        assert a[4] == b[4], what


def _seeded_solo(aloam, synth, prior, T, scans, maxpts=20000):
    """scans as a seeded trajectory from T on a fresh one-lane context whose prior map is `prior` (a snapshot, or a pair of clouds
    and centre offsets to build from)"""
    key = ("solo", id(prior), T.tobytes(), tuple(scans), maxpts)
    if key not in _CACHE:
        c = _ctx(aloam, 1, maxpts)
        _load(c, prior)
        c.lane_map_on_prior(0, T[:4], T[4:])
        _CACHE[key] = _run(c, 1, {0: [(s, START if k == 0 else SCAN) for k, s in enumerate(scans)]})[0]
        c.close()
    return _CACHE[key]


def _load(c, prior):
    if isinstance(prior, tuple):
        c.prior_map_build(prior[0], prior[1], prior[2])
    else:
        c.prior_map_load(prior)


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def _check_start(aloam, orc, synth, c, lane, scene, T, res, bounded=None):
    """the START frame of a seeded lane (the first row of res) against the seeded oracle: the map pose is T, a thin frame; centre,
    valid list and every cube of the lane's store after the frame bit for bit (bounded: the cubes the store holds, each equal to
    the oracle's, and the set of cubes holding a slab).  Returns the oracle CubeMap after the frame."""
    cm = M.seeded_cubemap(orc, scene, T)
    assert np.array_equal(res[0][0], np.concatenate([M.IDENT_Q, np.zeros(3)]))
    poses, infos = M.oracle_steps(cm, _features(aloam)[:1], res[0][:1])
    assert not infos[0]["optimised"] and np.array_equal(poses[0], T) and np.array_equal(res[1][0], T)
    assert res[2]["flags"][0] & aloam.FLAG_MAP_TOO_THIN
    sg, so = c.mapper_state(lane), cm.state()
    assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
    got, counts = M.split_store(c.lane_save(lane))
    want = M.oracle_store(cm)
    if bounded is None:
        assert {k for k, v in got.items() if len(v)} == set(want) and (counts != 0).all()
    else:
        assert set(got) == bounded
    for k, v in got.items():
        assert np.array_equal(v, want.get(k, np.zeros((0, 4), np.float32))), k
    return cm


def _restored(aloam, synth, blob, res, n):
    """aloam_mapper_step on lane 0 of a scratch context restored from blob, fed the features of scans 0 .. n-1 and the odometry
    rows of res: (map poses, stats, the scratch context's snapshot)"""
    scans = _CACHE["scans"][0]
    scratch, feats = _ctx(aloam), _ctx(aloam)
    scratch.lane_restore(0, blob)
    poses, stats = [], []
    for j in range(n):
        f = feats.extract_features(scans[j])
        q, t, st = scratch.mapper_step(f["less_sharp"], f["less_flat"], res[0][j][:4], res[0][j][4:])
        poses.append(np.concatenate([q, t]))
        stats.append(st)
    saved = np.asarray(scratch.lane_save(0)).copy()
    scratch.close()
    feats.close()
    return np.array(poses), stats, saved


def _joined(a, b):
    """the results of _run for one lane over two consecutive calls as one (the exports after the second)"""
    return tuple(np.concatenate([a[i], b[i]]) for i in (0, 1)) + ({k: np.concatenate([a[2][k], b[2][k]]) for k in a[2]},
                                                                 a[3] + b[3] if a[3] is not None else None, b[4])


def _same_as_restored(res, ref, what):
    poses, stats, _ = ref
    assert np.array_equal(res[1], poses), what
    for j, st in enumerate(stats):
        for k in R.STAT_KEYS:
            got = list(res[2][k][j]) if k == "termination" else res[2][k][j]
            assert got == st[k], (what, j, k)


def _table(blob):
    b, s = E.store_section(blob)
    return b[s:s + 592], E.store_counts(blob), b[s + 39408:]


# ---- 1. crafted layouts

def _built_scene(aloam, c, scene):
    """scene as aloam_prior_map_build makes it (every point in a voxel of its own: the counts are exact; the order in a cube is the
    build's), read back from the prior map's export"""
    ex = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP)
    built, off = M.Scene(scene.cen, scene.init_ijk), 0
    built.t = scene.t
    for i in range(M.NCUBE):
        for ty in (0, 1):
            n = int(scene.counts[ty, i])
            if n > 0:
                built.put(ty, i, ex[off:off + n])
                assert np.array_equal(E.as_set(ex[off:off + n]), E.as_set(scene.cubes[ty, i])), (ty, i)
                off += n
    assert off == len(ex)
    return built


@pytest.mark.parametrize("how", ["loaded", "built"])
def test_crafted_layout_start_is_the_seeded_oracle_then_the_restored_path(aloam, orc, synth, how):
    """scene (a): cubes 0, 4850 and both sides of every chunk boundary, corner-only, surf-only and one-point cubes, centre (7, 12,
    4); loaded from a snapshot, or built from its clouds.  START bit for bit against the seeded oracle; then 5 frames: every row
    against the restored-snapshot path bit for bit, the map poses against the oracle at 1e-4"""
    s = M.scene_layout()
    base = _base(aloam, synth)
    n = 6
    c = _ctx(aloam)
    if how == "loaded":
        c.prior_map_load(M.scene_blob(base, s))
    else:
        corner, surf = s.clouds()
        assert c.prior_map_build(corner, surf, s.cen) == (0, 0)
        s = _built_scene(aloam, c, s)
    T = M.normalised(s.q, s.t)
    c.lane_map_on_prior(0, T[:4], T[4:])
    res = _run(c, 1, {0: [(0, START)]})[0]
    cm = _check_start(aloam, orc, synth, c, 0, s, T, res)
    res = _joined(res, _run(c, 1, {0: [(k, SCAN) for k in range(1, n)]})[0])
    poses, _ = M.oracle_steps(cm, _features(aloam)[1:n], res[0][1:n])
    R.assert_near(res[1][1:], poses, "map poses after the START")
    ref = _restored(aloam, synth, M.scene_blob(base, s, T), res, n)
    _same_as_restored(res, ref, how)
    mine, theirs = _table(c.lane_save(0)), _table(ref[2])
    assert mine[0] == theirs[0] and np.array_equal(mine[1], theirs[1]) and mine[2] == theirs[2]
    c.close()


# ---- 2. fit bounds

def _localise_kept(aloam, c, prior, T, what):
    """c's lane 0 holds an aloam_lane_localise arming from T: its next START localises as on a fresh context"""
    res = _run(c, 1, {0: [(k, START if k == 0 else SCAN) for k in range(3)]}, sink=False)[0]
    d = _ctx(aloam, 1, int(c.cfg.max_points))
    _load(d, prior)
    d.lane_localise(0, T[:4], T[4:])
    ref = _run(d, 1, {0: [(k, START if k == 0 else SCAN) for k in range(3)]}, sink=False)[0]
    d.close()
    assert (res[2]["kind"] == aloam.ROW_LOCALISED).all(), what
    assert np.array_equal(res[1], ref[1]), what


def test_a_full_slab_pool_seeds_runs_and_drops_new_cubes(aloam, orc, synth):
    """1024 cubes of each type outside the START's block: the seed takes every slab, the START's new cubes get none (flagged on
    the rows that insert), every seeded cube equals the oracle's.  1023 arms; 1025 is refused and keeps a localise arming"""
    base = _base(aloam, synth)
    s = M.scene_pool(1024)
    prior = M.scene_blob(base, s)
    T = M.normalised(s.q, s.t)
    c = _ctx(aloam)
    c.prior_map_load(prior)
    c.lane_map_on_prior(0, T[:4], T[4:])
    res = _run(c, 1, {0: [(0, START)]})[0]
    held = {(ty, int(i)) for ty in (0, 1) for i in np.flatnonzero(s.counts[ty] >= 0)}
    _check_start(aloam, orc, synth, c, 0, s, T, res, bounded=held)
    more = _run(c, 1, {0: [(1, SCAN), (2, SCAN)]})[0]
    assert (np.concatenate([res[2]["flags"], more[2]["flags"]]) & aloam.FLAG_CUBE_OVERFLOW).all()
    assert set(M.split_store(c.lane_save(0))[0]) == held   # still no new slab
    c.prior_map_load(M.scene_blob(base, M.scene_pool(1023)))
    c.lane_map_on_prior(0, T[:4], T[4:])
    _expect(aloam, aloam.ERR_SNAPSHOT, lambda: c.prior_map_load(M.scene_blob(base, M.scene_pool(1025))))   # a snapshot holds <= 1024
    s25 = M.scene_pool(1025)
    prior25 = tuple(s25.clouds()) + (s25.cen,)
    _load(c, prior25)
    c.lane_localise(0, T[:4], T[4:])
    _expect(aloam, ERR_CAPACITY, lambda: c.lane_map_on_prior(0, T[:4], T[4:]))
    _localise_kept(aloam, c, prior25, T, "1025 cubes")
    c.close()


@pytest.mark.parametrize("ty,maxpts", [(0, 20000), (1, 65536)])
def test_capacity_exact_cubes_seed_and_overflow_on_the_start_only(aloam, orc, synth, ty, maxpts):
    """one cube of exactly the slab capacity (corner 16384; surf 65536 at max_points 65536), two points in each of its voxels, in
    the START's own cube: the START's appends to it are dropped and flagged, its re-filter is the oracle filter of the seeded
    points alone and halves it, so the next frames append and are not flagged.  Capacity + 1 (built) is refused and keeps a
    localise arming."""
    cap = (16384, 65536)[ty]
    base = _base(aloam, synth, maxpts)
    s = M.scene_capacity(ty, cap, True)
    T = M.normalised(s.q, s.t)
    c = _ctx(aloam, 1, maxpts)
    c.prior_map_load(M.scene_blob(base, s))
    c.lane_map_on_prior(0, T[:4], T[4:])
    res = _run(c, 1, {0: [(0, START)]}, sink=False)[0]
    full = E.cube_index(*s.init_ijk)
    alone = M.seeded_cubemap(orc, s, T)
    alone.step(np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32), M.IDENT_Q, np.zeros(3), *M.LEAVES)
    cm = M.seeded_cubemap(orc, s, T)
    M.oracle_steps(cm, _features(aloam)[:1], res[0][:1])
    assert len(cm.cube(ty, full)) > len(alone.cube(ty, full))   # the scan reached the full cube
    got, _ = M.split_store(c.lane_save(0))
    assert np.array_equal(got[ty, full], alone.cube(ty, full)) and len(got[ty, full]) == cap // 2
    for k, v in got.items():
        if k != (ty, full):
            assert np.array_equal(v, cm.cube(*k)), k
    assert np.array_equal(res[1][0], T) and res[2]["flags"][0] & aloam.FLAG_CUBE_OVERFLOW
    more = _run(c, 1, {0: [(1, SCAN), (2, SCAN)]}, sink=False)[0]
    assert not (more[2]["flags"] & aloam.FLAG_CUBE_OVERFLOW).any()
    c.close()
    # capacity + 1: a built map (a snapshot's counts are bounded by its slab capacity)
    over = M.scene_capacity(ty, cap + 1 if ty == 0 else cap, False)
    r = _ctx(aloam, 1, maxpts if ty == 0 else cap - 1)
    prior = tuple(over.clouds()) + (over.cen,)
    _load(r, prior)
    assert r.mapper_export_size(aloam.EXPORT_MAP, aloam.PRIOR_MAP) == int(np.maximum(over.counts, 0).sum())
    r.lane_localise(0, T[:4], T[4:])
    _expect(aloam, ERR_CAPACITY, lambda: r.lane_map_on_prior(0, T[:4], T[4:]))
    _localise_kept(aloam, r, prior, T, "capacity + 1")
    r.close()


# ---- 3. the slack bound

@pytest.mark.parametrize("axis,side", [(a, s) for a in range(3) for s in ("low", "high")])
def test_the_slack_bound_arms_and_runs(aloam, orc, synth, axis, side):
    """the start position on the slack bound: the refused double returns ALOAM_ERR_INVALID_ARG; the accepted one arms, its START
    shifts the buffer 19 cubes, past every seeded cube, bit for bit against the seeded oracle and the model's centre and valid
    list; the next frames equal the restored path"""
    s = M.scene_layout()
    base = _base(aloam, synth)
    a, sd, acc, ref = [x for x in M.slack_inits(s.cen, s.t) if x[0] == axis and x[1] == side][0]
    c = _ctx(aloam)
    c.prior_map_load(M.scene_blob(base, s))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_map_on_prior(0, s.q, ref))
    T = M.normalised(s.q, acc)
    c.lane_map_on_prior(0, T[:4], T[4:])
    n = 4
    res = _run(c, 1, {0: [(0, START)]})[0]
    _check_start(aloam, orc, synth, c, 0, s, T, res)
    centre, valid = M.start_model(s, T)
    st = c.mapper_state(0)
    assert (st["centre"], st["valid"]) == (centre, valid) and abs(centre[axis] - s.cen[axis]) == 19
    full = _joined(res, _run(c, 1, {0: [(k, SCAN) for k in range(1, n)]})[0])
    ref_path = _restored(aloam, synth, M.scene_blob(base, s, T), full, n)
    _same_as_restored(full, ref_path, (axis, side))
    assert _table(c.lane_save(0))[2] == _table(ref_path[2])[2]
    c.close()


# ---- 4. record indexing

def _prior_layout(aloam, synth):
    if "prior_layout" not in _CACHE:
        _CACHE["prior_layout"] = M.scene_blob(_base(aloam, synth), M.scene_layout())
    return _CACHE["prior_layout"]


def _inits(n):
    """n inits around the layout scene's start, the first two on both slack extremes along i"""
    s = M.scene_layout()
    out = [M.normalised(s.q, x[2]) for x in M.slack_inits(s.cen, s.t)[:2]]
    rng = np.random.default_rng(12)
    while len(out) < n:
        q = np.array(E.quat(rng.normal(size=3), rng.uniform(-0.3, 0.3)))
        out.append(M.normalised(q, s.t + rng.uniform(-30, 30, 3)))
    return out


def test_sixteen_lanes_seeded_in_one_step_equal_their_solo_runs(aloam, synth):
    prior = _prior_layout(aloam, synth)
    inits = _inits(16)
    c = _ctx(aloam, 16)
    c.prior_map_load(prior)
    for l, T in enumerate(inits):
        c.lane_map_on_prior(l, T[:4], T[4:])
    n = 3
    got = _run(c, 16, {l: [(k, START if k == 0 else SCAN) for k in range(n)] for l in range(16)})
    c.close()
    for l, T in enumerate(inits):
        _same(got[l], _seeded_solo(aloam, synth, prior, T, tuple(range(n))), "lane %d" % l)


def test_seeded_lanes_three_seven_fifteen_beside_fresh_and_localising_lanes(aloam, synth):
    """lanes 3, 7 and 15 seeded at steps 0, 1 and 2 while lane 0 maps fresh, lane 1 localises (both STARTing at step 0, beside
    lane 3's seeded START) and lane 2 maps fresh from step 1"""
    prior = _prior_layout(aloam, synth)
    inits = _inits(6)[2:]
    c = _ctx(aloam, 16)
    c.prior_map_load(prior)
    n = 3
    first = {0: 0, 1: 0, 2: 1, 3: 0, 7: 1, 15: 2}
    for l, T in ((3, inits[0]), (7, inits[1]), (15, inits[2])):
        c.lane_map_on_prior(l, T[:4], T[4:])
    c.lane_localise(1, inits[3][:4], inits[3][4:])
    plan = {l: [(None, IDLE)] * f + [(k, START if k == 0 else SCAN) for k in range(n)] for l, f in first.items()}
    got = _run(c, 16, plan)
    c.close()
    for l, T in ((3, inits[0]), (7, inits[1]), (15, inits[2])):
        ref = _seeded_solo(aloam, synth, prior, T, tuple(range(n)))
        _same(got[l], ref, "lane %d" % l)
    solo = _ctx(aloam)
    fresh = _run(solo, 1, {0: [(k, START if k == 0 else SCAN) for k in range(n)]})[0]
    solo.close()
    solo = _ctx(aloam)
    solo.prior_map_load(prior)
    solo.lane_localise(0, inits[3][:4], inits[3][4:])
    loc = _run(solo, 1, {0: [(k, START if k == 0 else SCAN) for k in range(n)]})[0]
    solo.close()
    _same(got[0], fresh, "fresh lane 0")
    _same(got[2], fresh, "fresh lane 2")
    _same(got[1], loc, "localising lane 1")


# ---- 5. stale lanes

def _shifting_blob(aloam, synth):
    """the layout scene's store with the vehicle in cube i = 2 (T_wmap_wodom a translation): the next frame shifts the buffer one
    cube up in i, and layer i = 20, whose cubes hold slabs, wraps out -- their slabs go back to the pool out of order.  Returns the
    snapshot and the store's centre offsets"""
    s = M.scene_layout()
    assert any(E.ijk_of(i)[0] == 20 for i in np.flatnonzero((s.counts >= 0).any(0)))
    t = M.cube_centre((2,) + s.init_ijk[1:], s.cen) + np.array([3.25, -4.5, 1.75])
    return M.scene_blob(_base(aloam, synth), s, M.normalised(s.q, t)), s.cen


@pytest.mark.parametrize("before", ["shifted", "localising", "seeded_one_row", "seeded_then_fresh"])
def test_a_seeded_start_on_a_stale_lane(aloam, synth, before):
    """lane 3 runs another trajectory and then STARTs seeded in the same call: a restored store whose previous frame shifted the
    buffer and freed slabs out of order, a localising trajectory, a 1-row seeded trajectory (the last two begun in an earlier call);
    or lane 3 STARTs seeded and then STARTs again unarmed, which is a fresh trajectory.  Every seeded part equals the
    same seeded run on a fresh context, the fresh part an unarmed lane's"""
    prior = _prior_layout(aloam, synth)
    T = _inits(3)[2]
    seeded = tuple(range(3))
    ref = _seeded_solo(aloam, synth, prior, T, seeded)
    c = _ctx(aloam, 4)
    c.prior_map_load(prior)
    plan = [(k, START if k == 0 else SCAN) for k in seeded]
    if before == "shifted":
        blob, cen = _shifting_blob(aloam, synth)
        c.lane_restore(3, blob)
        _run(c, 4, {3: [(1, SCAN)]}, sink=False)
        assert c.mapper_state(3)["centre"] == (cen[0] + 1, cen[1], cen[2])   # shifted up in i: layer 20 wrapped out
        c.lane_map_on_prior(3, T[:4], T[4:])
        got = _run(c, 4, {3: [(2, SCAN)] + plan})[3]
    elif before == "localising":
        c.lane_localise(3, T[:4], T[4:])
        _run(c, 4, {3: [(k, START if k == 0 else SCAN) for k in range(3)]}, sink=False)
        c.lane_map_on_prior(3, T[:4], T[4:])
        got = _run(c, 4, {3: [(3, SCAN)] + plan})[3]
    elif before == "seeded_one_row":
        c.lane_map_on_prior(3, T[:4], T[4:])
        _run(c, 4, {3: [(5, START)]}, sink=False)
        c.lane_map_on_prior(3, T[:4], T[4:])
        got = _run(c, 4, {3: plan})[3]
    else:
        c.lane_map_on_prior(3, T[:4], T[4:])
        got = _run(c, 4, {3: plan + [(k, START if k == 0 else SCAN) for k in range(3)]})[3]
        solo = _ctx(aloam)
        fresh = _run(solo, 1, {0: [(k, START if k == 0 else SCAN) for k in range(3)]})[0]
        solo.close()
        _same(got, ref, before, rows=slice(0, 3))
        _same(got, fresh, before, rows=slice(3, 6))
        assert got[4] == fresh[4]
        c.close()
        return
    k0 = len(got[0]) - 3
    _same(got, ref, before, rows=slice(k0, None))
    assert got[4] == ref[4], before   # the seeded trajectory ends the call: the stores are the same
    c.close()


# ---- 6. lifecycle gaps

def test_the_arming_survives_a_failed_load_and_a_lockstep_call_and_a_seeded_lane_ignores_later_loads(aloam, synth):
    prior = _prior_layout(aloam, synth)
    T = _inits(3)[2]
    ref = _seeded_solo(aloam, synth, prior, T, tuple(range(4)))
    plan = [(k, START if k == 0 else SCAN) for k in range(4)]
    c = _ctx(aloam, 2)
    c.prior_map_load(prior)
    # a lockstep call (on a context that has run no lane call: the lane schedule takes over the frame counter) keeps it
    c.lane_map_on_prior(0, T[:4], T[4:])
    dev = _CACHE["scans"][1]
    ptrs = np.array([d.data_ptr() for d in dev[:2]], np.uint64)
    counts = np.array([d.shape[0] for d in dev[:2]], np.int64)
    c.scan_stream_mapped(ptrs, counts, True)
    _same(_run(c, 2, {0: plan})[0], ref, "after a lockstep call")
    # a load that fails keeps it
    c.lane_map_on_prior(0, T[:4], T[4:])
    with pytest.raises(aloam.AloamError):
        c.prior_map_load(prior[:-16])   # malformed: shorter than its header says
    _same(_run(c, 2, {0: plan})[0], ref, "after a failed load")
    # after its START a seeded lane does not read the prior map: another map loaded between calls changes nothing
    c.lane_map_on_prior(0, T[:4], T[4:])
    a = _run(c, 2, {0: plan[:2]})[0]
    c.prior_map_load(M.scene_blob(_base(aloam, synth), M.scene_pool(40)))
    b = _run(c, 2, {0: plan[2:]})[0]
    _same(_joined(a, b), ref, "across a later load")
    c.close()


# ---- 7. count-0 cubes

def test_count_zero_cubes_seed_without_a_slab(aloam, synth):
    """scene (d): a prior snapshot with count-0 cubes inside and outside the START's valid block.  The seeded lane gives them no
    slab, the restored lane a slab of 0 points: map poses and rows are bit-identical, and the saved stores differ only by -1 for 0
    at the count-0 cubes the trajectory never inserted into"""
    s = M.scene_zero()
    base = _base(aloam, synth)
    T = M.normalised(s.q, s.t)
    n = 6
    c = _ctx(aloam)
    c.prior_map_load(M.scene_blob(base, s))
    c.lane_map_on_prior(0, T[:4], T[4:])
    res = _run(c, 1, {0: [(k, START if k == 0 else SCAN) for k in range(n)]})[0]
    ref = _restored(aloam, synth, M.scene_blob(base, s, T), res, n)
    _same_as_restored(res, ref, "count-0 cubes")
    head_a, counts_a, pts_a = _table(c.lane_save(0))
    head_b, counts_b, pts_b = _table(ref[2])
    assert head_a == head_b and pts_a == pts_b
    differ = {(ty, int(i)) for ty in (0, 1) for i in np.flatnonzero(counts_a[ty] != counts_b[ty])}
    assert differ <= set(s.zeros) and all(counts_a[k] == -1 and counts_b[k] == 0 for k in differ)
    outside = {(ty, i) for ty, i in s.zeros if i not in M.block(s.init_ijk)}
    assert outside <= differ
    c.close()


def test_count_zero_cubes_at_a_full_pool(aloam, orc, synth):
    """a snapshot whose 1024 slabs of each type are all taken, 96 of them by count-0 cubes.  The restored lane's pool is full, so the
    START's new cubes get no slab and its row is flagged; the seeded lane gave the count-0 cubes no slab, so its 96 free slabs take
    the new cubes and the START equals the unbounded seeded oracle.  The equivalence with the restored path holds only while the
    restored lane's pool is not exhausted."""
    s = M.scene_zero_pool(96)
    base = _base(aloam, synth)
    assert M.fits(s.counts, s.cen, s.t, 20000) == "ok" and ((s.counts >= 0).sum(1) == M.POOL).all()
    T = M.normalised(s.q, s.t)
    c = _ctx(aloam)
    c.prior_map_load(M.scene_blob(base, s))
    c.lane_map_on_prior(0, T[:4], T[4:])
    res = _run(c, 1, {0: [(0, START)]})[0]
    _check_start(aloam, orc, synth, c, 0, s, T, res)
    assert not res[2]["flags"][0] & aloam.FLAG_CUBE_OVERFLOW
    got, _ = M.split_store(c.lane_save(0))
    new = {k for k in got if s.counts[k] < 0}
    assert 0 < len(new) <= 96
    poses, stats, saved = _restored(aloam, synth, M.scene_blob(base, s, T), res, 1)
    assert np.array_equal(poses[0], res[1][0]) and stats[0]["flags"] & aloam.FLAG_CUBE_OVERFLOW
    rgot, rcounts = M.split_store(saved)
    assert not new & set(rgot) and all(rcounts[k] == 0 for k in s.zeros)
    c.close()
