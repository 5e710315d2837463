"""GPU: cube growth's slab allocator at its edges (cubemap.cu take_run, cube_insert_body, rotate_line, store_import_body).
aloam_mapper_step on lane 0 runs the scenarios of tests/growth_edge_cases.py -- crafted growth-on snapshots restored with
aloam_lane_restore, or stores built from aloam_mapper_reset -- and after every frame the pose, centre, flags, totals, the
ALOAM_EXPORT_MAP export (byte for byte, in store order) and every cube the frame changed equal the model's; stores built from
aloam_mapper_reset also hold the oracle's CubeMap points (its prefix where the device dropped the rest).  Every pool is exactly
tight, and every negative control (one more one-slab cube) flags where the model says.  A real growth-on VLP-16 store, relabelled
so that its first mapped frame wraps a plane of one-slab cubes whose freed block its densest cube grows into, runs in 16 lanes of
one mapped lane-stream call, each equal to its solo run."""
import struct

import numpy as np
import pytest

import cube_edge_cases as E
import growth_edge_cases as G

pytestmark = pytest.mark.gpu


def _run(aloam, orc, sc):
    """the scenario on a new context and in the model, compared after every frame; returns per frame (flags, export bytes)"""
    cfg = G.config(sc.max_points)
    c = aloam.Aloam(**cfg)
    cm = orc.CubeMap() if sc.fresh else None
    out = []
    try:
        c.set_cube_growth(sc.growth)
        c.mapper_reset()
        before = {}
        for j, (step, m, pose, flag) in enumerate(G.walk(sc)):
            if step[0] == "restore":
                c.lane_restore(0, G.snapshot(cfg, step[1], step[2]))
                before = {k: m.count(*k) for k in m.held()}
                continue
            if step[0] == "reset":
                c.set_cube_growth(step[1])
                c.mapper_reset()
                before = {}
                continue
            _, t, corner, surf = step
            gq, gt, st = c.mapper_step(corner, surf, G.IDENT, t)
            what = (sc.name, j)
            assert np.array_equal(np.concatenate([gq, gt]), pose), what
            assert st["flags"] == aloam.FLAG_MAP_TOO_THIN | (aloam.FLAG_CUBE_OVERFLOW if flag else 0), (what, st["flags"])
            state = c.mapper_state()
            assert state["centre"] == tuple(m.cen) and (state["total_corner"], state["total_surf"]) == m.totals(), what
            export = c.mapper_export(aloam.EXPORT_MAP).tobytes()
            assert export == m.payload().tobytes(), what
            now = {k: m.count(*k) for k in m.held()}
            for k in set(now) | set(before):
                if now.get(k) != before.get(k):
                    assert np.array_equal(E.as_set(c.mapper_cube(*k)), E.as_set(m.cube(*k))), (what, k)
            before = now
            if cm is not None:
                cm.step(corner, surf, G.IDENT, t, G.LEAF, G.LEAF)
                for k, n in now.items():
                    assert c.mapper_cube(*k).tobytes() == cm.cube(*k)[:n].tobytes(), (what, k)
            out.append((st["flags"], export))
    finally:
        c.close()
    return out


NAMES = [n for n in G.scenarios() if not n.startswith("restart")]


@pytest.mark.parametrize("name", NAMES)
def test_scenario_against_the_model(aloam, orc, name):
    """wraps that free runs of 2-256 slabs (one bitmap word freed by four lines of one shift step, towards high and low indices),
    the whole-pool run, competing growths with growth on and off, the deferred free, a retry after a wrap, an aligned block that
    two free slabs do not make, growth by two orders in one insert, and their negative controls"""
    _run(aloam, orc, G.scenarios()[name])


@pytest.mark.parametrize("growth", [1, 0])
def test_restart_on_a_fragmented_pool_equals_a_fresh_context(aloam, orc, growth):
    """a lane left with a fragmented growth-on pool, restarted by aloam_mapper_reset under growth on or off: 1024 one-slab cubes
    fit and the 1025th is flagged, and both frames equal those of a fresh context byte for byte (flags and exports)"""
    g = "on" if growth else "off"
    a = _run(aloam, orc, G.scenarios()["restart_" + g])
    b = _run(aloam, orc, G.scenarios()["restart_%s_fresh" % g])
    assert a[-2:] == b
    assert not b[0][0] & aloam.FLAG_CUBE_OVERFLOW and b[1][0] & aloam.FLAG_CUBE_OVERFLOW
    assert len(b[0][1]) == 16 * len(G.NEW78) and len(b[1][1]) == 16 * 1024


# ---- a real growth-on store in the mapped lane streams, its shift wrapping a plane of synthetic runs

N0, N1 = 24, 8
LOW = ((1, 0, 0), (2, 0, 0))                      # one-slab fillers whose cube indices come before the plane's cubes
PLANE = tuple((20, j, 0) for j in range(4))       # four one-slab cubes on the plane the first frame wraps: slabs 4 .. 7


def _real_store(aloam, synth):
    """a growth-on VLP-16 lane at the default leaves, mapped over N0 scans and saved, relabelled by d = 2 - (its centre cube) in i
    so that the first frame of its continuation shifts towards high indices and wraps plane i = 20.  Returns (config, the
    continuation's scans on the device, the relabelled snapshot, its counts and points per cube, the densest corner cube).  The
    corner slab capacity is min(16384, max_points)"""
    import test_gpu_cube_edges as CE
    import test_gpu_cube_growth_edges as GE
    import lane_refs as R
    scans = R.traj(synth, 0, N0 + N1)
    kw = dict(n_scans=16, max_points=R.maxn([scans]) + 1024, max_map_points=400000)
    dev = R.to_device(scans)
    c = aloam.Aloam(max_batch=1, **kw)
    try:
        c.set_cube_growth(1)
        ptrs, counts = CE._entries(dev[:N0], 1)
        ops = np.full((N0, 1), aloam.LANE_SCAN, np.int32)
        ops[0, 0] = aloam.LANE_START
        _, mp = c.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
        blob = np.asarray(c.lane_save(0)).copy()
        export = c.mapper_export(aloam.EXPORT_MAP, 0).copy()
    finally:
        c.close()
    cen = E.store_centre(blob)
    ctr = E.cube_coord(mp[-1, 0, 4], cen[0])
    rel = E.relabel(blob, (2 - ctr, 0, 0))
    counts, cubes = GE._split(rel, export)
    dense = int(np.argmax(counts[0]))
    cap = min(16384, kw["max_points"])
    assert cap < counts[0, dense] <= 2 * cap, "the densest corner cube holds a run of two slabs"
    return kw, dev[N0:], rel, counts, cubes, dense


def _variant(rel, counts, cubes, dense, extra):
    """the real store with its densest corner cube padded to two full slabs by points on a 0.2 m grid 0.1 m above
    its cube's floor, far below every scan (each alone in its voxel: the re-filter keeps them); the LOW fillers, the PLANE cubes and
    fillers on layers k = 1 .. 3 make 1023 corner slabs (extra: one LOW filler more, 1024).  Packing puts the dense cube on slabs
    0, 1, the LOW fillers after it and the plane on the aligned block 4 .. 7 (extra: 5 .. 8)"""
    import test_gpu_cube_growth_edges as GE
    rng = np.random.default_rng(21)
    cap = struct.unpack_from("<i", np.asarray(rel).tobytes(), 68)[0]   # the snapshot's corner slab capacity
    cen = E.store_centre(rel)
    counts, cubes = counts.copy(), dict(cubes)
    ijk = E.ijk_of(dense)
    lo = [(ijk[a] - cen[a]) * 50.0 - 25.0 for a in range(3)]
    pad = 2 * cap - int(counts[0, dense])
    g = np.arange(pad)
    p = np.zeros((pad, 4), np.float32)
    p[:, 0] = lo[0] + 0.1 + 0.2 * (g % 250)
    p[:, 1] = lo[1] + 0.1 + 0.2 * (g // 250)
    p[:, 2] = lo[2] + 0.1
    cubes[(0, dense)] = np.concatenate([cubes[(0, dense)], p])
    counts[0, dense] = 2 * cap
    low = LOW + (((3, 0, 0),) if extra else ())
    far = [(i, j, k) for k in (1, 2, 3) for j in range(E.CH) for i in range(20)]
    for c in low + PLANE + tuple(far):
        i = E.cube_index(*c)
        if GE._slabs(counts[0], cap) == 1023 + extra:
            break
        assert counts[0, i] < 0 and counts[1, i] < 0
        counts[0, i] = 1
        cubes[(0, i)] = G.at(c, rng, 1, cen)
    assert GE._slabs(counts[0], cap) == 1023 + extra
    runs, _ = G.pack(counts[0], cap)
    assert runs[dense] == (0, 1) and [runs[E.cube_index(*c)][0] for c in PLANE] == list(range(4 + extra, 8 + extra))
    return E.with_store_fields(rel, counts=counts, points=GE._payload(counts, cubes))


def test_sixteen_lanes_whose_shift_frees_a_block_for_a_dense_cube(aloam, synth):
    """a real growth-on VLP-16 store whose densest corner cube fills two slabs, 1023 corner slabs held and the only aligned free
    block of four the one the first frame's wrap of plane i = 20 frees (four one-slab cubes, freed by four lines of one shift
    step).  The dense cube grows into it on that frame.  The variant with one filler more puts the plane's cubes on slabs 5 .. 8:
    no aligned block of four comes free, the dense cube cannot grow and its rows are flagged (error word bit 4).  16 lanes of the
    two variants in one mapped lane-stream call equal their solo runs bit for bit: map poses, every row's record including `err`,
    registered clouds and both exports"""
    import torch
    import test_gpu_cube_edges as CE
    kw, dev, rel, counts, cubes, dense = _real_store(aloam, synth)
    blobs = [_variant(rel, counts, cubes, dense, extra) for extra in (False, True)]
    many = aloam.Aloam(max_batch=16, **kw)
    solo = aloam.Aloam(max_batch=1, **kw)
    try:
        run = CE._continue(aloam, many, [blobs[l % 2] for l in range(16)], dev,
                           torch.zeros((16 * N1 * 20000, 4), dtype=torch.float32, device="cuda"))
        for l in range(16):
            assert many.mapper_state(l)["centre"][0] == E.store_centre(rel)[0] + 1, l   # the first frame shifted once
        cap = min(16384, kw["max_points"])
        grown = len(many.mapper_cube(0, dense + 1, 0))   # (the shift towards high moved it one index up)
        assert grown > 2 * cap and len(many.mapper_cube(0, dense + 1, 1)) == 2 * cap
        refs = []
        for extra in (False, True):
            refs.append(CE._continue(aloam, solo, [blobs[extra]], dev,
                                     torch.zeros((N1 * 20000, 4), dtype=torch.float32, device="cuda")))
        for l in range(16):
            CE._same_lane(run, l, refs[l % 2], 0, "lane %d" % l)
        base, tight = run[2][0], run[2][1]
        assert not (base["flags"] & aloam.FLAG_CUBE_OVERFLOW).any() and not (base["err"] & 4).any()
        hit = np.flatnonzero(tight["flags"] & aloam.FLAG_CUBE_OVERFLOW)
        assert hit.size and (tight["err"][hit] & 4).all(), (tight["flags"], tight["err"])
    finally:
        many.close()
        solo.close()
