"""CPU: the crafted cases of tests/map_on_prior_edge_cases.py for mapping trajectories that start on a copy of the prior map.  Each
scene has the property the device tests rely on: the chunk-boundary cubes lie where the seed's table walk splits its chunks, the
slack doubles are adjacent and straddle the arming rule, the bit-exact scenes give a thin START frame on the seeded oracle.  And
the oracle's seeded CubeMap equals the reference's own laserMapping.cpp seeded the same way, bit for bit, on the START frame and
the next frames of every scene whose store the unbounded oracle models, both slack extremes included."""
import numpy as np
import pytest

import lane_refs as R
import map_on_prior_edge_cases as M

NCUBE = M.NCUBE


@pytest.fixture(scope="module")
def layout():
    return M.scene_layout()


def test_chunk_edges_land_where_the_table_walk_splits(layout):
    edges = M.chunk_edges()
    assert edges[0] == 0 and edges[-1] == NCUBE - 1 and M.PER == 5
    assert M.chunk_of(NCUBE - 1) == (970, 0)                 # thread 970 holds cube 4850 alone
    assert all(M.chunk_of(5 * t)[0] * M.PER >= NCUBE for t in range(971, 1024))   # threads 971 .. 1023 hold no cube
    for t in range(1, 971):
        assert M.chunk_of(5 * t - 1) == (t - 1, 4) and M.chunk_of(5 * t) == (t, 0)
    held = set(np.flatnonzero((layout.counts >= 0).any(0)))
    assert held == set(edges)
    kinds = {(bool(layout.counts[0, i] >= 0), bool(layout.counts[1, i] >= 0)) for i in edges}
    assert kinds == {(True, False), (False, True), (True, True)}   # corner-only, surf-only and both
    assert (layout.counts == 1).any(1).all()                        # one-point cubes of both types
    assert layout.cen != (10, 10, 5)
    assert all(n <= M.POOL for n in (layout.counts >= 0).sum(1))


def test_points_lie_in_their_cubes(layout):
    for (ty, idx), pts in layout.cubes.items():
        ijk = M.E.ijk_of(idx)
        for p in pts:
            assert tuple(M.E.cube_coord(float(p[a]), layout.cen[a]) for a in range(3)) == ijk, (ty, idx)


def test_slack_doubles_are_adjacent_and_straddle_the_arming_rule(layout):
    for cen in (layout.cen, (10, 10, 5), M.scene_pool(1).cen):
        for a, side, acc, ref in M.slack_inits(cen, layout.t):
            assert np.nextafter(acc[a], ref[a]) == ref[a] and acc[a] != ref[a], (a, side)
            assert M.fits(layout.counts, cen, acc, 20000) == "ok" and M.fits(layout.counts, cen, ref, 20000) == "invalid", (a, side)
            c = M.E.cube_coord(acc[a], cen[a])
            assert c == (-M.SLACK if side == "low" else M.DIMS[a] + M.SLACK - 1)


def test_the_arming_rule_on_the_crafted_scenes():
    for n, want in ((1023, "ok"), (1024, "ok"), (1025, "capacity")):
        s = M.scene_pool(n)
        assert (s.counts >= 0).sum(1).tolist() == [n, n] and M.fits(s.counts, s.cen, s.t, 20000) == want
    cases = ((0, 16384, 20000, "ok"), (0, 16384, 16384, "ok"), (0, 16385, 65536, "capacity"), (1, 65536, 65536, "ok"),
             (1, 65536, 65535, "capacity"), (1, 20000, 20000, "ok"), (1, 20001, 20000, "capacity"))
    for ty, n, maxpts, want in cases:
        counts = np.full((2, NCUBE), -1, np.int32)
        counts[ty, 7] = n
        assert M.fits(counts, (10, 10, 5), (0.0, 0.0, 0.0), maxpts) == want, (ty, n, maxpts)
    z = M.scene_zero()
    assert M.fits(z.counts, z.cen, z.t, 20000) == "ok" and (z.counts == 0).sum() == len(z.zeros)


def _odom(orc, synth, n):
    return R.oracle(orc, synth, M.edge_scans(synth, n), ("map-on-prior-edges", n), False)[0]


@pytest.mark.parametrize("name", ["layout", "zero", "pool_1024", "corner_16384", "surf_65536"])
def test_bit_exact_scenes_give_a_thin_start_frame(orc, synth, name):
    s = {"layout": M.scene_layout, "zero": M.scene_zero, "pool_1024": lambda: M.scene_pool(1024),
         "corner_16384": lambda: M.scene_capacity(0, 16384, True), "surf_65536": lambda: M.scene_capacity(1, 65536, True)}[name]()
    assert s.thin()
    T = M.normalised(s.q, s.t)
    cm = M.seeded_cubemap(orc, s, T)
    poses, infos = M.oracle_frames(orc, synth, cm, M.edge_scans(synth, 1), _odom(orc, synth, 1))
    assert not infos[0]["optimised"] and np.array_equal(poses[0], T)
    centre, valid = M.start_model(s, T)
    assert cm.state()["centre"] == centre and cm.state()["valid"] == valid


def test_slack_starts_are_thin_and_shift_past_the_seeded_cubes(orc, synth, layout):
    for a, side, acc, _ in M.slack_inits(layout.cen, layout.t):
        T = M.normalised(layout.q, acc)
        cm = M.seeded_cubemap(orc, layout, T)
        poses, infos = M.oracle_frames(orc, synth, cm, M.edge_scans(synth, 1), _odom(orc, synth, 1))
        assert not infos[0]["optimised"] and np.array_equal(poses[0], T)
        st = cm.state()
        assert (st["centre"], st["valid"]) == M.start_model(layout, T)
        shift = abs(st["centre"][a] - layout.cen[a])
        assert shift == 19, (a, side, shift)


def _ref(orc, tag):
    from refsource import RefMapping, private_copy
    try:
        return RefMapping(private_copy("libref_mapping.so", "edge_" + tag), *M.LEAVES, orc.SORT_CANONICAL)
    except OSError as e:
        pytest.skip("oracle/_ref is not usable here: %r" % (e,))


def _both(orc, synth, tag, s, T, n):
    """scans 0 .. n-1 on the oracle and the reference, both seeded with scene s at T: every frame bit for bit"""
    from map_on_prior_seed import seed_ref
    ref = _ref(orc, tag)
    seed_ref(ref, s.cen, T[:4], T[4:], s.counts, s.points())
    cm = M.seeded_cubemap(orc, s, T)
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    odom = _odom(orc, synth, n)
    for k, raw in enumerate(M.edge_scans(synth, n)):
        f = orc.Features(raw, ns, mr)
        po, _ = cm.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], *M.LEAVES)
        r = ref.process(f.less_sharp, f.less_flat, f.less_flat, odom[k, :4], odom[k, 4:], stamp=0.1 * (k + 1))
        so = cm.state()
        assert np.array_equal(po, r["pose"]) and so["centre"] == r["centre"], (tag, k)
        assert np.array_equal(so["q_wmap_wodom"], r["q_wmap_wodom"]) and np.array_equal(so["t_wmap_wodom"], r["t_wmap_wodom"]), (tag, k)
        for ty in range(2):
            sizes = ref.sizes(ty)
            assert int(sizes.sum()) == so["total_corner" if ty == 0 else "total_surf"], (tag, k, ty)
            for i in np.flatnonzero(sizes):
                assert np.array_equal(cm.cube(ty, int(i)), ref.cube(ty, int(i), int(sizes[i]))), (tag, k, ty, int(i))


@pytest.mark.parametrize("name", ["layout", "zero", "slack_low", "slack_high"])
def test_seeded_oracle_equals_the_seeded_reference(orc, synth, layout, name):
    s = M.scene_zero() if name == "zero" else layout
    t = s.t
    if name.startswith("slack"):
        inits = M.slack_inits(s.cen, s.t)
        t = inits[0][2] if name == "slack_low" else inits[1][2]
    _both(orc, synth, name, s, M.normalised(s.q, t), 4)


def test_the_crafted_snapshot_writer_round_trips():
    """crafted_blob (cube_edge_cases.with_store_fields) over a minimal mapped snapshot: the store reads back as written, the point
    total and the snapshot's size follow the payload"""
    import struct
    s = M.scene_zero()
    base = bytearray(256 + M.E.TABLE)
    struct.pack_into("<ii", base, 28, 0, 0)
    blob = M.crafted_blob(np.frombuffer(bytes(base), np.uint8), s.cen, s.counts, s.points(), (0.0, 0.0, 0.6, 0.8), (1.0, 2.0, 3.0))
    b = blob.tobytes()
    cubes, counts = M.split_store(blob)
    assert np.array_equal(counts, s.counts) and M.E.store_centre(blob) == s.cen
    assert all(np.array_equal(cubes[k], s.cubes[k]) for k in s.cubes) and set(cubes) == set(s.cubes)
    sec = 256 + M.E.TABLE
    assert struct.unpack_from("<q", b, 16)[0] == len(b) == sec + 16 * len(s.points())
    assert struct.unpack_from("<q", b, 256 + 39408)[0] == len(s.points())
    assert struct.unpack_from("<ii", b, 256 + 12)[0] == 0 and struct.unpack_from("<i", b, 256 + 528)[0] == 0
    assert struct.unpack_from("<7d", b, 256 + 536) == (0.0, 0.0, 0.6, 0.8, 1.0, 2.0, 3.0)


def test_the_full_pool_count_zero_scene():
    s = M.scene_zero_pool(96)
    assert ((s.counts >= 0).sum(1) == M.POOL).all() and ((s.counts > 0).sum(1) == M.POOL - 96).all()
    assert M.fits(s.counts, s.cen, s.t, 20000) == "ok" and s.thin()
