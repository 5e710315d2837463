"""CPU: the mapper's ring buffer at its decisions (laserMapping.cpp:142-146, :309-529, :741-758).  The crafted poses and points of
tests/cube_edge_cases.py straddle every decision of the cube rule; the host restatement there equals the oracle's cube store and
the reference's own laserMapping.cpp on every crafted path, and each plausible mis-transcription of the rule, the triggers and
the loop orders disagrees with it somewhere.  The lane-snapshot check refuses a store whose next frame could not end its shift."""
import numpy as np
import pytest

import cube_edge_cases as E
from test_lane_snapshot_format import _blob, _code

ERR_SNAPSHOT = -11


def _frames(name):
    return E.decision_paths().get(name) or E.jump_paths()[name]


def test_every_crafted_decision_is_straddled():
    for a in range(3):
        c = E.CEN0[a]
        for k in range(-c - 1, E.DIMS[a] - c + 1):
            lo, hi = E.straddle(50.0 * k - 25.0, c)
            assert np.nextafter(lo, np.inf) == hi and E.cube_coord(lo, c) + 1 == E.cube_coord(hi, c), (a, k)
            assert lo in E.decisions(a) and hi in E.decisions(a)
        (v2, v3), (v17, v18) = E.trigger_pairs(a)
        assert [E.cube_coord(v, c) for v in (v2, v3, v17, v18)] == [2, 3, E.DIMS[a] - 4, E.DIMS[a] - 3]
        for f in E.face_values(a):
            below, above = np.nextafter(f, E.F32(-np.inf)), np.nextafter(f, E.F32(np.inf))
            if f < -25:   # truncation: a negative face belongs to the cube below it
                assert E.cube_coord(below, c) == E.cube_coord(f, c) == E.cube_coord(above, c) - 1, (a, f)
            else:
                assert E.cube_coord(below, c) + 1 == E.cube_coord(f, c) == E.cube_coord(above, c), (a, f)
    # int() truncates towards zero: x = -75 lies in relative cube -2, x = -25 in cube 0 and its predecessor in cube -1
    assert (E.cube_coord(-75.0, 0), E.cube_coord(-25.0, 0), E.cube_coord(np.nextafter(-25.0, -np.inf), 0)) == (-2, 0, -1)
    assert E.cube_coord(-0.0, 0) == E.cube_coord(0.0, 0) == 0


def test_crafted_poses_and_points_land_on_their_decisions():
    """every frame of a decision path puts its pose exactly on its target, and its points include faces hit bit for bit"""
    rng = np.random.default_rng(5)
    for a in range(3):
        m = E.Model()
        for j, v in enumerate([v for v in E.decisions(a) if v != 0.0][::7]):
            q = E.ROT[j % 3]
            t = E.pose_for(m.T, q, v, a)
            x = E.associate(m.T, q, t)
            assert x[4 + a] == v
            m.frame(np.zeros((0, 4), E.F32), np.zeros((0, 4), E.F32), q, t)
        cloud, placed = E.face_frame(rng, x)
        w = E.to_map(cloud, x)
        on = {(ax, v) for ax, v in placed}
        assert len(on) > 100
        for ax, v in on:
            assert (w[:, ax] == E.F32(v)).any()


def test_every_face_holds_stored_points():
    """along the decision paths a stored point lies on every face of every axis inside the buffer -- the negative ones, where
    truncation and the < 0 test decide, included -- and on the float either side of each; no path needs more than the 1024
    slabs of a cloud type"""
    paths = E.decision_paths()
    assert E.faces_missed(paths) == set()
    for frames in paths.values():
        m, _ = E.run_model(frames)
        assert len(m.held()) <= 1024


@pytest.mark.parametrize("name", E.DECISION_PATHS + E.JUMP_PATHS)
def test_model_equals_oracle_and_reference(orc, name):
    """pose, T_wmap_wodom, centre, valid list and every cube (as sets: the store keeps a cube in voxel order) of the host model,
    the oracle's CubeMap and the reference's compiled laserMapping.cpp, on every frame of every crafted path"""
    from refsource import RefMapping, private_copy
    frames = _frames(name)
    try:
        ref = RefMapping(private_copy("libref_mapping.so", "cube_" + name), *E.LEAVES, orc.SORT_CANONICAL)
    except OSError as e:
        pytest.skip("oracle/_ref is not usable here: %r" % (e,))
    m, cm = E.Model(), orc.CubeMap()
    empty = np.zeros((0, 4), E.F32)
    for j, (q, t, surf) in enumerate(frames):
        assert E.distinct_voxels(surf, E.LEAVES[1])
        pose, st = m.frame(empty, surf, q, t)
        po, info = cm.step(empty, surf, q, t, *E.LEAVES)
        r = ref.process(empty, surf, surf, q, t, stamp=0.1 * (j + 1))
        assert np.array_equal(po, pose) and np.array_equal(r["pose"], pose) and not info["optimised"], j
        so = cm.state()
        assert so["centre"] == r["centre"] == st["centre"] and so["valid"] == st["valid"], j
        assert tuple(so["q_wmap_wodom"]) == m.T[0] and tuple(so["t_wmap_wodom"]) == m.T[1], j
        assert np.array_equal(r["q_wmap_wodom"], so["q_wmap_wodom"]) and np.array_equal(r["t_wmap_wodom"], so["t_wmap_wodom"]), j
        sizes = ref.sizes(1)
        held = {i for ty, i in m.held() if ty == 1}
        assert set(np.flatnonzero(sizes).tolist()) == held and int(sizes.sum()) == so["total_surf"], j
        for i in held:
            mine = E.as_set(m.cube(1, i))
            assert E.distinct_voxels(mine, E.LEAVES[1]), (j, i)
            assert np.array_equal(E.as_set(cm.cube(1, i)), mine) and np.array_equal(E.as_set(ref.cube(1, i, int(sizes[i]))), mine), (j, i)
    assert sum(len(f[2]) for f in frames) > 0


def _states(frames, mut=None):
    _, out = E.run_model(frames, mut)
    return [(st["centre"], st["valid"], {k: v.tobytes() for k, v in cubes.items()}) for _, st, cubes in out]


@pytest.mark.parametrize("mut", E.MUTATIONS)
def test_each_mis_transcription_disagrees_somewhere(mut):
    """floor for int(), <= for < 0, the decrement dropped, v + 25 in float, trigger <= 3 and the valid loop in k, j, i order each
    change a crafted frame.  The six shift loops in another axis order do not: shifts along different axes commute (each is a
    permutation of its lines plus the emptying of one plane), so the order is invisible in every result and is checked equal."""
    differs = False
    for frames in list(E.decision_paths().values()) + list(E.jump_paths().values()):
        if _states(frames) != _states(frames, mut):
            differs = True
            break
    if mut in E.RULE_MUTATIONS:
        rule = any(E.cube_coord(v, E.CEN0[a]) != E.cube_coord(v, E.CEN0[a], mut) for a in range(3) for v in E.decisions(a))
        assert rule or mut == "float_sum"
    assert differs == (mut != "axes_kji"), mut


@pytest.mark.parametrize("d", [(-8, 0, 0), (8, 0, 0), (0, -8, 0), (0, 8, 0), (0, 0, -3), (0, 0, 3), (4, -5, 2)])
def test_relabelled_store_runs_identically(d):
    """a store whose every cube and centre offset move by d gives the same poses, T and cubes (moved by d) -- as long as the
    points of both runs land inside the buffer and the cubes that scroll out are empty, which the crafted path here keeps"""
    rng = np.random.default_rng(31)
    frames = [(np.array(E.ROT[k % 3]), np.array([8.0 * k, -6.0 * k, 1.0 * k]), E.spread(rng, 40, [0, 0, 0], [30, 30, 8])) for k in range(6)]
    a = E.Model()
    b = E.Model(cen=tuple(E.CEN0[k] + d[k] for k in range(3)))
    off = d[0] + E.CW * d[1] + E.CW * E.CH * d[2]
    shifted = False
    for q, t, surf in frames:
        pa, sa = a.frame(np.zeros((0, 4), E.F32), surf, q, t)
        pb, sb = b.frame(np.zeros((0, 4), E.F32), surf, q, t)
        shifted |= sb["centre"] != tuple(E.CEN0[k] + d[k] for k in range(3))
        assert np.array_equal(pa, pb) and a.T == b.T and sa["dropped"] == sb["dropped"] == 0
        moved = {(ty, i + b.cen[0] - a.cen[0] + E.CW * (b.cen[1] - a.cen[1]) + E.CW * E.CH * (b.cen[2] - a.cen[2])) for ty, i in a.held()}
        assert moved == set(b.held())
        assert [v + (b.cen[0] - a.cen[0]) + E.CW * (b.cen[1] - a.cen[1]) + E.CW * E.CH * (b.cen[2] - a.cen[2]) for v in sa["valid"]] == sb["valid"]
    assert a.scrolled == b.scrolled == 0
    assert shifted == (d != (4, -5, 2)) and off != 0


# ---- the snapshot check: a store whose next frame could not end its ring-buffer shift is refused on the host

def _mapped():
    return bytearray(_blob(mapped=True))


def test_snapshot_check_refuses_out_of_range_centres_and_poses(aloam):
    """aloam_snapshot_check: the crafted blob (centre (10, 10, 5), T t = (1, 2, 3), world t = (3, -1, 0.25)) passes, and passes
    with its map position moved to the 16th cube outside the buffer on each side of each axis; one cube further, a non-finite or
    a ~1e12 m position, a centre offset beyond +-2^20 and a non-finite warm start, world pose or T_wmap_wodom are refused"""
    good = np.frombuffer(bytes(_mapped()), np.uint8)
    assert _code(aloam, good.tobytes()) == 0
    ok, bad = [], []
    for a in range(3):
        c, dim = E.CEN0[a], E.DIMS[a]
        for cube, refused in ((-16, False), (-17, True), (dim + 15, False), (dim + 16, True)):
            # T t on axis a so that world + t lies in the middle of centre cube `cube` (T's rotation is the identity)
            t = [1.0, 2.0, 3.0]
            t[a] = 50.0 * (cube - c) - (3.0, -1.0, 0.25)[a]
            (bad if refused else ok).append(E.with_store_fields(good, t_wmap=t))
    for cen in ((2 ** 20, 10, 5), (10, -(2 ** 20), 5)):
        ok.append(E.with_store_fields(good, cen=cen, t_wmap=[-50.0 * (cen[0] - 10), -50.0 * (cen[1] - 10), 3.0]))
    bad += [E.with_store_fields(good, cen=(2 ** 20 + 1, 10, 5)), E.with_store_fields(good, cen=(10, 10, -(2 ** 20) - 1)),
            E.with_store_fields(good, cen=(2 ** 31 - 1, 10, 5)), E.with_store_fields(good, t_wmap=(1e12, 2.0, 3.0)),
            E.with_store_fields(good, t_wmap=(1.0, np.inf, 3.0)), E.with_store_fields(good, t_wmap=(1.0, 2.0, np.nan)),
            E.with_store_fields(good, q_wmap=(0.0, 0.0, np.nan, 1.0)), E.with_store_fields(good, q_wmap=(0.0, 0.0, 1e300, 1e300)),
            E.with_store_fields(good, world=(0, 0, 0, 1.0, -np.inf, 0, 0)), E.with_store_fields(good, warm=(0, 0, 0, 1.0, np.nan, 0, 0)),
            E.with_store_fields(good, world=(0, 0, 0, 1.0, 1e11, 0, 0))]
    for k, b in enumerate(ok):
        assert _code(aloam, b.tobytes()) == 0, k
    for k, b in enumerate(bad):
        assert _code(aloam, b.tobytes()) == ERR_SNAPSHOT, k
    # an unmapped snapshot has no store: only its poses are checked
    plain = np.frombuffer(bytes(_blob(mapped=False)), np.uint8)
    assert _code(aloam, plain.tobytes()) == 0
    assert _code(aloam, E.with_store_fields(plain, world=(0, 0, 0, 1.0, 0, np.nan, 0)).tobytes()) == ERR_SNAPSHOT
