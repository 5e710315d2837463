"""CPU: the oracle's prior-map build (prior_build_cases.oracle_build: vectorised binning and pyoracle's VoxelGrid) against a
scalar numpy model of the
cube rule and the per-cube VoxelGrid, on the rule's edges; and snapshot_store_clouds on a hand-made snapshot."""
import struct

import numpy as np
import pytest

import prior_build_cases as P


def _same(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _check(corner, surf, line_res, plane_res, centre):
    m, dropped = P.oracle_build(corner, surf, line_res, plane_res, centre)
    got = m.packed()
    # the same cubes reach the oracle's frozen frames
    f = m.frozen()
    for (t, i), q in m.cubes.items():
        assert _same(f.cube(t, i), q)
    ref, ref_dropped = P.build_model(corner, surf, line_res, plane_res, centre)
    assert dropped == ref_dropped
    assert np.array_equal(got["cube_start"], ref["cube_start"])
    assert _same(got["corner"], ref["corner"]) and _same(got["surf"], ref["surf"])
    return got, dropped


def test_cube_rule_edges():
    # x + 25 == 0 goes to the centre cube, one float below to the cube before; -50 is the int() edge (cube centre - 2, not floor's - 1)
    assert P.cube_of(-25.0, 10) == 10
    assert P.cube_of(np.nextafter(np.float32(-25.0), np.float32(-100)), 10) == 9
    assert P.cube_of(-75.0, 10) == 8 and P.cube_of(np.nextafter(np.float32(-75.0), np.float32(0)), 10) == 9
    assert P.cube_of(25.0, 10) == 11 and P.cube_of(49975.0, -990) == 10 and P.cube_of(-50025.0, 1010) == 9
    assert P.cube_of(np.nan, 10) is None and P.cube_of(np.inf, 10) is None and P.cube_of(-np.inf, 10) is None
    assert P.cube_of(1e12, 10) is None and P.cube_of(-1e12, 10) is None


@pytest.mark.parametrize("leaves", [(0.2, 0.4), (0.4, 0.8), (0.7, 1.3)])
def test_build_on_the_cube_edges_equals_the_model(leaves):
    corner, surf = P.edge_clouds()
    got, dropped = _check(corner, surf, *leaves, (10, 10, 5))
    # every non-finite and beyond-int point is dropped, and the buffer's outer faces drop their outer side
    assert dropped[0] >= 3 * 3 * 5 and dropped[1] >= 3 * 3 * 5
    assert len(got["corner"]) > 0 and len(got["surf"]) > 0


@pytest.mark.parametrize("centre", [(-990, 10, 5), (1010, 10, 5), (10, -990, 1005), (2**20, -2**20, 5)])
def test_build_at_far_centres_equals_the_model(centre):
    pts = P.far_clouds()
    swapped = pts[:, [1, 0, 2, 3]].copy()
    _check(pts, swapped, 0.4, 0.8, centre)


def test_an_overflowing_cube_is_kept_in_input_order():
    rng = np.random.default_rng(3)
    c = rng.uniform(-24, 24, (200, 4)).astype(np.float32)
    got, _ = _check(c, c[:10], 0.001, 0.8, (10, 10, 5))
    assert _same(got["corner"], c)   # one cube, unfiltered, input order


def test_empty_clouds_give_an_empty_map():
    e = np.zeros((0, 4), np.float32)
    got, dropped = _check(e, e, 0.2, 0.4, (10, 10, 5))
    assert dropped == (0, 0) and len(got["corner"]) == len(got["surf"]) == 0 and not got["cube_start"].any()


def test_snapshot_store_clouds_splits_a_hand_made_snapshot(aloam):
    import test_lane_snapshot_format as F
    counts = np.full((2, P.NCUBE), -1, np.int32)
    counts[0, [3, 100, 4850]] = [5, 0, 17]
    counts[1, [3, 2000]] = [30, 1]
    blob = F._blob(counts=counts)
    got = aloam.snapshot_store_clouds(blob)
    b = np.frombuffer(blob, np.uint8)
    s = 256 + 16 * (40 + 90)
    pts = np.frombuffer(blob, np.float32, offset=s + P.STORE).reshape(-1, 4)
    # export order: corner 3 (5), surf 3 (30), corner 100 (0), corner 2000 - none, surf 2000 (1), corner 4850 (17)
    assert _same(got["corner"], np.concatenate([pts[0:5], pts[36:53]]))
    assert _same(got["surf"], np.concatenate([pts[5:35], pts[35:36]]))
    assert got["centre"] == struct.unpack_from("<3i", b, s) == (10, 10, 5)
    assert np.array_equal(got["counts"], counts)
    with pytest.raises(ValueError):
        aloam.snapshot_store_clouds(F._blob(mapped=False, nls=0, nlf=7, scan_index=1))
