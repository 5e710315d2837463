"""CPU: the crafted scenes of the relocaliser's edge-case tests (tests/reloc_cases.py, used by tests/test_gpu_reloc_edges.py) have
the properties the GPU tests rely on: every scan point alone in its stack voxel (exact stack sizes and scoring-point counts), the
walk scenes' inlier alone in its cell at the flat walk index claimed, their d2 values, the 64-bit subsample indices, and the
oracle's score equal to the brute force and to the expected count."""
import numpy as np
import pytest

import prior_build_cases as PB
import pyoracle
import reloc_cases as RC

LEAVES = (0.2, 0.4)


def test_stage_pools_give_exact_stack_sizes():
    scan, _ = RC.stage_pool(*LEAVES)
    for t, leaf in enumerate(LEAVES):
        assert RC.alone_in_voxels(scan[t], leaf)
    for n_c, n_s, mp in RC.STAGE_CASES:
        stacks = [pyoracle.voxel_grid(scan[0][:n_c], LEAVES[0]), pyoracle.voxel_grid(scan[1][:n_s], LEAVES[1])]
        assert [len(s) for s in stacks] == [n_c, n_s]
        pts = RC.scoring_points(scan[0][:n_c], scan[1][:n_s], mp, *LEAVES)
        m_c = min(n_c, mp)
        assert len(pts[0]) == m_c and m_c % 32 and len(pts[0]) + len(pts[1]) in (31, 32, 33, 2047, 2048, 2049, 4096, 4097, 6145)
    assert sorted(min(a, c) + min(b, c) for a, b, c in RC.STAGE_CASES) == [31, 32, 33, 2047, 2048, 2049, 4096, 4097, 6145]


def test_the_big_stack_needs_64_bit_subsample_indices():
    (corner, surf), _ = RC.big_stack()
    assert RC.alone_in_voxels(surf, LEAVES[1]) and len(pyoracle.voxel_grid(surf, LEAVES[1])) == 60000
    n, m = 60000, 50000
    idx = RC.subsample_index(n, m)
    assert idx[-1] == (m - 1) * n // m and (np.arange(m, dtype=np.int64) * n > 2**31).sum() > m // 4
    wrapped = ((np.arange(m, dtype=np.int64) * n) & 0xFFFFFFFF).astype(np.int32).astype(np.int64) // m   # 32-bit products
    assert (wrapped != idx).sum() > m // 4 and (idx > 2**31 // n).any()


@pytest.mark.parametrize("scene", RC.WALK_SCENES, ids=lambda s: "lane%s-flat%d-of%d" % s)
def test_walk_scenes_put_the_inlier_where_they_claim(scene):
    lane, flat, total = scene
    s = RC.walk_scene(*scene)
    m, q = s["map"], s["query"]
    assert len(m) == total and RC.alone_in_voxels(m, RC.WALK_LEAF)
    assert (RC.cell_of(q) == RC.WALK_CELL).all()
    assert (s["lane"] >= 0).all() and (s["lane"] < 27).all()
    assert np.array_equal(np.bincount(s["lane"], minlength=27), s["counts"])
    thr = np.float32(s["inlier_sq"])
    inl = np.flatnonzero(s["d2"] < thr)
    assert (s["d2"] < np.float32(1.0)).all()
    if lane is None:
        assert len(inl) == 0
        expect = 0
    else:
        assert len(inl) == 1 and s["lane"][inl[0]] == lane and s["counts"][lane] == 1
        assert s["counts"][:lane].sum() == flat   # the flat walk index of a point alone in its cell
        expect = 1
    S = RC.FrozenScorer(PB.oracle_build(m, np.zeros((0, 4), np.float32), RC.WALK_LEAF, RC.WALK_LEAF)[0].frozen())
    assert len(S.clouds[0]) == total   # the map build keeps every point
    hyps = np.array([RC.IDENT7, RC.FAR_POSE])
    got = S.score(q, np.zeros((0, 4), np.float32), hyps, s["inlier_sq"], 1 << 20, RC.WALK_LEAF, RC.WALK_LEAF)
    assert got.tolist() == [expect, 0]
    assert np.array_equal(got, RC.brute_score(m, np.zeros((0, 4), np.float32), (q, np.zeros((0, 4), np.float32)), hyps, s["inlier_sq"]))


@pytest.mark.parametrize("below", [False, True])
def test_the_d2_edge_inside_a_dense_cell(below):
    s = RC.edge_walk_scene(below)
    thr = np.float32(RC.EDGE_WALK_SQ)
    assert RC.alone_in_voxels(s["map"], RC.WALK_LEAF)
    assert (s["lane"] == 14).sum() > 1000
    assert ((s["d2"] == thr) & (s["lane"] == 14)).sum() == 1
    assert ((s["d2"] == np.nextafter(thr, np.float32(0))) & (s["lane"] == 14)).sum() == int(below)
    assert (s["d2"] < thr).sum() == int(below) and (s["d2"] < np.float32(1.0)).all()
    empty = np.zeros((0, 4), np.float32)
    S = RC.FrozenScorer(PB.oracle_build(s["map"], empty, RC.WALK_LEAF, RC.WALK_LEAF)[0].frozen())
    got = S.score(s["query"], empty, np.array([RC.IDENT7]), RC.EDGE_WALK_SQ, 1 << 20, RC.WALK_LEAF, RC.WALK_LEAF)
    assert got.tolist() == [s["score"]]
    assert got.tolist() == RC.brute_score(s["map"], empty, (s["query"], empty), np.array([RC.IDENT7]), RC.EDGE_WALK_SQ).tolist()


def test_the_line_scene_grades_its_scores():
    scan, maps = RC.line_scene()
    shifts = [RC.shift(0.025 + 0.05 * k) for k in range(-9, 25)]
    got = RC.brute_score(maps[0], maps[1], scan, np.array(shifts), 0.25)
    assert len(set(got.tolist())) >= 8 and got.max() == 32
    S = RC.FrozenScorer(PB.oracle_build(maps[0], maps[1], *LEAVES)[0].frozen())
    assert np.array_equal(S.score(scan[0], scan[1], np.array(shifts), 0.25, 1 << 20, *LEAVES), got)
    assert RC.brute_score(maps[0], maps[1], scan, RC.FAR_POSE[None], 0.25).tolist() == [0]
    sc = np.array([0, 3, 0, 3, 5, 0, 1])
    assert RC.host_top(sc, 5).tolist() == np.lexsort((np.arange(7), -sc))[:5].tolist()
