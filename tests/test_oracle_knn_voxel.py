"""CPU: oracle kd-tree (FLANN KDTreeSingleIndex restatement) vs brute force; voxel grid vs a numpy restatement of PCL."""
import numpy as np
import pytest
from hypothesis import example, given, settings, strategies as st


def _cloud(rng, n, scale=20.0):
    c = np.zeros((n, 4), np.float32)
    c[:, :3] = (rng.standard_normal((n, 3)) * scale).astype(np.float32)
    return c


@pytest.mark.parametrize("n,k", [(1, 1), (14, 5), (16, 5), (1000, 1), (5000, 5), (20000, 8)])
def test_kdtree_matches_bruteforce(orc, n, k):
    rng = np.random.default_rng(n * 7 + k)
    cloud = _cloud(rng, n)
    q = _cloud(rng, 300)
    idx, sqd = orc.KdTree(cloud).knn(q, k)
    ridx, rsqd = orc.bruteforce_knn(cloud, q, k)
    assert np.array_equal(idx, ridx) and np.array_equal(sqd, rsqd)


def test_kdtree_ties_by_index(orc):
    cloud = np.zeros((64, 4), np.float32)
    cloud[:, 0] = np.repeat(np.arange(8), 8)      # lattice with many duplicate points / equal distances
    cloud[:, 1] = np.tile(np.arange(8), 8) // 2
    q = np.array([[3.5, 1.5, 0, 0], [0, 0, 0, 0]], np.float32)
    idx, sqd = orc.KdTree(cloud).knn(q, 6)
    ridx, rsqd = orc.bruteforce_knn(cloud, q, 6)
    assert np.array_equal(idx, ridx) and np.array_equal(sqd, rsqd)


@settings(max_examples=40, deadline=None)
@given(st.integers(1, 400), st.integers(1, 6), st.integers(0, 2 ** 31 - 1))
@example(264, 1, 48329025)   # every point at the origin: the far query's box bound rounds above the points' equal distances
def test_kdtree_property(n, k, seed):
    import pyoracle as orc
    rng = np.random.default_rng(seed)
    cloud = _cloud(rng, n, scale=rng.uniform(0.01, 100))
    cloud[:, :3] = np.round(cloud[:, :3], rng.integers(0, 4))   # force coincident coordinates / ties
    q = _cloud(rng, 20, scale=50)
    idx, sqd = orc.KdTree(cloud).knn(q, k)
    ridx, rsqd = orc.bruteforce_knn(cloud, q, k)
    assert np.array_equal(idx, ridx) and np.array_equal(sqd, rsqd)


def _voxel_numpy(cloud, leaf):
    """pcl::VoxelGrid::applyFilter in numpy float32 (SURVEY.md 8a 'V'), ties by point index"""
    inv = np.float32(1.0) / np.float32(leaf)
    xyz = cloud[:, :3]
    mn, mx = xyz.min(0), xyz.max(0)
    min_b = np.floor(mn * inv).astype(np.int64)
    div = np.floor(mx * inv).astype(np.int64) - min_b + 1
    ijk = (np.floor(xyz * inv) - min_b.astype(np.float32)).astype(np.int64)
    idx = ijk[:, 0] + ijk[:, 1] * div[0] + ijk[:, 2] * div[0] * div[1]
    order = np.lexsort((np.arange(len(idx)), idx))
    out = []
    i = 0
    while i < len(order):
        j = i
        s = np.zeros(4, np.float32)
        while j < len(order) and idx[order[j]] == idx[order[i]]:
            s = s + cloud[order[j]]
            j += 1
        out.append(s / np.float32(j - i))
        i = j
    return np.array(out, np.float32)


@pytest.mark.parametrize("leaf", [0.2, 0.4, 0.8])
def test_voxel_grid(orc, leaf):
    rng = np.random.default_rng(int(leaf * 10))
    cloud = _cloud(rng, 3000, scale=3.0)
    cloud[:, 3] = rng.uniform(0, 64, 3000).astype(np.float32)
    got = orc.voxel_grid(cloud, leaf, orc.SORT_CANONICAL)
    assert np.array_equal(got, _voxel_numpy(cloud, leaf))
    lit = orc.voxel_grid(cloud, leaf, orc.SORT_LITERAL)
    assert lit.shape == got.shape and np.abs(lit - got).max() < 1e-4
    assert orc.voxel_grid(np.zeros((0, 4), np.float32), leaf).shape == (0, 4)


def test_voxel_grid_overflow_returns_input(orc):
    """leaf too small for the extent: PCL warns and returns the input unchanged"""
    cloud = np.array([[0, 0, 0, 1], [3000, 3000, 3000, 2], [1, 1, 1, 3]], np.float32)
    assert np.array_equal(orc.voxel_grid(cloud, 0.2), cloud)
