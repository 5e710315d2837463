"""CPU: the oracle of place recognition (oracle/place.cc) against the definitions of include/aloam_b200.h -- ring and sector edges,
the range cut, negative and signed-zero maxima, empty scans, skipped columns, tie rules for shifts and keyframes, rolled
descriptors, and the keyframe gate."""
import numpy as np
import pytest

import pyplace as P

TWO_PI = np.float32(6.28318548)


def _pts(*xyz):
    a = np.zeros((len(xyz), 4), np.float32)
    a[:, :3] = np.asarray(xyz, np.float32)
    return a


def _bin(d, r, s):
    return d[r * 60 + s]


def test_empty_scan_is_all_positive_zero():
    d = P.describe(np.zeros((0, 4)), np.zeros((0, 4)))
    assert d.shape == (1200,) and not np.signbit(d).any() and not d.any()


def test_ring_edges_and_range_cut():
    mr = np.float32(80.0)
    # r exactly 4 m is ring 1 ((4 * 20) / 80 = 1); just below is ring 0; r == max_range is dropped; just below is ring 19
    below = np.nextafter(np.float32(4.0), np.float32(0))
    top = np.nextafter(mr, np.float32(0))
    d = P.describe(_pts((4.0, 0, 1.0), (below, 0, 2.0), (80.0, 0, 3.0), (top, 0, 5.0), (100.0, 0, 7.0)), np.zeros((0, 4)), mr, 0.0)
    assert _bin(d, 1, 0) == 1.0 and _bin(d, 0, 0) == 2.0 and _bin(d, 19, 0) == 5.0
    assert np.count_nonzero(d) == 3


def test_sector_edges_and_negative_azimuth():
    # +y (pi / 2 in float: exactly the edge of sector 15) opens sector 15; -pi/2 lands in sector 45; y = -0 with x < 0 is -pi
    pts = _pts((0.0, 10.0, 1.0), (0.0, -10.0, 2.0), (-10.0, -0.0, 3.0), (-10.0, 0.0, 4.0), (10.0, 0.0, 5.0))
    d = P.describe(pts, np.zeros((0, 4)), 80.0, 0.0)
    assert _bin(d, 2, 15) == 1.0 and _bin(d, 2, 0) == 5.0
    assert _bin(d, 2, 45) == 2.0
    # atan2(+0, -10) = pi and atan2(-0, -10) = -pi, + 2 pi in float = pi: both in sector 30, which holds the larger
    assert _bin(d, 2, 30) == 4.0 and np.count_nonzero(d) == 4


def test_negative_maxima_and_signed_zero_order():
    # all points of a bin below zero: the bin holds the largest negative value, not the empty +0
    d = P.describe(_pts((10, 0, -3.0), (10.1, 0, -1.5)), np.zeros((0, 4)), 80.0, 0.0)
    assert _bin(d, 2, 0) == -1.5
    # -0 < +0: a bin of -0 and +0 holds +0 in either order; a bin of -0 alone holds -0
    for order in ([-0.0, 0.0], [0.0, -0.0]):
        d = P.describe(_pts(*[(10, 0, z) for z in order]), np.zeros((0, 4)), 80.0, 0.0)
        assert _bin(d, 2, 0) == 0.0 and not np.signbit(_bin(d, 2, 0))
    d = P.describe(_pts((10, 0, -0.0)), np.zeros((0, 4)), 80.0, -0.0)   # -0 + -0 = -0 (with +0 it would be +0)
    assert np.signbit(_bin(d, 2, 0))
    # z_offset is added in float before the maximum
    d = P.describe(_pts((10, 0, -2.0)), _pts((10, 0, -2.5)), 80.0, 2.0)
    assert _bin(d, 2, 0) == 0.0


def test_point_order_does_not_change_the_descriptor():
    rng = np.random.default_rng(3)
    a = (rng.normal(size=(3000, 4)) * 30).astype(np.float32)
    d0 = P.describe(a[:1000], a[1000:])
    p = rng.permutation(3000)
    assert np.array_equal(P.describe(a[p][:10], a[p][10:]).view(np.uint32), d0.view(np.uint32))


def test_zero_columns_are_skipped_and_all_skipped_is_one():
    q = np.zeros((20, 60), np.float32); d = np.zeros((20, 60), np.float32)
    assert P.distance(q, d) == (1.0, 0)
    q[3, 5] = 2.0
    assert P.distance(q, d) == (1.0, 0)   # no column pair has both norms non-zero
    d[7, 9] = 1.0                          # only shift 4 pairs column 5 with column 9: dot 0 -> dist 1 - 0 = 1
    D, s = P.distance(q, d)
    assert D == 1.0 and s == 0
    d[3, 9] = 1.0
    D, s = P.distance(q, d)
    assert s == 4 and D == 1.0 - (2.0 / (2.0 * np.sqrt(2.0)))


def test_shift_ties_take_the_smallest_shift():
    q = np.ones((20, 60), np.float32)
    D, s = P.distance(q, q)   # a constant descriptor matches equally at every shift
    assert s == 0
    # a descriptor with period 30 matches equally at s and s + 30
    rng = np.random.default_rng(1)
    half = rng.uniform(0, 5, (20, 30)).astype(np.float32)
    q = np.concatenate([half, half], axis=1)
    d = np.roll(q, 7, axis=1)
    D, s = P.distance(q, d)
    assert s == 7


def test_distance_ties_take_the_smallest_index():
    rng = np.random.default_rng(2)
    q = rng.uniform(0, 5, 1200).astype(np.float32)
    other = rng.uniform(0, 5, 1200).astype(np.float32)
    db = np.stack([other, q, other, q, q])
    idx, sh, dist = P.query(q[None], db, 5)
    assert list(idx[0][:3]) == [1, 3, 4] and list(idx[0][3:]) == [0, 2]
    assert dist[0][0] == dist[0][1] == dist[0][2]


@pytest.mark.parametrize("k", [0, 1, 13, 30, 59])
def test_rolled_descriptor_matches_at_its_shift(k):
    rng = np.random.default_rng(10 + k)
    q = rng.uniform(-1, 6, (20, 60)).astype(np.float32)
    q[:, rng.integers(0, 60, 5)] = 0.0   # a few empty columns
    d = np.roll(q, k, axis=1)
    D, s = P.distance(q, d)
    assert s == k
    for other in range(60):
        if other != k:
            Do, _ = P.distance(q, np.roll(q, other, axis=1))
            assert D <= Do


def test_gate():
    assert P.gate(None, [5, 5, 5], 100.0)
    assert P.gate([0, 0, 0], [3, 4, 0], 5.0)          # exactly at the gap
    assert not P.gate([0, 0, 0], [3, 4, 0], 5.0000001)
    assert P.gate([1, 1, 1], [1, 1, 1], 0.0)          # gap 0: every mapped row


def test_keyframe_table_records_and_loops():
    rng = np.random.default_rng(4)
    scans = [(rng.normal(size=(500, 4)) * 20).astype(np.float32) for _ in range(4)]
    T = P.KeyframeTable(lane=2, keyframe_gap=1.0, exclude_recent=1, max_keyframes=3)
    poses = [[0, 0, 0, 1, 0, 0, 0], [0, 0, 0, 1, 0.5, 0, 0], [0, 0, 0, 1, 2, 0, 0], [0, 0, 0, 1, 4, 0, 0], [0, 0, 0, 1, 9, 0, 0]]
    rows = [T.add(scans[i % 4][:100], scans[i % 4][100:], poses[i], i) for i in range(5)]
    assert [r["keyframe"] for r in rows] == [0, -1, 1, 2, -1]
    assert rows[4]["full"] == 1
    assert rows[2]["loop"] == -1 and rows[3]["loop"] in (0,)
    assert T.records["lane"].tolist() == [2, 2, 2] and T.records["scan_index"].tolist() == [0, 2, 3]
    T.add(scans[0][:100], scans[0][100:], poses[0], 0, start=True)
    assert len(T.records) == 1
