"""Scenes of short dense rings for the ring feature kernel, and the CPU checks that make them count.  TEST INFRASTRUCTURE.

A ring of 17..39 returns has a segment shorter than 5 positions past its first one, so a pick's marks can run past that
segment into the ones after it.  The reference (scanRegistration.cpp:282-398) walks the six segments in order with one
cloudNeighborPicked array, so such marks reach them.  The scenes put these rings on dense arcs (consecutive returns under
0.22 m apart, so every pick marks 5 positions) and the checks show, on the oracle's own curvatures and reaches, that the
sequential model of test_kernel_reformulations gives the oracle's labels on every ring while passing on only a segment's own
marks (fixed_point_adjacent) does not on at least one: a scene that passes on the device pins the pass-through."""
import numpy as np

import edge_scenes as es
import pyoracle as orc
from test_kernel_reformulations import fixed_point_adjacent, sequential

SIZES = list(range(16, 49))                                   # 16 (skipped: end - start = 5) .. 48
FIELD_RINGS = SIZES + [600] * 7                               # 40 driver rings: 33 short ones and 7 whole turns
ELEVATION = {   # n_scans -> (counts, scale of the room): short dense rings among whole turns, the ring-skip edge included
    16: ([600, 600, 600, 17, 20, 22, 23, 28, 29, 34, 35, 39, 40, 41, 600, 600], 1.0),
    32: ([600] * 6 + list(range(16, 42)), 1.0),
    64: ([0] + [600] * 3 + [17 + (r * 5) % 32 for r in range(4, 47)] + [600] * 4 + [0] * 13, 2.0),   # rings 51..63 never fill
}
MIN_RANGE = {16: 0.3, 32: 0.3, 64: 5.0}


def wide_counts():
    """128 driver rings: 8 whole turns, then 120 short rings cycling through 17..48 returns"""
    return [600] * 8 + [17 + (r * 7) % 32 for r in range(120)]


def wide_styles():
    return [es.DENSE_STYLES[r % 3] for r in range(128)]


def field_scan(style, shift=(0.0, 0.0)):
    return es.short_ring_scan(FIELD_RINGS, style, shift=shift)


def wide_scan():
    return es.short_ring_scan(wide_counts(), wide_styles())


# (style, sensor motion per frame in metres) of the 40-ring trajectories: the first for the odometry chain, the other two as
# the two trajectories of a batch
TRAJECTORIES = [("zigzag", (0.06, -0.03)), ("smooth", (0.05, 0.02)), ("dyadic", (-0.04, 0.05))]
FRAMES = 5


def trajectory_scan(traj, k):
    style, (dx, dy) = TRAJECTORIES[traj]
    return field_scan(style, shift=(k * dx, k * dy))


def elevation_scan(ns, style):
    counts, scale = ELEVATION[ns]
    dense = [r for r, n in enumerate(counts) if 0 < n < 64]
    return es.room_scan(counts, dense=dense, dense_style=style, n_scans=ns, scale=scale)


def oracle(raw, ns, mode):
    """the oracle's features (SORT_CANONICAL): mode 'elevation', 'field' (up to 64 driver rings) or 'wide' (up to 128)"""
    if mode == "elevation":
        return orc.Features(raw, ns, MIN_RANGE[ns], orc.SORT_CANONICAL)
    if mode == "field":
        import ring_field_oracle as RF
        return RF.Features(raw, ns, 0.3)
    import wide_ring_oracle as WR
    return WR.Features(raw, ns, 0.3)


def ring_labels(picks, n):
    """labels of a ring from per-segment (less_sharp, flat) picks: 2 for the first two sharp picks of a segment, 1 for the
    rest, -1 for flat picks"""
    lab = np.zeros(n, np.int64)
    for less, flat in picks:
        for i, p in enumerate(less):
            lab[p] = 2 if i < 2 else 1
        for p in flat:
            lab[p] = -1
    return lab


def ring_inputs(ref, r):
    """(first index, n, curvatures as the models take them, backward and forward reach) of ring r of the oracle's cloud"""
    rings = ref.full[:, 3].astype(np.int32)
    a, b = int(np.searchsorted(rings, r)), int(np.searchsorted(rings, r + 1))
    n = b - a
    curv = np.zeros(n, np.float32)
    if n >= 17:
        curv[5:n - 6] = ref.curvature[a + 5:b - 6]
    rb, rf = es.suppression_reach(ref.full[a:b])
    return a, n, curv, rb, rf


def adjacent_misses(ref, ns):
    """rings where passing on only a segment's own marks gives other labels than the oracle; asserts that the sequential
    sweep (one picked array per ring) gives the oracle's labels on every ring of 17 returns or more"""
    miss = []
    for r in range(ns):
        a, n, curv, rb, rf = ring_inputs(ref, r)
        if n < 17:
            continue
        want = ref.label[a:a + n].astype(np.int64)
        assert np.array_equal(ring_labels(sequential(curv, rb, rf), n), want), r
        if not np.array_equal(ring_labels(fixed_point_adjacent(curv, rb, rf)[0], n), want):
            miss.append(r)
    return miss


def dense_rings(ref, ns, below=64):
    """rings of 17..below-1 returns in the oracle's cloud whose picks reach 5 positions forward everywhere in the segments"""
    out = []
    for r in range(ns):
        a, n, curv, rb, rf = ring_inputs(ref, r)
        if 17 <= n < below and (rf[5:n - 6] == 5).all():
            out.append(r)
    return out
