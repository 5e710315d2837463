"""CPU: cube growth (aloam_set_cube_growth) without a GPU -- a numpy model of the run allocator and of the restore packing, the
snapshot header's cube_growth field and the store checks that depend on it (aloam_snapshot_check), and the prior-map tag layout."""
import struct

import numpy as np

import test_lane_snapshot_format as F

ERR_SNAPSHOT = -11
POOL, MAX_CUBE = 1024, 262144


def max_order(cap):
    """the largest run of a store, 2^k slabs: the largest power of two r <= 1024 with r x cap <= 2^18"""
    o = 0
    while o < 10 and cap << (o + 1) <= MAX_CUBE:
        o += 1
    return o


def run_order(n, cap):
    o = 0
    while cap << o < n:
        o += 1
    return o


class Pool:
    """one type's slab pool: an occupancy bitmap; take() = the lowest-address aligned free block of 2^o slabs"""

    def __init__(self):
        self.used = np.zeros(POOL, bool)

    def take(self, o):
        n = 1 << o
        for s in range(0, POOL, n):
            if not self.used[s:s + n].any():
                self.used[s:s + n] = True
                return s
        return -1

    def free(self, s, o):
        self.used[s:s + (1 << o)] = False


def pack(counts, cap):
    """restore packing: runs by decreasing size, cube order within a size; returns {cube: (first slab, order)} and the slabs used"""
    orders = {i: run_order(n, cap) for i, n in enumerate(counts) if n >= 0}
    out, base = {}, 0
    for o in sorted(set(orders.values()), reverse=True):
        for i in sorted(k for k, v in orders.items() if v == o):
            out[i] = (base, o)
            base += 1 << o
    return out, base


def test_max_orders_at_the_default_and_small_capacities():
    assert (max_order(16384), max_order(65536)) == (4, 2)   # 16 corner / 4 surf slabs
    assert max_order(2048) == 7 and (2048 << 7) == MAX_CUBE
    assert max_order(3000) == 6 and max_order(1) == 10


def test_allocator_model_runs_are_aligned_and_deterministic():
    p = Pool()
    assert [p.take(0) for _ in range(3)] == [0, 1, 2]
    assert p.take(2) == 4          # slabs 0-2 taken: the first aligned block of 4 starts at 4
    assert p.take(0) == 3          # the hole below it
    p.free(1, 0)
    assert p.take(1) == 8 and p.take(0) == 1
    # a fragmented pool: every other slab taken, so no run of 2 exists although half the pool is free
    q = Pool()
    q.used[::2] = True
    assert q.take(1) == -1 and q.take(0) == 1


def test_restore_packing_is_aligned_and_equals_the_slab_layout_without_growth():
    cap = 16384
    counts = np.full(4851, -1)
    counts[[5, 9, 40, 41, 300]] = [16384, 16385, 70000, 0, 40000]
    runs, used = pack(counts, cap)
    for i, (s, o) in runs.items():
        assert s % (1 << o) == 0 and (cap << o) >= counts[i]
    assert runs[40] == (0, 3) and runs[300] == (8, 2) and runs[9] == (12, 1) and runs[5] == (14, 0) and runs[41] == (15, 0)
    assert used == 8 + 4 + 2 + 1 + 1
    flat = np.full(4851, -1)
    flat[[3, 7, 4850]] = [1, 16384, 0]
    assert pack(flat, cap)[0] == {3: (0, 0), 7: (1, 0), 4850: (2, 0)}   # slabs 0, 1, 2, ... in cube order


def _growth(blob, g):
    b = bytearray(blob)
    struct.pack_into("<i", b, 220, g)
    return bytes(b)


def test_snapshot_cube_growth_field(aloam):
    blob = F._blob()
    assert F._code(aloam, blob) == 0 and F._code(aloam, _growth(blob, 1)) == 0
    for bad in (2, -1, 1 << 20):
        assert F._code(aloam, _growth(blob, bad)) == ERR_SNAPSHOT, bad


def _counts(corner=(), surf=()):
    c = np.full((2, F.NCUBE), -1, np.int32)
    for i, n in corner:
        c[0, i] = n
    for i, n in surf:
        c[1, i] = n
    return c


def test_counts_above_each_ceiling(aloam):
    """growth off: a count above the slab capacity is refused; growth on: up to the largest run's capacity (2^18 at the default
    capacities), one more is refused"""
    for n, off_ok, on_ok in ((16384, True, True), (16385, False, True), (MAX_CUBE, False, True), (MAX_CUBE + 1, False, False)):
        blob = F._blob(nls=0, nlf=0, counts=_counts(corner=[(7, n)]))
        assert (F._code(aloam, blob) == 0) == off_ok, n
        assert (F._code(aloam, _growth(blob, 1)) == 0) == on_ok, n
    blob = F._blob(nls=0, nlf=0, counts=_counts(surf=[(7, MAX_CUBE)]))
    assert F._code(aloam, blob) == ERR_SNAPSHOT and F._code(aloam, _growth(blob, 1)) == 0


def test_runs_that_overfill_the_pool(aloam):
    """63 corner cubes of 16 slabs (1008) + 16 single-slab cubes pack exactly into 1024 slabs; one more cube needs 1025"""
    big = [(i, 16 * 16384) for i in range(63)]
    small = [(100 + i, 1) for i in range(16)]
    blob = F._blob(nls=0, nlf=0, counts=_counts(corner=big + small))
    assert F._code(aloam, _growth(blob, 1)) == 0 and F._code(aloam, blob) == ERR_SNAPSHOT
    blob = F._blob(nls=0, nlf=0, counts=_counts(corner=big + small + [(200, 0)]))
    assert F._code(aloam, _growth(blob, 1)) == ERR_SNAPSHOT
    assert pack(_counts(corner=big + small)[0], 16384)[1] == 1024


def tag(i, j, k, rank):
    """prior_tag (kernels.h): i << 27 | j << 22 | k << 18 | rank, 32 bits unsigned"""
    return (i << 27) | (j << 22) | (k << 18) | rank


def untag(t):
    return t >> 27, (t >> 22) & 31, (t >> 18) & 15, t & 0x3FFFF


def test_prior_tag_round_trip():
    t = tag(20, 20, 10, (1 << 18) - 1)
    assert t < 1 << 32 and t >= 1 << 31   # i >= 16 sets bit 31: the tag is decoded unsigned
    assert untag(t) == (20, 20, 10, (1 << 18) - 1)
    word = np.array([t], np.uint32).view(np.float32).view(np.uint32)[0]   # stored in gpts.w as a float's bits
    assert untag(int(word)) == (20, 20, 10, (1 << 18) - 1)
    for i, j, k, r in ((0, 0, 0, 0), (15, 20, 10, 65536), (16, 0, 0, 1), (20, 0, 10, 123457)):
        assert untag(tag(i, j, k, r)) == (i, j, k, r)
