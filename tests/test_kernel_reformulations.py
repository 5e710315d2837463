"""CPU models of two re-formulations the ring feature kernel (a-loam_b200/csrc/features.cu) relies on.  They restate the ARGUMENT,
not the kernel: the GPU parity tests compare the kernel itself with the oracle bit for bit.

1. Greedy picks (scanRegistration.cpp:282-398): the reference walks the six segments of a ring one after the other with ONE
   cloudNeighborPicked array (`sequential`).  The kernel walks them in parallel assuming no marks spill in from the previous
   segment, then re-walks them in parallel fixed-point rounds (`fixed_point`), where what a segment passes on is the marks of its
   own picks and the incoming marks that run past its end.  Claim: the two are equal.  `fixed_point_adjacent` passes on only a
   segment's own marks; it is wrong exactly on rings with a segment shorter than 5 positions past segment 0 (17..39 returns).
2. Per-ring VoxelGrid (scanRegistration.cpp:401-407): the kernel sorts EVERY in-range position by its absolute voxel coordinates
   before the picks are known and drops the picked positions afterwards.  Claim: the order equals PCL's sort by the voxel index
   relative to the bounding box of the surviving points (stable by position).
"""
import numpy as np
import pytest

ALPHABET = np.array([0.0, 0.05, 0.1, 0.2, 0.5, 1.0, 3.0], np.float32)


def walk_segment(curv, reach_b, reach_f, sp, ep, spill_in):
    """One segment: picks in the reference's order with `spill_in` (set of positions already marked).  Returns
    (less_sharp picks, flat picks, set of positions beyond ep marked by this segment's picks)."""
    picked = set(p for p in spill_in if sp <= p <= ep)
    spill_out = set()

    def mark(ind):
        for p in range(ind - reach_b[ind], ind + reach_f[ind] + 1):
            if sp <= p <= ep:
                picked.add(p)
            elif p > ep:
                spill_out.add(p)

    less = []
    order = sorted(range(sp, ep + 1), key=lambda i: (curv[i], i))
    for i in reversed(order):                       # largest curvature first, ties -> larger index
        if i in picked or not curv[i] > 0.1:
            continue
        if len(less) >= 20:
            break
        less.append(i)
        mark(i)
    flat = []
    for i in order:                                 # smallest first, ties -> smaller index
        if i in picked or not curv[i] < 0.1:
            continue
        flat.append(i)
        if len(flat) >= 4:
            break
        mark(i)
    return less, flat, spill_out


def bounds(n, w):
    s_loc, e_loc = 5, n - 6
    span = e_loc - s_loc
    return s_loc + span * w // 6, s_loc + span * (w + 1) // 6 - 1


def sequential(curv, rb, rf):
    """the reference: the six segments in order, one picked array for the whole ring"""
    n = len(curv)
    out, marked = [], set()
    for w in range(6):
        sp, ep = bounds(n, w)
        less, flat, spill = walk_segment(curv, rb, rf, sp, ep, marked)
        marked |= spill
        out.append((less, flat))
    return out


def _rounds(curv, rb, rf, publish):
    """the kernel's fixed-point rounds; publish(w, own, accepted) = the spill segment w passes on"""
    n = len(curv)
    res, own, assumed = [None] * 6, [set()] * 6, [set()] * 6
    for w in range(6):                              # speculative pass: nothing spills in
        sp, ep = bounds(n, w)
        less, flat, so = walk_segment(curv, rb, rf, sp, ep, set())
        res[w], own[w] = (less, flat), so
    rounds = 0
    while True:
        todo = []
        for w in range(1, 6):                       # all decisions of a round read the state of the previous round
            S, A = publish(w - 1, own[w - 1], assumed[w - 1]), assumed[w]
            if S == A:
                continue
            mine = set(res[w][0]) | set(res[w][1])
            hit = bool(A - S) or bool((S - A) & mine)
            moves = publish(w, own[w], S) != publish(w, own[w], A)   # accepting S without a walk changes what w passes on
            todo.append((w, S, hit, moves))
        if not any(h or m for _, _, h, m in todo):
            break
        rounds += 1
        new = {}
        for w, S, hit, _ in todo:
            if hit:
                sp, ep = bounds(n, w)
                new[w] = walk_segment(curv, rb, rf, sp, ep, S)
        for w, S, hit, _ in todo:
            assumed[w] = S
            if hit:
                less, flat, so = new[w]
                res[w], own[w] = (less, flat), so
        assert rounds <= 5
    return res, rounds


def fixed_point(curv, rb, rf):
    """the kernel: a segment passes on its own marks and the accepted incoming marks beyond its end"""
    n = len(curv)
    return _rounds(curv, rb, rf, lambda w, own, acc: own | {p for p in acc if p > bounds(n, w)[1]})


def fixed_point_adjacent(curv, rb, rf):
    """the kernel before marks passed through short segments: a segment passes on its own marks only"""
    return _rounds(curv, rb, rf, lambda w, own, acc: own)


def draw(seed, lo=17, hi=400, n=None):
    """a ring of n (or lo..hi-1) positions: curvatures from a coarse alphabet (many ties, many picks next to the segment
    boundaries) and random reaches of 0..5"""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(lo, hi)) if n is None else n
    return rng.choice(ALPHABET, size=n), rng.integers(0, 6, size=n), rng.integers(0, 6, size=n)


@pytest.mark.parametrize("seed", range(40))
def test_parallel_rewalk_rounds_equal_the_sequential_sweep(seed):
    curv, rb, rf = draw(seed)
    want = sequential(curv, rb, rf)
    got, rounds = fixed_point(curv, rb, rf)
    assert got == want
    if len(curv) >= 40:
        assert fixed_point_adjacent(curv, rb, rf)[0] == want


def test_the_rewalk_model_exercises_conflicts():
    hits = 0
    for seed in range(40):
        curv, rb, rf = draw(seed, 60, 400)
        hits += fixed_point(curv, rb, rf)[1] > 0
    assert hits >= 10          # the equality above is not vacuous


@pytest.mark.parametrize("n", range(17, 49))
def test_short_rings_every_size(n):
    """every ring of 17..48 returns (segments of 1..7 positions), 60 draws each: the pass-through rounds equal the sequential
    sweep; passing on only a segment's own marks differs from it for some draw at every size up to 39 and never from 40 on
    (from 40 every segment past the first holds at least 5 positions, so no mark runs past one)"""
    lens = [bounds(n, w)[1] - bounds(n, w)[0] + 1 for w in range(6)]
    assert (min(lens[1:]) < 5) == (n < 40)
    differ = 0
    for seed in range(60):
        curv, rb, rf = draw(1000 * n + seed, n=n)
        want = sequential(curv, rb, rf)
        assert fixed_point(curv, rb, rf)[0] == want, seed
        differ += fixed_point_adjacent(curv, rb, rf)[0] != want
    if n < 40:
        assert differ > 0
    else:
        assert differ == 0


def test_marks_run_through_four_one_position_segments():
    """17 returns: six segments of one position each.  A flat pick in segment 0 marks the next five positions, so the
    reference picks nothing in segments 1..5; the adjacent-only model sees the marks in segment 1 only and picks again in 2 and 4"""
    n = 17
    curv = np.zeros(n, np.float32)
    rb = np.zeros(n, int); rf = np.full(n, 5)
    want = sequential(curv, rb, rf)
    assert want == [([], [5])] + [([], [])] * 5
    assert fixed_point(curv, rb, rf)[0] == want
    assert fixed_point_adjacent(curv, rb, rf)[0] == [([], [5])] + [([], [])] + [([], [7])] + [([], [])] + [([], [9])] + [([], [])]


@pytest.mark.parametrize("seed", range(10))
def test_absolute_voxel_order_equals_pcl_relative_index_order(seed):
    rng = np.random.default_rng(100 + seed)
    n = 1500
    pts = (rng.normal(size=(n, 3)) * np.array([30.0, 30.0, 2.0])).astype(np.float32)
    keep = rng.random(n) > 0.1                      # "label <= 0": the picks are removed AFTER the sort in the kernel
    inv = np.float32(1.0) / np.float32(0.2)
    fl = np.floor(pts * inv).astype(np.int64)       # floorf(x * inverse_leaf)
    # PCL: bounding box of the surviving points -> relative index -> sort by (index, position)
    surv = np.nonzero(keep)[0]
    mn, mx = pts[surv].min(0), pts[surv].max(0)
    min_b = np.floor(mn * inv).astype(np.int64)
    div_b = np.floor(mx * inv).astype(np.int64) - min_b + 1
    rel = (fl[surv] - min_b)
    idx = rel[:, 0] + rel[:, 1] * div_b[0] + rel[:, 2] * div_b[0] * div_b[1]
    pcl_order = surv[np.lexsort((surv, idx))]
    # kernel: all positions by (z, y, x) absolute voxel coordinates then position, picked positions dropped afterwards
    key = ((fl[:, 2] + 65536) << 34) | ((fl[:, 1] + 65536) << 17) | (fl[:, 0] + 65536)
    all_order = np.lexsort((np.arange(n), key))
    mine = all_order[keep[all_order]]
    assert np.array_equal(mine, pcl_order)
    # and the voxel boundaries coincide
    assert np.array_equal(np.diff(key[mine]) != 0, np.diff(idx[np.argsort(surv)[np.searchsorted(np.sort(surv), pcl_order)]]) != 0)
