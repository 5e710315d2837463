"""CPU: the scenes and host models of the 128-wide scan-to-scan search tests (tests/wide_search_cases.py) do what
tests/test_gpu_wide_search.py relies on -- the vectorised association equals the literal loops and the oracle, the window scene
straddles its ring window, planted entries past the break indices are nearest and skipped, the refusal scenes are refused
only where claimed, and the asymmetric NEARBY_SCAN values are asymmetric exactly where claimed."""
import numpy as np
import pytest

import config_cases as K
import edge_scenes as es
import wide_search_cases as W

IDENT_Q, ZERO_T = np.array([0, 0, 0, 1.0]), np.zeros(3)


def _oracle_rows(orc, last, queries, thr, nearby):
    od = orc.Odometry(dist_sq_thresh=thr, nearby_scan=nearby)
    od.set_last(last, last)
    cc, pc, _ = od.associate(queries, queries, IDENT_Q, ZERO_T)
    return [(int(a), int(b), int(c), -1) for a, b, c in cc], [tuple(int(v) for v in r) for r in pc]


def test_64_ring_scenes_are_unchanged_by_the_width_parameter():
    """the scenes of test_gpu_config.py / test_gpu_search_edges.py are the explicit width=64 ones, byte for byte"""
    for seed in range(3):
        for a, b in zip(K.window_scene(seed), K.window_scene(seed, width=64, rcs=K.WINDOW_RCS)):
            assert a.tobytes() == b.tobytes()
        for a, b in zip(es.assoc_scene(seed), es.assoc_scene(seed, width=64)):
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
        a, b = es.search_clouds(np.random.default_rng(seed)), es.search_clouds(np.random.default_rng(seed), width=64)
        for name in a:
            assert all(x.tobytes() == y.tobytes() for x, y in zip(a[name], b[name])), name
    for n in K.NEARBY:
        assert all(K.window(rc, n) == K.window(rc, n, 64) for rc in range(64))


def _small_scenes():
    """(name, last, queries, nearby values): every small 128-wide scene of the GPU file, and the 64-wide window scene"""
    out = []
    last, q = K.window_scene(width=128, rcs=W.WIDE_RCS)
    out.append(("window128", last, q, 128, W.NEARBY))
    last, q = K.window_scene()
    out.append(("window64", last, q, 64, [2.5, 3.0 - 2.0 ** -48, 63.0, np.inf]))
    for name, last in W.break_scenes().items():
        out.append((name, last, last, 128, [1.0, 2.5, 127.0]))
    corner, _, p_start, _ = es.assoc_scene(seed=1, width=128)
    out.append(("assoc128", corner, es._pts(p_start), 128, [2.5]))
    return out


@pytest.mark.parametrize("case", range(len(_small_scenes())), ids=[s[0] for s in _small_scenes()])
def test_vectorised_associate_equals_the_loops_and_the_oracle(orc, case):
    name, last, queries, width, nearbys = _small_scenes()[case]
    n_rows = 0
    for nearby in nearbys:
        cc, pc = _oracle_rows(orc, last, queries, 25.0, nearby)
        for corner, want in ((True, cc), (False, pc)):
            loops = K.associate(last, queries, 25.0, nearby, corner)
            vec = W.associate(last, queries, 25.0, nearby, corner, width)
            assert vec == loops == want, (name, nearby, corner)
        n_rows += min(len(cc), len(pc))
    assert n_rows > 10, name


@pytest.mark.parametrize("nearby", W.NEARBY, ids=W.NEARBY_IDS)
def test_every_window_case_straddles_its_window_at_128(nearby):
    """each query's 2nd / 3rd point is the outermost in-window ring of its near side (or the clamp at 0 / 127), and wherever the
    ring just outside that window exists, it holds a point nearer to the query: a window one ring wider changes the answer"""
    last, queries = K.window_scene(width=128, rcs=W.WIDE_RCS)
    ring = W.rings_of(last)
    cc = K.associate(last, queries, 25.0, nearby, True)
    pc = K.associate(last, queries, 25.0, nearby, False)
    assert len(cc) == len(pc) == len(queries) == 2 * len(W.WIDE_RCS)
    for (i, j, m2, _), (_, _, _, m3) in zip(cc, pc):
        rc = int(ring[j])
        dn, up = K.window(rc, nearby, 128)
        forward = i % 2 == 0                       # side 0: the near side is forward
        edge = min(rc + up, 127) if forward else max(rc - dn, 0)
        other = max(rc - dn, 0) if forward else min(rc + up, 127)
        near = edge if (edge != rc) else other
        assert int(ring[m2]) in (edge, other) and int(ring[m3]) in (edge, other), (i, rc, ring[m2], ring[m3])
        assert near in (int(ring[m2]), int(ring[m3])), (i, rc)
        beyond = rc + up + 1 if forward else rc - dn - 1
        if 0 <= beyond <= 127:
            d = K.sqd(last, queries[i])
            assert d[ring == beyond].min() < min(d[m2], d[m3]), (i, rc, beyond)


def test_planted_entries_are_nearest_and_the_loops_skip_them():
    last, pairs = W.planted_scene()
    assert W.invariant_holds(W.rings_of(last))
    cc = {r[0]: r for r in K.associate(last, last, 25.0, 2.5, True)}
    pc = {r[0]: r for r in K.associate(last, last, 25.0, 2.5, False)}
    plants = {}
    for q, i in pairs:
        plants.setdefault(q, []).append(i)
    assert sorted(plants) and len(pairs) == 13
    for q, mine in plants.items():
        d = K.sqd(last, last[q])
        d[q] = np.inf
        others = np.setdiff1d(np.arange(len(last)), mine + [q])
        assert d[mine].max() < d[others].min(), q                       # nearer than every other point
        assert cc[q][1] == q and pc[q][1] == q
        assert not set(mine) & set(cc[q][2:]) and not set(mine) & set(pc[q][2:]), (q, mine, cc[q], pc[q])
        # a search that ignored the break indices would pick them
        wide = W.associate(last, last[q:q + 1], 25.0, 2.5, True, tables=(np.full(129, len(last)), np.zeros(129, np.int64)))
        assert wide[0][2] in mine, (q, wide)


def test_the_slot_carry_is_visible_only_in_the_ring_major_check():
    """The no-carry break tables differ from k_rab_scan's in every scene with an empty ring in a slot, yet no correspondence of a
    valid cloud changes: a point past the true break that the wider range lets in follows a ring of the slot above, so
    (int_i >= max_{j<i} int_j - 1) its own ring is at least the break ring and the ring slice drops it.  What the carry decides
    is the ring-major check: a three-ring drop whose ring r + 2 ends a slot and is absent passes without it."""
    for name, last in W.break_scenes().items():
        ring = W.rings_of(last)
        good, bad = W.break_tables(ring), W.break_tables(ring, carry=False)
        if len(np.unique(ring)) < 128:
            assert not (np.array_equal(good[0], bad[0]) and np.array_equal(good[1], bad[1])), name
        for nearby in (1.0, 2.5, 127.0):
            for corner in (True, False):
                assert (W.associate(last, last, 25.0, nearby, corner, tables=good)
                        == W.associate(last, last, 25.0, nearby, corner, tables=bad)), (name, nearby, corner)
    for name, (cloud, needs_carry) in W.refusal_scenes().items():
        ring = W.rings_of(cloud)
        assert not W.ring_major_ok(ring), name
        assert W.ring_major_ok(ring, tables=W.break_tables(ring, carry=False)) == needs_carry, name
        assert not W.invariant_holds(ring) or ring.max() > 127, name


def test_asymmetric_nearby_values_at_128():
    """by the double arithmetic of config_cases.window at W = 128, over the rings where W does not clamp the window"""
    def asym(n):
        return [rc for rc in range(3, 125) if K.window(rc, n, 128)[0] != K.window(rc, n, 128)[1]]
    assert asym(3.0 - 2.0 ** -48) == [30, 31, 32, 33, 34]
    assert asym(3.0 - 2.0 ** -47) == [62, 63, 64, 65, 66]                 # across the 63 / 64 boundary
    for k in range(1, 60):
        assert not [rc for rc in asym(3.0 - 2.0 ** -k) if rc >= 67], k    # rc +- N share an exponent there
    assert 3.0 - 2.0 ** -47 in W.NEARBY


def test_packed_words_at_the_bounds():
    """index << log2 W | ring as an int32: INT_MAX is the search's "no candidate", and the accepted bounds stay below it"""
    def packed(i, width):
        return (i << (7 if width == 128 else 6)) | (i * width // ((1 << 24) - 1 if width == 128 else (1 << 25) - 1))
    assert ((1 << 24) - 1) << 7 | 127 == 2 ** 31 - 1 and ((1 << 25) - 1) << 6 | 63 == 2 ** 31 - 1     # the refused sizes
    for width, n in ((128, (1 << 24) - 1), (64, (1 << 25) - 1)):
        assert packed(n - 1, width) < 2 ** 31 - 1 and (n - 1) * width // n == width - 1
        inf_from, single, ties = W.bound_sites(n, width)
        assert packed(inf_from, width) & 0x7F800000 == 0x7F800000
        words = np.array([packed(i, width) for i in single + [t[0] for t in ties]], np.int64).astype(np.int32)
        assert np.isnan(words.view(np.float32)).sum() >= 3 and all(i > 1 << 23 for i in single)
        assert all(late > early for late, early in ties)
