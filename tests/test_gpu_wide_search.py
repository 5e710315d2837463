"""GPU parity at the edges of the 128-wide scan-to-scan searches (k_rab_scan<128>, k_rab_fill<128>, k_ring_offsets<128>,
k_odom_assoc<128>, k_knn_last<128>) in contexts of aloam_create_wide with 65, 96 and 128 rings: exact nearest neighbours and
correspondences on rings 0..127, ring windows that end on both sides of every 32-ring slot boundary, break tables across the
slots, refusals, real wide scan pairs, and the packed index (index << 7 | ring) at the largest max_points it takes.  Scenes and
host models: tests/wide_search_cases.py (checked on the CPU by tests/test_oracle_wide_search.py)."""
import numpy as np
import pytest

import config_cases as K
import edge_scenes as es
import wide_ring_oracle as WR
import wide_search_cases as W
from test_gpu_search_edges import WARM, _dups

pytestmark = pytest.mark.gpu

IDENT_Q, ZERO_T = np.array([0, 0, 0, 1.0]), np.zeros(3)
ERR_NOT_RING_MAJOR = -8


def _wide(aloam, ns, max_points=20000, **kw):
    return aloam.Aloam(n_scans=ns, max_points=max_points, ring_source=aloam.RING_FIELD, wide=True, **kw)


@pytest.fixture(scope="module")
def ctxs(aloam):
    out = {(ns, d): _wide(aloam, ns, distortion=d) for ns in W.N_SCANS for d in (0, 1)}
    yield out
    for c in out.values():
        c.close()


def _rows(gcc, gpc):
    return [(i, a, b) for i, (a, b, v) in enumerate(gcc) if v], [(i, a, b, c) for i, (a, b, c, v) in enumerate(gpc) if v]


def _assoc(ctx, orc, corner, surf, sharp, flat, q, t, distortion=0, nearby=2.5, tag=""):
    """the device's correspondences equal Odometry.associate's exactly (query, closest, 2nd[, 3rd])"""
    od = orc.Odometry(distortion=bool(distortion), nearby_scan=nearby)
    od.set_last(corner, surf)
    cc, pc, _ = od.associate(sharp, flat, q, t)
    ctx.odometry_set_last(corner, surf)
    got = _rows(*ctx.odometry_associate(sharp, flat, q, t))
    want = ([tuple(int(v) for v in r) for r in cc], [tuple(int(v) for v in r) for r in pc])
    for g, w, kind in zip(got, want, ("corner", "surf")):
        if g != w:
            diff = [(x, y) for x, y in zip(g, w) if x != y][:4]
            pytest.fail("%s nearby=%r distortion=%d: %s rows differ (%d vs %d), first (got, expected): %s"
                        % (tag, nearby, distortion, kind, len(g), len(w), diff))
    return want


# ------------------------------------------------------------------------------------------------ 1. nearest neighbour
@pytest.mark.parametrize("name", ["uniform", "one_point", "one_azimuth", "dense_cells"])
def test_knn_exact_on_rings_up_to_127(ctxs, orc, name):
    """rab_nearest<128> with no distance limit == float32 brute force bit for bit, rings drawn from 0..127 (the 1000-point cell
    on ring 104, the sweep round the whole circle for one_azimuth)"""
    cloud, q = es.search_clouds(np.random.default_rng(3), width=128)[name]
    assert int(cloud[:, 3].max()) >= 64 or name == "one_point"
    ridx, rsqd = orc.bruteforce_knn(cloud, q, 1)
    for ns in W.N_SCANS:
        ctx = ctxs[(ns, 0)]
        ctx.odometry_set_last(cloud, cloud)
        for which in (0, 1):
            idx, sqd = ctx.knn(which, q, 1)
            assert np.array_equal(idx, ridx) and np.array_equal(sqd, rsqd), (name, ns, which)


# ------------------------------------------------------------------------------------------------ 2. association under warm starts
@pytest.mark.parametrize("distortion", [0, 1])
@pytest.mark.parametrize("warm", range(len(WARM)))
def test_association_edges_exact_at_128(ctxs, orc, warm, distortion):
    """test_gpu_search_edges.test_association_edges_exact on assoc_scene(width=128): ties in all three points, sweeps that grow
    or wrap past +-pi, current rings 0..127, and edge sites whose closest point is on ring 0, 127, 63 or 64"""
    ns = W.N_SCANS[warm]
    corner, surf, p_start, tags = es.assoc_scene(seed=warm, width=128)
    yaw, t = WARM[warm]
    q = es.quat([0, 0, 1], yaw); t = np.array(t, np.float64)
    rng = np.random.default_rng(10 + warm)
    frac = rng.uniform(0.09, 0.0999, len(p_start)) if distortion else 0.05
    cur = es.to_current_frame(p_start, q, t, rng.integers(0, 128, len(p_start)), frac)
    perm = np.argsort(cur[:, 3].astype(np.int32), kind="stable")
    cur, tags = cur[perm], tags[perm]
    cc, pc = _assoc(ctxs[(ns, distortion)], orc, corner, surf, cur, cur, q, t, distortion, tag="warm%d" % warm)
    assert len(cc) >= 20 and len(pc) >= 20
    if distortion:
        return
    rows = {r[0]: r for r in cc}
    edge = [i for i in np.flatnonzero(tags == "edge") if i in rows]
    assert {int(corner[rows[i][1], 3]) for i in edge} == {0, 63, 64, 127}
    tie = [i for i in np.flatnonzero(tags == "tie") if i in rows]
    assert sum(len(_dups(corner, rows[i][2])) > 0 for i in tie) >= 10


# ------------------------------------------------------------------------------------------------ 3. ring windows
@pytest.mark.parametrize("nearby", W.NEARBY, ids=W.NEARBY_IDS)
@pytest.mark.parametrize("distortion", [0, 1])
def test_ring_windows_at_128(aloam, orc, nearby, distortion):
    """window_scene(width=128): for rc in {0, 1, 31..33, 63..65, 95..97, 126, 127} nearer points sit just outside the window
    on the near side, so a window one ring off either way changes the 2nd / 3rd point"""
    ns = W.N_SCANS[W.NEARBY.index(nearby) % 3]
    last, queries = K.window_scene(width=128, rcs=W.WIDE_RCS)
    ctx = _wide(aloam, ns, nearby_scan=nearby, distortion=distortion)
    try:
        cc, pc = _assoc(ctx, orc, last, last, queries, queries, IDENT_Q, ZERO_T, distortion, nearby, "window")
    finally:
        ctx.close()
    assert len(cc) == len(pc) == len(queries)
    if nearby >= 127:   # up < W, not up < 64: from rc = 0 the window reaches ring 127
        assert int(last[cc[0][2], 3]) == 127 and int(last[cc[0][1], 3]) == 0


# ------------------------------------------------------------------------------------------------ 4. break tables across the slots
@pytest.mark.parametrize("scene", sorted(W.break_scenes()))
@pytest.mark.parametrize("distortion", [0, 1])
def test_break_tables_across_the_slots(aloam, orc, scene, distortion):
    """clouds that descend by one at every ring change (32 -> 31, 64 -> 63, 96 -> 95) with entries past the break indices
    nearer than every in-window candidate, empty-ring runs 20..40 and 60..100, and clouds of rings {0, 127}, {31, 32},
    {63, 64}; the queries are the points themselves and the points moved by ~5 cm, at identity and a moved pose"""
    last = W.break_scenes()[scene]
    rng = np.random.default_rng(7)
    queries = np.ascontiguousarray(np.concatenate([last, last + rng.normal(0, 0.05, last.shape).astype(np.float32) * [1, 1, 1, 0]]),
                                   np.float32)
    moved = np.array([0, 0, 0.01, 0.99995]); moved /= np.linalg.norm(moved)
    total = 0
    for k, nearby in enumerate((1.0, 2.5, 127.0)):
        ctx = _wide(aloam, W.N_SCANS[k], nearby_scan=nearby, distortion=distortion)
        try:
            for q, t in ((IDENT_Q, ZERO_T), (moved, np.array([0.05, 0.0, 0.0]))):
                cc, pc = _assoc(ctx, orc, last, last, queries, queries, q, t, distortion, nearby, scene)
                total += len(cc) + len(pc)
                if scene == "planted" and nearby == 2.5 and not np.any(t):
                    for qi, planted in W.planted_scene()[1]:
                        row = [r for r in cc if r[0] == qi] + [r for r in pc if r[0] == qi]
                        assert len(row) == 2 and all(r[1] == qi and planted not in r[2:] for r in row), (qi, row)
        finally:
            ctx.close()
    assert total > 100


def test_refused_clouds_leave_no_trace(aloam, orc):
    """-8 for a two-ring drop across a slot boundary (65 then 63), a run 65, 64, 63, int(intensity) 128, and three-ring drops
    32 -> 29 / 64 -> 61 / 96 -> 93 where ring 31 / 63 / 95 is absent (only the carry across the slots catches those), as corner
    or as surf cloud; afterwards the context associates as a fresh one"""
    good = W.break_scenes()["planted"]
    used, fresh = _wide(aloam, 128), _wide(aloam, 128)
    try:
        for name, (bad, _) in W.refusal_scenes().items():
            for pair in ((good, bad), (bad, good)):
                with pytest.raises(aloam.AloamError) as e:
                    used.odometry_set_last(*pair)
                assert e.value.code == ERR_NOT_RING_MAJOR, name
        q = np.array([0, 0, 0.004, 1.0]); q /= np.linalg.norm(q); t = np.array([0.05, 0, 0.0])
        for c in (used, fresh):
            c.odometry_set_last(good, good)
        a, b = used.odometry_associate(good, good, q, t), fresh.odometry_associate(good, good, q, t)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[0][:, 2].sum() > 100
    finally:
        used.close(); fresh.close()


# ------------------------------------------------------------------------------------------------ 5. real wide pairs
@pytest.mark.parametrize("sensor,reverse,distortion", [("OS128", False, 0), ("OS128", True, 1), ("V128", False, 1), ("V128", True, 0),
                                                       ("L96", False, 0), ("L96", True, 1), ("E65", False, 1), ("E65", True, 0)])
def test_correspondences_of_real_wide_pairs(aloam, orc, synth, sensor, reverse, distortion):
    """scans 1 -> 2 of the wide tables at the oracle chain's warm pose (its registration of scan 1 on scan 0): every corner and
    surf correspondence equals the oracle's"""
    ns = WR.n_rings(synth, sensor)
    f = [WR.Features(WR.scan(synth, sensor, k, reverse=reverse), ns, synth.RING_RANGES[0]) for k in range(3)]
    od = orc.Odometry(distortion=bool(distortion))
    od.set_last(f[0].less_sharp, f[0].less_flat)
    q, t, _ = od.register(f[1].sharp, f[1].flat, np.array([0, 0, 0, 1.0]), np.zeros(3))
    assert float(np.abs(t).max()) > 0.01
    ctx = _wide(aloam, ns, max(len(x.less_flat) for x in f) + 1024, distortion=distortion)
    try:
        cc, pc = _assoc(ctx, orc, f[1].less_sharp, f[1].less_flat, f[2].sharp, f[2].flat, q, t, distortion, tag=sensor)
    finally:
        ctx.close()
    assert len(cc) > 100 and len(pc) > 300
    rings = {int(f[1].less_flat[r[1], 3]) for r in pc}
    assert max(rings) >= 64


# ------------------------------------------------------------------------------------------------ 6. the packed index at its bounds
BYTES_PER_POINT = 430     # create_ctx's buffers per point of max_points for one lane (arithmetic from its allocations)


def bound_case(aloam, orc, width, n, max_points=None):
    """a ring-major cloud of n points in a context of max_points (default n) and `width` rings (nearby_scan = inf, so that
    every ring is in the window): aloam_knn and aloam_odometry_associate against brute force and wide_search_cases.associate.
    Returns a list of mismatches (empty when the device is exact)."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    need = BYTES_PER_POINT * (max_points or n) + (2 << 30)
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 1e9, free / 1e9))
    cloud = W.bound_cloud(n, width)
    queries, want = W.plant_bounds(cloud, width)
    ridx, rsqd = orc.bruteforce_knn(cloud, queries, 1)
    assert np.array_equal(ridx[:, 0], want)                         # the planted points are the nearest ones
    tables = W.break_tables(W.rings_of(cloud), width)
    want_c = W.associate(cloud, queries, 25.0, np.inf, True, width, tables)
    want_p = W.associate(cloud, queries, 25.0, np.inf, False, width, tables)
    assert want_c[0][1:3] == (0, n - 1) and want_p[0][3] == n - 1       # the largest forward rank
    kw = dict(ring_source=aloam.RING_FIELD, wide=True) if width == 128 else {}
    ctx = aloam.Aloam(n_scans=width, max_points=max_points or n, max_batch=1, nearby_scan=np.inf, **kw)
    bad = []
    try:
        ctx.odometry_set_last(cloud, cloud)
        for which in (0, 1):
            idx, sqd = ctx.knn(which, queries, 1)
            bad += [("knn", which, int(i), int(g), int(w)) for i, (g, w) in enumerate(zip(idx[:, 0], ridx[:, 0])) if g != w]
            bad += [("knn d2", which)] if not np.array_equal(sqd, rsqd) and not bad else []
        got_c, got_p = _rows(*ctx.odometry_associate(queries, queries, IDENT_Q, ZERO_T))
        want_c = [r[:3] for r in want_c]
        bad += [("corner", g, w) for g, w in zip(got_c, want_c) if g != w] + ([("corner rows", len(got_c), len(want_c))] if len(got_c) != len(want_c) else [])
        bad += [("surf", g, w) for g, w in zip(got_p, want_p) if g != w] + ([("surf rows", len(got_p), len(want_p))] if len(got_p) != len(want_p) else [])
    finally:
        ctx.close()
    return bad


@pytest.mark.parametrize("width,n", [(128, (1 << 24) - 1), (64, (1 << 25) - 1)], ids=["128-2^24-1", "64-2^25-1"])
def test_packed_index_at_the_largest_max_points(aloam, orc, width, n):
    """max_points at its bound and a cloud that fills it: nearest neighbours planted at the last index (top ring), past 2^23, where
    the packed word is an inf / NaN pattern as a float, in exact-distance ties with early indices, and a forward 2nd / 3rd point
    at the largest forward rank n - 1"""
    bad = bound_case(aloam, orc, width, n)
    assert not bad, bad[:8]
