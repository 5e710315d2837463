"""GPU parity at the edges of the prior-map search (cubemap.cu k_locate_begin / k_prior_tag, mapping.cu k_map_knn5_prior): the
window filter, ties between cubes ordered by window offset + rank, full cubes and the 16-bit rank, cube tags around empty cubes,
the acceptance boundary across cubes, clipped windows and lanes on different windows in one launch.

Every prior map here is a crafted store: a real mapped lane snapshot whose store table and payload are replaced, as aloam_lane_save
writes them.  The store does not check geometry, so a cube may hold points anywhere; the search must follow the stored cube.  The
association of a lane (aloam_debug_prior_associate at the identity pose, so the stack points are the queries bit for bit) is
checked against a numpy model of k_locate_begin (centre cube, clipped window in the reference's loop order, window offsets,
gathered submaps): a float32 brute-force 5-NN on the gathered submap, the oracle's fits, and aloam_mapping_associate on a context
that uploaded that submap, row for row and byte for byte."""
import struct

import numpy as np
import pytest

import lane_refs as R

pytestmark = pytest.mark.gpu

NCUBE, CW, CH, CD = 4851, 21, 21, 11
HEADER, TABLE = 256, 39424            # sizeof(SnapHeader), sizeof(SnapStore)
MAXPTS = 65536                        # slab capacities 16384 corner / 65536 surf
MAXMAP = 20000
SENSOR = "VLP-16"
IDENT = np.array([0, 0, 0, 1.0, 0, 0, 0])
Q0 = np.array([0, 0, 0, 1.0])
F32 = np.float32


def _cfg(batch):
    return dict(n_scans=16, max_points=MAXPTS, max_batch=batch, max_ring_points=4096, max_map_points=MAXMAP)


def cube_coord(v, cen):
    """int((v + 25) / 50) + cen, minus one when v + 25 < 0 (laserMapping.cpp:314-325)"""
    c = int((v + 25.0) / 50.0) + cen
    return c - 1 if v + 25.0 < 0 else c


def cube_index(i, j, k):
    return i + CW * j + CW * CH * k


def inside(i, j, k):
    return 0 <= i < CW and 0 <= j < CH and 0 <= k < CD


def d2(pts, q):
    """float32 (dx^2 + dy^2) + dz^2, the search's distance"""
    d = pts[:, :3].astype(F32) - np.asarray(q, F32)[:3]
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def cloud(rows):
    a = np.zeros((len(rows), 4), F32)
    if len(rows):
        a[:, :3] = np.asarray(rows, np.float64)
    return a


class Store:
    """a cube store: per (type, cube index) the points in rank order; a key without points is a count-0 cube, a missing key -1"""

    def __init__(self, cen=(10, 10, 5)):
        self.cen = tuple(cen)
        self.cubes = {}

    def put(self, ty, ijk, pts):
        """appends pts to cube ijk of type ty; returns the rank of the first one"""
        key = (ty, cube_index(*ijk))
        old = self.cubes.get(key, np.zeros((0, 4), F32))
        self.cubes[key] = np.concatenate([old, np.asarray(pts, F32).reshape(-1, 4)])
        return old.shape[0]

    def counts(self):
        c = np.full((2, NCUBE), -1, np.int32)
        for (ty, i), p in self.cubes.items():
            c[ty, i] = p.shape[0]
        return c

    def payload(self):
        parts = [self.cubes[(ty, i)] for i in range(NCUBE) for ty in (0, 1) if (ty, i) in self.cubes]
        return np.concatenate(parts) if parts else np.zeros((0, 4), F32)

    def blob(self, tmpl):
        nls, nlf = struct.unpack_from("<ii", tmpl, 28)
        store = HEADER + 16 * (nls + nlf)
        table = bytearray(tmpl[store:store + TABLE].tobytes())
        counts, pay = self.counts(), self.payload()
        struct.pack_into("<3i", table, 0, *self.cen)
        table[592:592 + counts.nbytes] = counts.tobytes()
        struct.pack_into("<iiqq", table, 592 + counts.nbytes, 0, 0, pay.shape[0], 0)
        out = np.concatenate([tmpl[:store], np.frombuffer(bytes(table), np.uint8), pay.view(np.uint8).reshape(-1)])
        struct.pack_into("<q", out, 16, out.size)   # total_bytes
        return out

    def frozen(self):
        import pyfrozen
        return pyfrozen.FrozenMap.from_export(self.cen, self.counts(), self.payload())

    def window(self, t):
        """k_locate_begin at hand-off translation t: centre cube, the valid cubes in loop order (dk fastest), per type the window
        offsets (-1 outside the buffer) and the gathered submap with each point's (window entry, cube index, rank)"""
        ctr = [cube_coord(float(t[a]), self.cen[a]) for a in range(3)]
        valid, win = [], np.full((2, 75), -1, np.int64)
        sub, meta, off = [[], []], [[], []], [0, 0]
        for w in range(75):
            i, j, k = ctr[0] - 2 + w // 15, ctr[1] - 2 + (w // 3) % 5, ctr[2] - 1 + w % 3
            if not inside(i, j, k):
                continue
            c = cube_index(i, j, k)
            valid.append(c)
            for ty in (0, 1):
                win[ty, w] = off[ty]
                p = self.cubes.get((ty, c))
                if p is not None and p.shape[0]:
                    sub[ty].append(p)
                    meta[ty].append(np.stack([np.full(p.shape[0], w), np.full(p.shape[0], c), np.arange(p.shape[0])], 1))
                    off[ty] += p.shape[0]
        sub = [np.concatenate(s) if s else np.zeros((0, 4), F32) for s in sub]
        meta = [np.concatenate(m) if m else np.zeros((0, 3), np.int64) for m in meta]
        return {"ctr": ctr, "valid": valid, "win": win, "sub": sub, "meta": meta}


def knn_by(sub, keys, q, k=5):
    """the submap positions of the k candidates of smallest (d^2, key): the search under another candidate order"""
    return np.lexsort((keys, d2(sub, q)))[:k]


# ---- the environment: one localiser with 16 lanes, a context for aloam_mapping_associate, a crafted-snapshot template

@pytest.fixture(scope="module")
def env(aloam, synth):
    scans = R.traj(synth, 0, 4, sensor=SENSOR)
    dev = R.to_device(scans)
    c = aloam.Aloam(**_cfg(1))
    ops = np.array([[2]] + [[1]] * 2, np.int32)
    _, m = c.scan_stream_lanes([[d.data_ptr()] for d in dev[:3]], [[d.shape[0]] for d in dev[:3]], ops, True, mapped=True)
    tmpl = np.asarray(c.lane_save(0)).copy()
    real = c.mapper_export(aloam.EXPORT_MAP, 0).copy()
    c.close()
    nls, nlf = struct.unpack_from("<ii", tmpl, 28)
    counts = np.frombuffer(tmpl.tobytes(), np.int32, 2 * NCUBE, HEADER + 16 * (nls + nlf) + 592).reshape(2, NCUBE)
    # the real store's points per type (the export is corner cube, surf cube of every cube in index order)
    n = np.maximum(counts, 0).T.reshape(-1)
    ends = np.cumsum(n)
    segs = [real[e - k:e] for e, k in zip(ends, n)]
    real_t = [np.concatenate(segs[0::2]), np.concatenate(segs[1::2])]
    loc = aloam.Aloam(**_cfg(16))
    ref = aloam.Aloam(n_scans=16, max_points=MAXPTS, max_map_points=200000)
    e = {"tmpl": tmpl, "scans": scans, "dev": dev, "loc": loc, "ref": ref, "real": real_t}
    yield e
    loc.close()
    ref.close()


def load(env, store):
    env["loc"].reset_odometry()            # ends every trajectory: a prior map loads only while no lane localises
    env["loc"].prior_map_load(store.blob(env["tmpl"]))


def arm(env, lanes, n_scans=1):
    """lanes = {lane: (q, t)}: each armed and STARTed in one aloam_scan_stream_lanes call on the trajectory's first n_scans scans;
    the hand-off pose of the START is (q, t) exactly (an identity odometry pose) -> {lane: (odometry rows, map rows)}"""
    c = env["loc"]
    for lane, (q, t) in lanes.items():
        c.lane_localise(lane, np.asarray(q, np.float64), np.asarray(t, np.float64))
    b = max(lanes) + 1
    ptrs, counts, ops = np.zeros((n_scans, b), np.uint64), np.zeros((n_scans, b), np.int64), np.zeros((n_scans, b), np.int32)
    for lane in lanes:
        for k in range(n_scans):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = env["dev"][k].data_ptr(), env["dev"][k].shape[0], 2 if k == 0 else 1
    o, m = c.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
    return {lane: (o[:, lane], m[:, lane]) for lane in lanes}


def check(env, orc, W, qc, qs, got):
    """got = prior_associate rows of corner queries qc then surf queries qs against the window model W: accepted / rejected and
    the five indices exact, fits as the oracle's, rows byte-identical to aloam_mapping_associate on the gathered submap.
    Returns per type (indices, d^2, accepted) of the float32 brute force."""
    import pyoracle
    out = []
    for ty, (qq, rows) in enumerate(((qc, got[:len(qc)]), (qs, got[len(qc):]))):
        sub = W["sub"][ty]
        if sub.shape[0]:
            idx, sqd = pyoracle.bruteforce_knn(sub, qq, 5)
        else:
            idx, sqd = np.full((len(qq), 5), -1, np.int32), np.full((len(qq), 5), np.inf, F32)
        acc = (idx[:, 4] >= 0) & (sqd[:, 4].astype(np.float64) < 1.0)
        reached = ~np.isnan(rows[:, 9])                                          # nn is written for an accepted neighbourhood
        assert np.array_equal(reached, acc), ("type", ty, np.nonzero(reached != acc)[0])
        assert np.array_equal(rows[acc, 9:14], idx[acc].astype(np.float64)), ("type", ty)
        assert np.all(rows[:, 1][~acc] == -1) and np.array_equal(rows[acc, 0], np.nonzero(acc)[0].astype(np.float64))
        out.append((idx, sqd, acc))
    # the fits: the oracle on the same submaps (an empty cloud stands in as one far point: nothing reaches it)
    far = cloud([[1e4, 1e4, 1e4]])
    om = orc.Mapping()
    om.set_map(W["sub"][0] if W["sub"][0].shape[0] else far, W["sub"][1] if W["sub"][1].shape[0] else far)
    fits, _ = om.associate(qc, qs, IDENT)
    acc = got[got[:, 1] >= 0]
    assert len(acc) == len(fits) and np.array_equal(acc[:, [0, 1]], fits[:, [0, 1]]) and np.array_equal(acc[:, 9:], fits[:, 9:])
    edges = fits[:, 1] == 0
    a_ok = np.abs(acc[edges, 2:8] - fits[edges, 2:8]).max(1, initial=0) < 1e-9
    sw = np.concatenate([fits[edges, 5:8], fits[edges, 2:5]], axis=1)
    b_ok = np.abs(acc[edges, 2:8] - sw).max(1, initial=0) < 1e-9
    assert np.all(a_ok | b_ok)
    pl = ~edges
    assert np.all(np.abs(acc[pl, 2:9] - fits[pl, 2:9]) <= 1e-10 * np.maximum(1.0, np.abs(fits[pl, 2:9])))
    # the same k_map_fit after gather + K0 + k_map_knn5: the claimed submap index, row for row
    env["ref"].map_upload(W["sub"][0], W["sub"][1])
    assert env["ref"].mapping_associate(qc, qs, IDENT).tobytes() == got.tobytes()
    return out


def associate(env, orc, store, t, qc, qs, lane=0):
    """arm `lane` at hand-off translation t, associate qc / qs through its window, check against the model"""
    load(env, store)
    arm(env, {lane: (Q0, t)})
    W = store.window(t)
    got = env["loc"].prior_associate(lane, qc, qs, IDENT)
    return W, check(env, orc, W, qc, qs, got)


def ring(q, r, n, axis_pair=(1, 2)):
    """n points at distance r from q in the plane of the two axes (dyadic radius, exact on the axes)"""
    out = []
    for a in range(n):
        p = np.array(q, np.float64)
        ang = 2 * np.pi * a / n
        p[axis_pair[0]] += r * np.cos(ang)
        p[axis_pair[1]] += r * np.sin(ang)
        out.append(p)
    return out


# ---- 1. the window filter

def test_out_of_window_neighbours_are_excluded(env, orc):
    """queries 0.25 m inside each face of the 5 x 5 x 3 window with nearer points just across the face: accepted from window
    points, or rejected when only out-of-window points are close enough; points stored in an out-of-window cube but lying in the
    centre cube, and window points lying far outside the window, follow their stored cube"""
    S, ctr = Store(), (10, 10, 5)
    qc, qs, inner_far = [], [], []
    for axis in range(3):
        for s in (-1, 1):
            half = 2 if axis < 2 else 1
            face = 50.0 * (half + 0.5) * s                            # x, y: +-125 m ; z: +-75 m
            for case, shift in (("accept", 0.0), ("reject", 16.0)):
                q = np.zeros(3)
                q[axis] = face - 0.25 * s
                q[(axis + 1) % 3] = shift
                cin, cout = list(ctr), list(ctr)
                cin[axis] += half * s
                cout[axis] += (half + 1) * s
                across = q.copy(); across[axis] = face + 0.125 * s   # 0.375 m away, across the face
                nearer = ring(across, 0.125, 5, ((axis + 1) % 3, (axis + 2) % 3))
                within = ring(q, 0.75, 5 if case == "accept" else 4, ((axis + 1) % 3, (axis + 2) % 3))
                if case == "reject":
                    within.append(q + np.eye(3)[(axis + 1) % 3] * 1.5)   # in the 27-cell block, beyond 1 m
                for ty in (0, 1):
                    S.put(ty, cout, cloud(nearer))
                    S.put(ty, cin, cloud(within))
                (qc if axis % 2 else qs).append(q)
                inner_far.append((case, q, cloud(nearer)))
    # stored out of the window (di = +3), lying in the centre cube; stored in the window (dj = -2), lying 300 m away
    q = np.array([3.0, 2.0, 1.0])
    for ty in (0, 1):
        S.put(ty, (13, 10, 5), cloud(ring(q, 0.125, 5)))
        S.put(ty, (10, 10, 5), cloud(ring(q, 0.625, 5, (0, 2))))
        S.put(ty, (10, 8, 5), cloud(ring(q + [300.0, 0, 0], 0.25, 5)))
    qc += [q, q + [300.0, 0, 0]]
    qs += [q, q + [300.0, 0, 0]]
    qc, qs = cloud(qc), cloud(qs)
    W, res = associate(env, orc, S, np.zeros(3), qc, qs)
    acc = np.concatenate([res[0][2], res[1][2]])
    queries = np.concatenate([qc, qs])
    # the edge was reached: every face query has out-of-window points nearer than its window's 5th neighbour
    for case, q, nearer in inner_far:
        row = np.nonzero(np.all(queries[:, :3] == F32(q), axis=1))[0][0]
        assert acc[row] == (case == "accept"), (case, q)
        assert d2(nearer, q).max() < 0.25
    assert acc.sum() == 6 + 4                                          # six face queries, and both stored-cube queries of each type
    assert W["ctr"] == [10, 10, 5] and len(W["valid"]) == 75


# ---- 2. ties across cubes

def test_ties_across_cubes_follow_window_offset_plus_rank(env, orc):
    """equal-d^2 pairs and triples split over cubes that differ in di, dj or dk, with ranks chosen so that ordering by rank alone,
    by cube_index (i fastest) or by the tag would give another order; 5th / 6th neighbours tied across cubes decide the set"""
    S, ctr = Store(), np.array([10, 10, 5])
    far = lambda n, x0: cloud([[x0 + 3.0 * a, 40.0, -20.0] for a in range(n)])   # rank fillers, out of every query's reach
    # cube pairs (second before first in the window's loop order, after it in cube_index order)
    pairs = [((1, 0, -1), (-1, 0, 1)), ((0, 1, 0), (0, -1, 1)), ((2, -2, 0), (-2, 2, 0)), ((0, 0, 1), (0, 0, -1))]
    qs = []
    for p, (ca, cb) in enumerate(pairs):
        q = np.array([4.0 * p, 0.0, 0.0])
        A, B = tuple(ctr + ca), tuple(ctr + cb)
        for ty in (0, 1):
            S.put(ty, B, far(3 + p, 100.0 * p))                       # B's tied point at rank 3 + p, A's at rank 0
            S.put(ty, A, cloud([q + [0.5, 0, 0]]))
            S.put(ty, B, cloud([q + [0, 0.5, 0]]))
            S.put(ty, A, cloud([q + [0, 0, 0.5], q + [0, -0.5, 0]]))       # a triple: two in A, one in B
            S.put(ty, tuple(ctr), cloud([q + [0.25, 0.25, 0.25]]))          # one nearer point in the centre cube
        qs.append(q)
    # the 5th / 6th tie: four near points in the centre cube, two tied at d^2 = 0.25 in (di -1) and (di +1, dk -1)
    for p, (ca, cb) in enumerate([((1, 0, -1), (-1, 0, 0)), ((0, 2, -1), (0, -2, 1)), ((0, 0, 1), (0, 0, -1))]):
        q = np.array([4.0 * p, 10.0, 0.0])
        for ty in (0, 1):
            S.put(ty, tuple(ctr), cloud(ring(q, 0.125, 4)))
            S.put(ty, tuple(ctr + ca), cloud([q + [0.5, 0, 0]]))
            S.put(ty, tuple(ctr + cb), far(2, 500.0 + 50 * p))
            S.put(ty, tuple(ctr + cb), cloud([q + [-0.5, 0, 0]]))
        qs.append(q)
    q = cloud(qs)
    W, res = associate(env, orc, S, np.zeros(3), q, q)
    # the edge was reached: each alternative order gives another neighbour list for some query, and some 5th neighbour is tied
    sub, meta = W["sub"][1], W["meta"][1]
    right = np.arange(sub.shape[0])
    alts = {"rank alone": meta[:, 2], "cube_index, i fastest": meta[:, 1] * 65536 + meta[:, 2]}
    for name, key in alts.items():
        assert any(not np.array_equal(knn_by(sub, right, qq), knn_by(sub, key, qq)) for qq in q), name
        # ... and another set, not only another order, for some 5th / 6th tie
        assert any(set(knn_by(sub, right, qq)) != set(knn_by(sub, key, qq)) for qq in q[len(pairs):]), name
    idx6, sqd6 = orc.bruteforce_knn(sub, q, 6)
    assert np.any((sqd6[:, 4] == sqd6[:, 5]) & (meta[idx6[:, 4], 1] != meta[idx6[:, 5], 1]))
    assert res[1][2].all() and res[0][2].all()


# ---- 3. full cubes and the 16-bit rank

def test_full_cubes_and_the_16_bit_rank(env, orc):
    """a surf cube of 65536 points and a corner cube of 16384 at the first window entry: neighbours at ranks 32767, 32768 and 65535
    (8191, 8192, 16383), and a tie between the last rank of the full cube and rank 0 of the next window cube (indices 65535 and
    65536; 16383 and 16384)"""
    S = Store()
    rng = np.random.default_rng(3)
    first, nxt = (8, 8, 4), (8, 8, 5)                                 # window entries 0 and 1 of centre (10, 10, 5)
    qa, qb = np.array([0.0, 0.0, 0.0]), np.array([0.0, 3.0, 0.0])
    for ty, full in ((0, 16384), (1, 65536)):
        pts = np.zeros((full, 4), F32)
        pts[:, :3] = rng.uniform([6, -30, -8], [60, 30, 8], (full, 3)).astype(F32)   # out of every query's reach
        mid = full // 2
        near = ring(qa, 0.5, 5)
        for r, p in zip((mid - 2, mid - 1, mid, mid + 1, mid + 2), near):
            pts[r, :3] = p
        for r, p in zip((100, 101, 102, 103), ring(qb, 0.125, 4)):
            pts[r, :3] = p
        pts[full - 1, :3] = qb + [0.5, 0, 0]
        S.put(ty, first, pts)
        S.put(ty, nxt, cloud([qb + [-0.5, 0, 0], qb + [0, 0, 40.0]]))
    q = cloud([qa, qb])
    W, res = associate(env, orc, S, np.zeros(3), q, q)
    for ty, full in ((0, 16384), (1, 65536)):
        idx, sqd, acc = res[ty]
        assert acc.all()
        assert {full // 2 - 1, full // 2} <= set(idx[0].tolist())
        assert idx[1][4] == full - 1 and sqd[1][4] == 0.25                  # the tie with index `full` (rank 0 of the next cube)
        assert d2(W["sub"][ty][full:full + 1], qb)[0] == 0.25 and W["win"][ty][1] == full


# ---- 4. cube tags around empty cubes

def test_cube_tags_around_empty_cubes(env, orc):
    """runs of count -1 and count 0 cubes before a non-empty cube (the boundary of k_prior_tag's last-prefix search): neighbours at
    rank 0 of such a cube, at index 0 of the map and at its last point; and a map whose corner type is empty"""
    S = Store()
    q0, q1, q2 = np.array([0.0, 0.0, 0.0]), np.array([5.0, 0.0, 0.0]), np.array([10.0, 0.0, 0.0])
    for ty in (0, 1):
        for c in range(0, 40, 3):                                     # count-0 cubes before the first non-empty one
            S.put(ty, (c % CW, (c // CW) % CH, 0), cloud([]))
        S.put(ty, (8, 8, 4), cloud([q0 + [0.125, 0, 0]] + ring(q0, 0.5, 4)))    # the first cube of the map: index 0
        S.put(ty, (10, 10, 5), cloud(ring(q1, 0.375, 3)))              # the cube before, in cube order, of the next one
        S.put(ty, (11, 10, 5), cloud([]))
        S.put(ty, (12, 10, 5), cloud([]))                              # (13, 10, 5) is -1: di = +3, out of the window anyway
        S.put(ty, (9, 11, 5), cloud([q1 + [0.0625, 0, 0]] + ring(q1, 0.5, 2)))  # rank 0 after two count-0 cubes and one -1
        S.put(ty, (12, 12, 6), cloud(ring(q2, 0.25, 4) + [q2 + [0, 0, 0.0625]]))  # the last cube of the map: its last point
    q = cloud([q0, q1, q2])
    W, res = associate(env, orc, S, np.zeros(3), q, q)
    for ty in (0, 1):
        idx, sqd, acc = res[ty]
        assert acc.all() and idx[0][0] == 0 and idx[2][0] == W["sub"][ty].shape[0] - 1
        first_in_cube = W["win"][ty][(-1 + 2) * 15 + (1 + 2) * 3 + (0 + 1)]      # window entry of cube (9, 11, 5)
        assert idx[1][0] == first_in_cube and W["sub"][ty][first_in_cube, 0] == F32(q1[0] + 0.0625)
    # a prior map without corner points: every corner query is rejected, the surf queries are not
    S0 = Store()
    for c in ((8, 8, 4), (10, 10, 5)):
        S0.put(0, c, cloud([]))
        S0.put(1, c, cloud(ring(q0, 0.25, 6)))
    W, res = associate(env, orc, S0, np.zeros(3), cloud([q0]), cloud([q0]))
    assert not res[0][2].any() and res[1][2].all()


# ---- 5. the acceptance boundary across cubes

def test_acceptance_boundary_across_cubes(env, orc):
    """a 5th neighbour at float d^2 = 1.0 (rejected) and at 1 - 2^-24 (accepted), stored in another window cube than the first four"""
    S = Store()
    qa, qb = np.array([40.0, 0.0, 0.0]), np.array([-0.5, 30.0, 0.0])
    near = lambda q: [q + [0.0625, 0, 0], q + [0, 0.0625, 0], q + [0, 0, 0.0625], q + [0, 0, -0.0625]]
    below = [float(F32(0.5) - F32(2.0 ** -24)), 30.0 + 2.0 ** -12, 0.0]
    for ty in (0, 1):
        S.put(ty, (10, 10, 5), cloud(near(qa) + near(qb)))
        S.put(ty, (9, 11, 4), cloud([qa + [1.0, 0, 0], below]))
    q = cloud([qa, qb])
    W, res = associate(env, orc, S, np.zeros(3), q, q)
    for ty in (0, 1):
        idx, sqd, acc = res[ty]
        assert sqd[0][4] == F32(1.0) and sqd[1][4] == F32(1.0) - F32(2.0 ** -24)
        assert list(acc) == [False, True] and idx[1][4] == 1               # cube (9, 11, 4) comes first in the window


# ---- 6 / 7. clipped windows, lanes on different windows

def _copy(env, shift, n_corner, n_surf):
    """the n points of the real store nearest the origin, where its first scan was taken, moved by `shift` (a multiple of 50 m:
    a vehicle armed there finds the map it was made in)"""
    out = []
    for ty, n in ((0, n_corner), (1, n_surf)):
        p = env["real"][ty]
        p = p[np.argsort((p[:, :3].astype(np.float64) ** 2).sum(1), kind="stable")[:n]].copy()
        p[:, :3] = (p[:, :3].astype(np.float64) + shift).astype(F32)
        out.append(p)
    return out


CEN = (9, 12, 6)   # a store that has shifted
# centre cubes of 16 lanes: the six faces of the buffer, an edge, a corner, wholly outside, two lanes in one cube, the interior
CENTRES = [(0, 12, 6), (20, 12, 6), (9, 0, 6), (9, 20, 6), (9, 12, 0), (9, 12, 10), (0, 0, 6), (20, 20, 10), (-4, 12, 6),
           (5, 5, 3), (5, 5, 3), (14, 5, 3), (5, 16, 8), (14, 16, 8), (9, 12, 6), (1, 19, 1)]


def _lane_store(env):
    S = Store(CEN)
    copies = {}
    for lane, ctr in enumerate(CENTRES):
        shift = 50.0 * (np.array(ctr) - CEN)
        if ctr in copies.values() or not any(inside(ctr[0] + a, ctr[1] + b, ctr[2] + c) for a in (-2, 0, 2) for b in (-2, 0, 2) for c in (-1, 0, 1)):
            continue                                                  # the shared cube is stored once; no cube for the lane outside
        copies[lane] = ctr
        cc, cs = _copy(env, shift, 400, 1600)
        # split over the window's cubes inside the buffer, in alternating order, as a mapped store would hold them
        cubes = [(ctr[0] + a, ctr[1] + b, ctr[2] + c) for a in (-1, 0, 1) for b in (0, 1) for c in (0, -1) if inside(ctr[0] + a, ctr[1] + b, ctr[2] + c)]
        for ty, p in ((0, cc), (1, cs)):
            for s, c in enumerate(cubes):
                S.put(ty, c, p[s::len(cubes)])
    return S


def test_lanes_on_clipped_and_different_windows(env, orc, synth):
    """16 lanes armed in 16 centre cubes in one launch of k_locate_begin -- clipped at every face, an edge and a corner, one wholly
    outside the buffer (no valid cube), two in one cube -- on a store whose centre is not (10, 10, 5): each lane's centre and valid
    list as the frozen oracle's, and its association through its own window as the model's"""
    import pyfrozen
    S = _lane_store(env)
    load(env, S)
    frozen = S.frozen()
    lanes = {l: (Q0, 50.0 * (np.array(c) - CEN)) for l, c in enumerate(CENTRES)}
    arm(env, lanes)
    ns, _, mr, line_res, plane_res = synth.SENSORS[SENSOR]
    f = orc.Features(env["scans"][0], ns, mr)
    base = [b[::step] for b, step in zip(_copy(env, np.zeros(3), 400, 1600), (10, 40))]   # 40 points of each type of every copy
    for lane, (q, t) in lanes.items():
        st = env["loc"].mapper_state(lane)
        ref = pyfrozen.Localiser(frozen, q, t)
        ref.step(f.less_sharp, f.less_flat, Q0, np.zeros(3), line_res, plane_res)
        W = S.window(t)
        assert st["centre"] == frozen.centre == CEN and st["valid"] == ref.valid == W["valid"], lane
        assert list(W["ctr"]) == list(CENTRES[lane])
        # queries near the lane's own copy and near the next lane's
        other = 50.0 * (np.array(CENTRES[(lane + 1) % 16]) - CEN)
        qq = [np.concatenate([(b[:, :3].astype(np.float64) + s + 0.03).astype(F32), b[:, 3:]], 1) for b in base for s in (t, other)]
        qc, qs = np.concatenate(qq[:2]), np.concatenate(qq[2:])
        got = env["loc"].prior_associate(lane, qc, qs, IDENT)
        res = check(env, orc, W, qc, qs, got)
        if lane == 8:
            assert W["valid"] == [] and not res[0][2].any() and not res[1][2].any()
        else:
            assert res[1][2][:40].any(), lane                          # the lane's own copy is reached


def test_lanes_on_different_windows_equal_their_solo_runs(env):
    """the 16 lanes' trajectories in one aloam_scan_stream_lanes call (every launch shared) against each lane run alone"""
    S = _lane_store(env)
    load(env, S)
    lanes = {l: (Q0, 50.0 * (np.array(c) - CEN)) for l, c in enumerate(CENTRES)}
    got = arm(env, lanes, n_scans=3)
    for lane in lanes:
        env["loc"].reset_odometry()
        solo = arm(env, {lane: lanes[lane]}, n_scans=3)[lane]
        assert np.array_equal(got[lane][0], solo[0]) and np.array_equal(got[lane][1], solo[1]), lane
    assert np.array_equal(got[8][1][0], np.concatenate(lanes[8]))       # no valid cube: thin, the hand-off pose
    assert not np.array_equal(got[14][1][0], np.concatenate(lanes[14]))  # a full window: registered


# ---- 8. whole frames on crafted maps

def test_whole_frames_on_crafted_maps(env, orc, aloam, synth):
    """real scans through the stream on one crafted map, each lane on its own window:
    thin-map threshold on window points only (10 / 51, 11 / 50, 11 / 51 with the rest of the map just outside the window),
    a window of more points than cfg.max_map_points (unbounded: as the frozen oracle), and a frame whose mapping counterpart would
    neither shift nor overflow, on a window with ties across cubes and out-of-window points beside the map (bit for bit as
    aloam_mapper_step from the same snapshot)"""
    import pyfrozen
    cen = np.array([10, 10, 5])
    S = Store(tuple(cen))
    plan = {0: ((4, 4, 5), 10, 51), 1: ((11, 4, 5), 11, 50), 2: ((17, 4, 5), 11, 51), 3: ((4, 11, 5), None, None), 4: ((11, 11, 5), None, None)}
    for lane, (ctr, nc, ns_) in plan.items():
        ctr = np.array(ctr)
        shift = 50.0 * (ctr - cen)
        cc, cs = _copy(env, shift, 3000, 9000)
        if nc is not None:
            for ty, p, n in ((0, cc, nc), (1, cs, ns_)):
                o = np.argsort(d2(p, shift))                          # the window keeps the points nearest the vehicle
                S.put(ty, tuple(ctr), p[o[:n]])
                S.put(ty, tuple(ctr + [3, 0, 0]), p[o[n:]])           # the rest just outside (di = +3)
        elif lane == 3:
            filler = np.zeros((MAXMAP + 5000, 4), F32)
            filler[:, :3] = shift + np.random.default_rng(1).uniform([-40, -40, -60], [40, 40, -50], (filler.shape[0], 3))
            S.put(1, tuple(ctr + [-2, -2, -1]), filler)                # the first window entry: a mapping frame would truncate
            S.put(0, tuple(ctr), cc)
            S.put(1, tuple(ctr + [1, 1, 1]), cs)
        else:
            for ty, p in ((0, cc), (1, cs)):
                S.put(ty, tuple(ctr + [0, 0, -1]), p[0::2])
                S.put(ty, tuple(ctr + [-1, 1, 0]), p[1::2])
                S.put(ty, tuple(ctr + [1, -1, 1]), p[0:200:4])        # exact duplicates in another cube: ties across cubes
                near = p.copy(); near[:, 2] += F32(0.0625)
                S.put(ty, tuple(ctr + [3, 0, 0]), near)               # nearer copies of the map out of the window
    load(env, S)
    frozen = S.frozen()
    lanes = {l: (Q0, 50.0 * (np.array(c) - cen)) for l, (c, _, _) in plan.items()}
    got = arm(env, lanes)
    ns, _, mr, line_res, plane_res = synth.SENSORS[SENSOR]
    f = orc.Features(env["scans"][0], ns, mr)
    for lane, (q, t) in lanes.items():
        ref = pyfrozen.Localiser(frozen, q, t)
        pose, info = ref.step(f.less_sharp, f.less_flat, Q0, np.zeros(3), line_res, plane_res)
        W = S.window(t)
        if lane < 3:
            assert (W["sub"][0].shape[0], W["sub"][1].shape[0]) == plan[lane][1:]
            assert info["optimised"] == (lane == 2), lane
        if not info["optimised"]:
            assert np.array_equal(got[lane][1][0], np.concatenate([q, t])), lane
        assert np.abs(got[lane][1][0] - pose).max() < 1e-6, (lane, np.abs(got[lane][1][0] - pose).max())
    assert S.window(lanes[3][1])["sub"][1].shape[0] > MAXMAP
    # the mapping counterpart of lane 4's frame: the same store restored into a scratch context, T_wmap_wodom patched in
    W4 = S.window(lanes[4][1])
    assert max(s.shape[0] for s in W4["sub"]) <= MAXMAP and all(3 <= c < d - 3 for c, d in zip(W4["ctr"], (CW, CH, CD)))
    blob = bytearray(S.blob(env["tmpl"]).tobytes())
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    off = HEADER + 16 * (nls + nlf)
    struct.pack_into("<4d", blob, off + 536, *Q0)
    struct.pack_into("<3d", blob, off + 568, *lanes[4][1])
    scratch = aloam.Aloam(**_cfg(1))
    try:
        scratch.lane_restore(0, np.frombuffer(bytes(blob), np.uint8))
        g = scratch.extract_features(env["scans"][0])
        o = got[4][0][0]
        qm, tm, st = scratch.mapper_step(g["less_sharp"], g["less_flat"], o[:4], o[4:])
        assert not st["flags"] & aloam.FLAG_MAP_TOO_THIN
        assert np.array_equal(got[4][1][0], np.concatenate([qm, tm]))
    finally:
        scratch.close()
