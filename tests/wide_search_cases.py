"""Scenes and host models for the scan-to-scan searches of 128-wide contexts (aloam_create_wide above 64 rings), shared by
tests/test_oracle_wide_search.py (CPU) and tests/test_gpu_wide_search.py (GPU).  TEST INFRASTRUCTURE.

* break_tables: a numpy model of the break tables k_rab_scan builds (fwd_end[r] = first index with ring >= r, bwd_begin[r] =
  one past the last index with ring < r), and its "no carry" mutation (each 32-ring slot of the 128-wide instance alone).
* associate: a vectorised form of config_cases.associate written the way k_odom_assoc searches -- the break tables, the ring
  window of config_cases.window and the ring slice rc - dn .. rc + up, argmin on (d2, visiting rank) -- for clouds of millions
  of points.
* Break scenes (int(intensity) dipping by one after every ring change, empty-ring runs across the slot boundaries, clouds of
  two rings), refusal scenes, and ring-major clouds of max_points points for the packed index at its bounds."""
import math

import numpy as np

import config_cases as K

WIDTH = 128
N_SCANS = (65, 96, 128)   # every n_scans above 64 gives a 128-wide context
SLOT = 32                 # rings per lane slot of k_rab_scan<128>
NO_RING = 0x7F7F7F7F      # first_of of an empty ring (create_ctx's memset), above every index

# closest-point rings of the 128-wide window scene: both ends, and both sides of every slot boundary
WIDE_RCS = [0, 1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 126, 127]
# NEARBY_SCAN values: as config_cases.NEARBY, around the 128-wide bound, and 3 - 2^-47, asymmetric across the 63 / 64 boundary
NEARBY = [1.0, 2.5, 3.0 - 2.0 ** -48, 3.0 - 2.0 ** -47, 63.0, 64.0, 65.0, 127.0, 128.0, 129.0, 1e300, math.inf]
NEARBY_IDS = ["1", "2.5", "3-2^-48", "3-2^-47", "63", "64", "65", "127", "128", "129", "1e300", "inf"]


def rings_of(cloud):
    return np.asarray(cloud, np.float32)[:, 3].astype(np.int32)


def break_tables(ring, width=WIDTH, carry=True):
    """(fwd_end, bwd_begin), width + 1 entries each, as k_rab_scan<width> writes them for int(intensity) `ring` (clamped to
    0 .. width - 1 as k_rab_count bins it).  carry=False: every 32-ring slot is computed alone -- the suffix minima of a slot
    stop at its last ring (and at n), the prefix maxima start at its first ring."""
    ring = np.clip(np.asarray(ring), 0, width - 1)
    n = len(ring)
    first = np.full(width, NO_RING, np.int64)
    last = np.full(width, -1, np.int64)
    u, i = np.unique(ring, return_index=True)
    first[u] = i
    u, i = np.unique(ring[::-1], return_index=True)
    last[u] = n - 1 - i
    seg = width if carry else SLOT
    fwd = np.empty(width + 1, np.int64)
    bwd = np.empty(width + 1, np.int64)
    for s0 in range(0, width, seg):
        f, l = first[s0:s0 + seg], last[s0:s0 + seg]
        fwd[s0:s0 + seg] = np.minimum(np.minimum.accumulate(f[::-1])[::-1], n)
        bwd[s0 + 1:s0 + seg + 1] = np.maximum.accumulate(l) + 1
    fwd[width], bwd[0] = n, 0
    return fwd, bwd


def ring_major_ok(ring, width=WIDTH, tables=None):
    """the check of k_ring_offsets<width> with the given break tables: every int(intensity) is a ring of 0 .. width - 1 and no
    earlier point has a ring two or more above (fwd_end[r + 2] >= i)"""
    ring = np.asarray(ring)
    if ring.min() < 0 or ring.max() > width - 1:
        return False
    fwd, _ = tables if tables is not None else break_tables(ring, width)
    return bool(np.all(fwd[np.minimum(ring + 2, width)] >= np.arange(len(ring))))


def invariant_holds(ring):
    """int_i >= max_{j<i} int_j - 1: the clouds scanRegistration.cpp can emit"""
    ring = np.asarray(ring)
    return bool(np.all(ring >= np.maximum.accumulate(ring) - 1))


def associate(last, queries, thr, nearby, corner, width=WIDTH, tables=None):
    """config_cases.associate (identity pose, rows (query, closest, 2nd, 3rd or -1)) in k_odom_assoc's formulation: brute-force
    nearest neighbour (first index on ties), the candidates (closest, fwd_end) then [bwd_begin, closest) in visiting order,
    restricted to the ring slice rc - dn .. rc + up, and argmin on (d2, visiting rank) per class.  tables: break_tables of the
    cloud (computed when None)."""
    last = np.asarray(last, np.float32)
    ring = rings_of(last)
    fwd, bwd = tables if tables is not None else break_tables(ring, width)
    rows = []
    for i, q in enumerate(np.asarray(queries, np.float32)):
        d = K.sqd(last, q)
        j = int(np.argmin(d))
        if not float(d[j]) < thr:
            continue
        rc = int(ring[j])
        dn, up = K.window(rc, nearby, width)
        fe, bb = int(fwd[min(rc + up + 1, width)]), int(bwd[max(rc - dn, 0)])
        f = np.arange(j + 1, max(fe, j + 1))
        b = np.arange(j - 1, min(bb, j) - 1, -1)
        cand = np.concatenate([f, b])                    # visiting order: forward ascending, then backward descending
        r = ring[cand]
        dc = d[cand].astype(np.float64)
        ok = (r >= max(rc - dn, 0)) & (r <= min(rc + up, width - 1)) & (dc < thr)
        same = np.concatenate([ring[f] <= rc, ring[b] >= rc])

        def pick(mask):
            if not mask.any():
                return -1
            k = np.flatnonzero(mask)
            return int(cand[k[np.argmin(dc[k])]])      # first minimum in visiting order = smallest rank

        if corner:
            m2 = pick(ok & ~same)
            if m2 >= 0:
                rows.append((i, j, m2, -1))
        else:
            m2, m3 = pick(ok & same), pick(ok & ~same)
            if m2 >= 0 and m3 >= 0:
                rows.append((i, j, m2, m3))
    return rows


# ------------------------------------------------------------------------------------------------ break scenes
def ring_cloud(rings, per_ring=12, dip=3, plants=()):
    """ring-major cloud: per ring of `rings` (ascending) `per_ring` returns on an arc at 10 + 0.5 b m, z = -1 + 0.05 b for the b-th
    ring of the list (consecutive rings of the list lie 0.5 m apart whatever their numbers); the last
    `dip` returns of every ring block but the first have int(intensity) one below (relTime < 0), so the cloud descends by one
    at every ring change.  plants: (index, xyz) overrides.  Returns (cloud, block start per ring)."""
    pts, start = [], {}
    for b, r in enumerate(rings):
        start[r] = len(pts)
        for j in range(per_ring):
            a = 0.05 * j + 0.002 * r
            rho = 10.0 + 0.5 * b
            it = r - 0.02 if (b > 0 and j >= per_ring - dip) else r + 0.005 * j
            pts.append([rho * math.cos(a), rho * math.sin(a), -1.0 + 0.05 * b, it])
    c = np.array(pts, np.float32)
    for i, xyz in plants:
        c[i, :3] = xyz
    return c, start


PLANT_RCS = (31, 32, 63, 64, 95, 96, 127)


def planted_scene(nearby=2.5, per_ring=12, dip=3):
    """every ring 0..127, dipping by one after each ring change (so across the slot boundaries 32 -> 31, 64 -> 63, 96 -> 95),
    and per closest ring rc of PLANT_RCS a query at the first return of ring rc with two entries 1 and 1.5 cm from it that lie
    past the loops' break indices at this nearby (up = dn = 2 at 2.5):
      forward   a dip return (int rc + up) of ring block rc + up + 1: it follows the first int >= rc + up + 1;
      backward  a return (int rc - dn) of ring block rc - dn, which precedes that block's dip returns (int rc - dn - 1).
    Returns (cloud, [(query index, planted index)])."""
    rings = list(range(WIDTH))
    plain, start = ring_cloud(rings, per_ring, dip)
    plants, pairs = [], []
    for rc in PLANT_RCS:
        dn, up = K.window(rc, nearby, WIDTH)
        q = start[rc]
        if rc + up + 1 <= WIDTH - 1:
            i = start[rc + up + 1] + per_ring - 1
            plants.append((i, plain[q, :3] + np.float32([0.0, 0.0, 0.01])))
            pairs.append((q, i))
        if rc - dn >= 1:
            i = start[rc - dn] + 1
            plants.append((i, plain[q, :3] + np.float32([0.0, 0.0, -0.015])))
            pairs.append((q, i))
    cloud, _ = ring_cloud(rings, per_ring, dip, plants)
    return cloud, pairs


def break_scenes():
    """{name: last cloud}: the planted scene, empty-ring runs that span slot boundaries, and clouds of two rings only"""
    out = {"planted": planted_scene()[0]}
    out["empty_runs"] = ring_cloud([r for r in range(WIDTH) if not (20 <= r <= 40 or 60 <= r <= 100)])[0]
    for pair in ((0, 127), (31, 32), (63, 64)):
        out["rings_%d_%d" % pair] = ring_cloud(list(pair), per_ring=24, dip=0)[0]
    return out


def refusal_scenes():
    """{name: (cloud, needs the carry)}: clouds outside the invariant or the ring range.  Two-ring drops across a boundary
    (65 then 63; a run 65, 64, 63) are caught by fwd_end entries of the offending ring's own slot; a three-ring drop whose
    ring r + 2 is the last of a slot and absent (32 then 29 without ring 31; 64 then 61 without 63; 96 then 93 without 95) is
    caught only through the carry from the slot above."""
    out = {}
    base = lambda rings: ring_cloud(rings, per_ring=6, dip=0)[0]
    c = base(list(range(WIDTH)))
    s = 65 * 6 + 3
    c[s, 3] = 63.05
    out["drop_65_63"] = (c, False)
    c = base(list(range(WIDTH)))
    c[66 * 6 - 3: 66 * 6, 3] = [64.05, 63.05, 63.06]   # ... 65, 65, 65, 64, 63, 63 | 66 ...
    out["run_65_64_63"] = (c, False)
    c = base(list(range(WIDTH)))
    c[-1, 3] = 128.02
    out["ring_128"] = (c, False)
    for top in (31, 63, 95):
        rings = [r for r in range(WIDTH) if r != top]
        c = base(rings)
        c[rings.index(top + 1) * 6 + 5, 3] = top - 2 + 0.05   # the last return of ring top + 1 block drops three rings
        out["drop_%d_%d" % (top + 1, top - 2)] = (c, True)
    return out


# ------------------------------------------------------------------------------------------------ the packed index at its bounds
def bound_cloud(n, width, seed=0):
    """n points, ring-major over rings 0 .. width - 1 (ring = index * width // n: index n - 1 on the top ring), uniform in a shell
    of 8..40 m and |z| <= 3 m (one azimuth bucket x ring cell holds about n / 16384 points)"""
    rng = np.random.default_rng(seed)
    c = np.empty((n, 4), np.float32)
    phi = rng.uniform(-np.pi, np.pi, n)
    rho = rng.uniform(8.0, 40.0, n)
    c[:, 0] = rho * np.cos(phi)
    c[:, 1] = rho * np.sin(phi)
    del phi, rho
    c[:, 2] = rng.uniform(-3.0, 3.0, n)
    c[:, 3] = (np.arange(n, dtype=np.int64) * width // n).astype(np.float32) + np.float32(0.05)
    return c


def bound_sites(n, width):
    """indices to plant nearest neighbours at: the last index (top ring), indices past 2^23, the range whose packed word
    (index << log2 width | ring) is an inf / NaN bit pattern as a float, and pairs (late, early) for exact-distance ties"""
    inf_from = 0x7F800000 >> (7 if width == 128 else 6)    # 0xFF0000 at 128 rings, 0x1FE0000 at 64
    single = [n - 1, (1 << 23) + 1, (1 << 23) + 123457, inf_from, inf_from + 4097, n - 2]
    ties = [(inf_from + 1, 7), (n - 3, 1 << 20), ((1 << 23) + 5, 1 << 22)]
    return inf_from, single, ties


DELTA = np.float32(2.0 ** -9)   # planted offsets: exact in float32 at |z| <= 3, far below the ~0.1 m point spacing


def plant_bounds(cloud, width, seed=1):
    """plants into a bound_cloud in place; returns (queries (m, 4), expected nearest index per query).
      - per single site i: the point moved to a fresh spot s, the query at s - DELTA z;
      - per tie (late, early): both at the same distance DELTA from the query, on either side in z (early wins);
      - the largest forward rank: index 0 (ring 0) DELTA above a query, index n - 1 (top ring) 2 DELTA below it, so that
        index n - 1 is the corner 2nd point (forward, ring above) and the surf 3rd point of the query with closest index 0.
    The spots lie on a circle of 20 m, 0.3 rad apart."""
    n = len(cloud)
    _, single, ties = bound_sites(n, width)
    rng = np.random.default_rng(seed)
    spots = iter(range(64))

    def spot():
        a = -3.0 + 0.3 * next(spots)
        return np.float32([20.0 * math.cos(a), 20.0 * math.sin(a), round(float(rng.uniform(-2, 2)), 3)])

    qs, want = [], []
    s = spot()                                    # the largest forward rank (index n - 1 is also a single site below)
    cloud[0, :3] = s + np.float32([0, 0, DELTA])
    cloud[n - 1, :3] = s - np.float32([0, 0, 2 * DELTA])
    qs.append(s); want.append(0)
    for i in single:
        if i != n - 1:
            s = spot()
            cloud[i, :3] = s + np.float32([0, 0, DELTA])
        else:
            s = cloud[i, :3] + np.float32([0, 0, DELTA / 2])   # nearer to n - 1 than to index 0 (2.5 DELTA away)
        qs.append(s); want.append(i)
    for late, early in ties:
        s = spot()
        cloud[late, :3] = s + np.float32([0, 0, DELTA])
        cloud[early, :3] = s - np.float32([0, 0, DELTA])
        qs.append(s); want.append(early)
    q = np.zeros((len(qs), 4), np.float32)
    q[:, :3] = np.array(qs, np.float32)
    q[:, 3] = np.float32(5.05)
    return q, np.array(want)
