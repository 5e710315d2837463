"""Hand-built "last" clouds and queries for the scan-to-scan association away from the default aloam_config, and a plain numpy
transcription of the two association loops of laserOdometry.cpp:299-483 that runs them.  Shared by tests/test_oracle_config.py
(CPU) and tests/test_gpu_config.py (GPU).  TEST INFRASTRUCTURE.

Every query sits at z = 0 and is associated at the identity pose, so the query the loops see is the point itself (with and
without DISTORTION: the identity rotates nothing).  Query clusters lie far enough apart that no point of another cluster is
ever a candidate below the thresholds used with them."""
import math

import numpy as np

# NEARBY_SCAN values: integers, where `int > rc + N` and `int >= rc + N` differ; the last ring; past every ring; a value whose
# rc + N and rc - N round differently in double (3 - 2^-48 keeps ring rc + 3 for rc >= 30 but ring rc - 3 only for rc >= 35)
NEARBY = [1.0, 1.5, 2.0, 3.0, 4.0, 63.0, 64.0, 1e3, 1e300, math.inf, 3.0 - 2.0 ** -48]
NEARBY_IDS = ["1", "1.5", "2", "3", "4", "63", "64", "1e3", "1e300", "inf", "3-2^-48"]
# DISTANCE_SQ_THRESHOLD values: float(thr) < thr for 4 + 2^-23, 0.7 and 25.3; float(thr) > thr for 0.1; exact for the rest;
# 1e40 is above FLT_MAX
THRESH = [0.25, 1.0, 4.0 + 2.0 ** -23, 0.7, 25.3, 0.1, 100.0, 400.0, 1e40]
THRESH_IDS = ["0.25", "1", "4+2^-23", "0.7", "25.3", "0.1", "100", "400", "1e40"]
# closest-point rings of the window scene: both ends of the ring range and the band where 3 - 2^-48 is asymmetric
WINDOW_RCS = [0, 1, 29, 30, 31, 32, 33, 34, 35, 62, 63]


def f32(v):
    return np.float32(v)


def sqd(pts, q):
    """((dx*dx + dy*dy) + dz*dz) in float32: k_odom_assoc's sqdist3, the kd-tree's L2_Simple and laserOdometry.cpp:322-327"""
    p = np.asarray(pts, np.float32)
    q = np.asarray(q, np.float32)
    dx, dy, dz = p[..., 0] - q[0], p[..., 1] - q[1], p[..., 2] - q[2]
    return (dx * dx + dy * dy) + dz * dz


def associate(last, queries, thr, nearby, corner):
    """laserOdometry.cpp:299-361 (corner) or :387-455 (surf) at the identity pose: brute-force nearest neighbour (first index on
    ties), then the literal forward and backward walks with their double break tests.  Rows (query, closest, 2nd, 3rd or -1)."""
    last = np.asarray(last, np.float32)
    ring = last[:, 3].astype(np.int32)
    n = len(last)
    rows = []
    for i, q in enumerate(np.asarray(queries, np.float32)):
        d = sqd(last, q)
        j = int(np.argmin(d))
        if not float(d[j]) < thr:
            continue
        rc = int(ring[j])
        b2, b3, m2, m3 = thr, thr, -1, -1
        for k in range(j + 1, n):
            r = int(ring[k])
            if corner and r <= rc:
                continue
            if r > rc + nearby:
                break
            dk = float(d[k])
            if corner or r <= rc:
                if dk < b2: b2, m2 = dk, k
            elif dk < b3: b3, m3 = dk, k
        for k in range(j - 1, -1, -1):
            r = int(ring[k])
            if corner and r >= rc:
                continue
            if r < rc - nearby:
                break
            dk = float(d[k])
            if corner or r >= rc:
                if dk < b2: b2, m2 = dk, k
            elif dk < b3: b3, m3 = dk, k
        if corner and m2 >= 0:
            rows.append((i, j, m2, -1))
        elif not corner and m2 >= 0 and m3 >= 0:
            rows.append((i, j, m2, m3))
    return rows


def window(rc, nearby, width=64):
    """(dn, up) after the fix: the rings rc - dn .. rc + up pass the break tests `int < rc - N` / `int > rc + N`; both are
    bounded by the context's ring width (64, or 128 in a context of aloam_create_wide above 64 rings)"""
    up = 0
    while up < width and float(rc + up + 1) <= rc + nearby:
        up += 1
    dn = 0
    while dn < width and float(rc - dn - 1) >= rc - nearby:
        dn += 1
    return dn, up


def _unit(rng, planar=False):
    v = rng.normal(size=3)
    if planar:
        v[2] = 0.0
    return v / np.linalg.norm(v)


def _centres(m, radius):
    a = 2 * math.pi * (np.arange(m) + 0.5) / m
    return np.stack([radius * np.cos(a), radius * np.sin(a), np.zeros(m)], axis=1).astype(np.float32)


def _sorted(points):
    """the cloud in ring order (stable): ascending int(intensity) satisfies the invariant aloam_odometry_set_last checks"""
    c = np.array(points, np.float32)
    return np.ascontiguousarray(c[np.argsort(c[:, 3].astype(np.int32), kind="stable")])


def window_scene(seed=0, width=64, rcs=WINDOW_RCS):
    """(last, queries): per closest ring rc of `rcs` two clusters.  Around each query the closest point (ring rc, 5 cm),
    a same-ring point (50 cm) and one point on every other ring of 0 .. width - 1.  Rings on one side sit nearer the farther
    they are from rc (1.98 m at rc +- 1 down to 0.72 m at +- width, in steps of 1.28 m / width), the other side's 2 m farther
    still, so the 2nd (corner) and 3rd (surf) point is the outermost in-window ring of the near side, and rings rc +- (up + 1)
    beyond it hold nearer points than every candidate inside the window.  One cluster has the near side forward, the other
    backward."""
    rng = np.random.default_rng(seed)
    step = 0.02 * 64 / width   # 0.02 exactly at 64 rings
    cases = [(rc, side) for rc in rcs for side in (0, 1)]
    centres = _centres(len(cases), 90.0)
    pts, queries = [], []
    for (rc, side), q in zip(cases, centres):
        queries.append([q[0], q[1], 0.0, rc + 0.03])
        pts.append(list(q[:3] + 0.05 * _unit(rng)) + [rc + 0.01])
        pts.append(list(q[:3] + 0.5 * _unit(rng)) + [rc + 0.02])
        for k in range(1, width + 1):
            near, far = 2.0 - step * k, 4.0 - step * k
            for r, dist in ((rc + k, near if side == 0 else far), (rc - k, far if side == 0 else near)):
                if 0 <= r <= width - 1:
                    pts.append(list(q[:3] + dist * _unit(rng)) + [r + 0.04])
    return _sorted(pts), np.array(queries, np.float32)


def plant(q, target, u):
    """a point p with sqd(p, q) == target exactly (float32): the bulk along the planar unit vector u, the rest on z (q[2] = 0)"""
    q = np.asarray(q, np.float32)
    target = np.float32(target)
    r = math.sqrt(float(target)) * (1.0 - 1e-4)
    p = np.array([q[0] + r * u[0], q[1] + r * u[1], 0.0], np.float32)
    s = sqd(p, q)
    rest = float(target) - float(s)
    assert rest > 0
    dz = np.float32(math.sqrt(rest))
    for _ in range(64):
        p[2] = dz
        got = sqd(p, q)
        if got == target:
            return p
        dz = np.nextafter(dz, np.float32(np.inf) if got < target else np.float32(0.0))
    raise AssertionError("no point at d2 = %r" % target)


def threshold_targets(thr):
    """the float squared distances around the threshold: float(thr) and its two float neighbours"""
    f = np.float32(thr)
    return [np.nextafter(f, np.float32(0.0)), f, np.nextafter(f, np.float32(np.inf))]


def threshold_scene(thr, seed=0):
    """(last, queries): clusters whose closest point lies at a tiny distance or at one of threshold_targets(thr), and whose
    same-ring (surf class 2) and next-ring (corner 2nd, surf class 3) points lie at a target at least as far.  thr must be
    finite in float32."""
    rng = np.random.default_rng(seed)
    t = threshold_targets(thr)
    combos = [(np.float32(float(t[1]) * 1e-3), o) for o in t] + [(c, o) for a, c in enumerate(t) for o in t[a:]]
    radius = max(60.0, 8.0 * math.sqrt(float(t[2])))
    centres = _centres(len(combos), radius)
    pts, queries = [], []
    for (c, o), q in zip(combos, centres):
        queries.append([q[0], q[1], 0.0, 5.03])
        a = rng.uniform(0, 2 * math.pi)
        dirs = [np.array([math.cos(a + k * 2.1), math.sin(a + k * 2.1), 0.0]) for k in range(3)]
        pts.append(list(plant(q, c, dirs[0])) + [5.01])     # closest, ring 5
        pts.append(list(plant(q, o, dirs[1])) + [5.02])     # same ring
        pts.append(list(plant(q, o, dirs[2])) + [6.02])     # next ring
    return _sorted(pts), np.array(queries, np.float32)
