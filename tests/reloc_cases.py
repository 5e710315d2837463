"""References for relocalisation (aloam_prior_relocalise): the oracle's score of pose hypotheses against a frozen map and an
independent numpy brute force, plus the scenario the recovery tests share.

The oracle score is built from the oracle's own parts: its stack filter (pyoracle.voxel_grid, the call a frozen frame makes),
the subsample, its pointAssociateToMap (pyclouds.associate_to_map) and a 1-NN per type in its kd-tree (pyoracle.KdTree, pinned to
FLANN) over every point of that type in the frozen map.  A scoring point is an inlier when its nearest map point lies at float
d2 < inlier_sq."""
import numpy as np

import pyclouds
import pyfrozen
import pyoracle

# the recovery scenario (chosen by tests/test_oracle_relocalise.py on the oracle alone): a scan of the mapped stretch, a search
# square of +-HALF m at STEP m around a guess GUESS_OFF metres from the true position, N_YAW headings, radius INLIER_SQ
N_MAP, SCAN, OFF_MAP = 10, 4, 200
HALF, STEP, N_YAW = 10.0, 1.0, 72
GUESS_OFF = (3.1, -2.1, 0.0)
INLIER_SQ, MAX_PTS = 0.25, 256
# bars the oracle scenario supports (test_oracle_relocalise.py): the best hypothesis lies within 0.15 m / 0.2 degrees of the true
# pose and scores every scoring point, the best translated or turned copy 381 of 512; a scan from OFF_MAP (160 m on) scores at most
# 329 of 512 anywhere in the search
NEAR_M, NEAR_RAD = 0.3, 0.05
OFF_MAP_RATIO = 0.75
# the crafted map of the d^2 edges
EDGE_SQ = 0.25


def normalised(hyps):
    """q / |q| per row with |q|^2 summed in index order (aloam_lane_localise's routine), t unchanged"""
    h = np.array(hyps, np.float64, copy=True).reshape(-1, 7)
    n2 = np.zeros(len(h))
    for k in range(4):
        n2 = n2 + h[:, k] * h[:, k]
    h[:, :4] = h[:, :4] / np.sqrt(n2)[:, None]
    return h


def subsample(stack, max_pts):
    """scoring point i < m = min(n, max_pts) is stack point floor(i n / m)"""
    n = len(stack)
    m = min(n, int(max_pts))
    return stack[(np.arange(m, dtype=np.int64) * n) // max(m, 1)]


def scoring_points(less_sharp, less_flat, max_pts, line_res, plane_res):
    """(corner, surf) scoring points: the frame's stack filters, then the subsample"""
    return (subsample(pyoracle.voxel_grid(less_sharp, line_res), max_pts), subsample(pyoracle.voxel_grid(less_flat, plane_res), max_pts))


def map_clouds(frozen):
    """every corner / surf point of a FrozenMap, cube by cube"""
    out = []
    for which in (0, 1):
        cubes = [frozen.cube(which, i) for i in range(pyfrozen.NCUBE)]
        out.append(np.concatenate(cubes) if cubes else np.zeros((0, 4), np.float32))
    return out


class FrozenScorer:
    """the oracle's scoring of hypotheses against one frozen map (kd-trees built once)"""

    def __init__(self, frozen):
        self.clouds = map_clouds(frozen)
        self.trees = [pyoracle.KdTree(c) if len(c) else None for c in self.clouds]

    def score(self, less_sharp, less_flat, hyps, inlier_sq, max_score_points, line_res, plane_res, normalise=True):
        pts = scoring_points(less_sharp, less_flat, max_score_points, line_res, plane_res)
        return self.score_points(pts, hyps, inlier_sq, normalise)

    def score_points(self, pts, hyps, inlier_sq, normalise=True):
        H = normalised(hyps) if normalise else np.asarray(hyps, np.float64).reshape(-1, 7)
        out = np.zeros(len(H), np.int64)
        thr = np.float32(inlier_sq)
        for t in (0, 1):
            if self.trees[t] is None or len(pts[t]) == 0:
                continue
            for h in range(len(H)):
                moved = pyclouds.associate_to_map(H[h], pts[t])
                _, d = self.trees[t].knn(moved[:, :3], 1)
                out[h] += int(np.count_nonzero(d[:, 0] < thr))
        return out


def brute_score(map_corner, map_surf, pts, hyps, inlier_sq, chunk=1 << 22):
    """independent model: numpy float32 ((dx^2 + dy^2) + dz^2) against every map point of the type, the transform restated in
    numpy (Eigen's operation order, double, stored as float); scoring points in chunks of about `chunk` point pairs"""
    H = normalised(hyps)
    out = np.zeros(len(H), np.int64)
    thr = np.float32(inlier_sq)
    for cloud, p in ((map_corner, pts[0]), (map_surf, pts[1])):
        if len(cloud) == 0 or len(p) == 0:
            continue
        m = np.asarray(cloud, np.float32)[:, :3]
        step = max(1, chunk // len(m))
        for h, x in enumerate(H):
            with np.errstate(over="ignore", invalid="ignore"):
                q = transform(x, p)
                for i in range(0, len(q), step):
                    d = q[i:i + step, None, :] - m[None, :, :]
                    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
                    out[h] += int(np.count_nonzero((d2 < thr).any(axis=1)))
    return out


def transform(x7, pts):
    """pointAssociateToMap: q * p + t in double (uv = 2 (u x v); v + w uv + u x uv + t), stored as float32"""
    ux, uy, uz, w = x7[:4]
    v = np.asarray(pts, np.float32)[:, :3].astype(np.float64)
    vx, vy, vz = v[:, 0], v[:, 1], v[:, 2]
    uvx, uvy, uvz = uy * vz - uz * vy, uz * vx - ux * vz, ux * vy - uy * vx
    uvx, uvy, uvz = uvx + uvx, uvy + uvy, uvz + uvz
    cx, cy, cz = uy * uvz - uz * uvy, uz * uvx - ux * uvz, ux * uvy - uy * uvx
    return np.stack([((vx + w * uvx) + cx) + x7[4], ((vy + w * uvy) + cy) + x7[5], ((vz + w * uvz) + cz) + x7[6]], axis=1).astype(np.float32)


def yaw_of(q):
    x, y, z, w = q
    return np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))


def search_grid(aloam, true_pose, offset=GUESS_OFF, half=HALF, step=STEP, n_yaw=N_YAW):
    """the recovery search: a lattice around a guess `offset` metres from the true position, n_yaw headings over a full turn
    relative to the true heading's frame (yaw 0 is heading 0 of the map)"""
    q0 = np.asarray(true_pose[:4], np.float64)
    yaw0 = yaw_of(q0)
    h = np.radians(-yaw0) / 2   # q0 with its heading removed: the lattice's headings are absolute
    dq = np.array([0, 0, np.sin(h), np.cos(h)])
    x, y, z, w = q0
    level = np.array([dq[3] * x + dq[0] * w + dq[1] * z - dq[2] * y, dq[3] * y - dq[0] * z + dq[1] * w + dq[2] * x,
                      dq[3] * z + dq[0] * y - dq[1] * x + dq[2] * w, dq[3] * w - dq[0] * x - dq[1] * y - dq[2] * z])
    yaws = np.arange(n_yaw) * (2 * np.pi / n_yaw)
    return aloam.pose_grid(level, np.asarray(true_pose[4:], np.float64) + np.asarray(offset), half, step, yaws)


def oracle_world(synth, sensor="VLP-16", n_extra=6, t=0):
    """the oracle chain over scans 0 .. N_MAP + n_extra - 1 of trajectory t (the GPU tests' lane_refs.traj): (scans, features,
    map poses of the first N_MAP scans, the FrozenMap of the store after them)"""
    import lane_refs as R
    ns, _, mr, line_res, plane_res = synth.SENSORS[sensor]
    scans = R.traj(synth, t, N_MAP + n_extra, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)
    od, cm = pyoracle.Odometry(), pyoracle.CubeMap()
    q = np.array([0, 0, 0, 1.0]); tt = np.zeros(3); qw = q.copy(); tw = tt.copy()
    feats, poses = [], []
    for k, raw in enumerate(scans):
        f = pyoracle.Features(raw, ns, mr)
        feats.append(f)
        if k >= N_MAP:
            continue
        if k > 0:
            q, tt, _ = od.register(f.sharp, f.flat, q, tt)
            qw, tw = pyoracle.integrate_pose(qw, tw, q, tt)
        od.set_last(f.less_sharp, f.less_flat)
        pose, _ = cm.step(f.less_sharp, f.less_flat, qw, tw, line_res, plane_res)
        poses.append(pose)
    cubes = {}
    for which in (0, 1):
        for i in range(pyfrozen.NCUBE):
            c = cm.cube(which, i)
            if len(c):
                cubes[(which, i)] = c
    frozen = pyfrozen.FrozenMap.from_cubes(cm.state()["centre"], cubes)
    return scans, feats, np.array(poses), frozen


def edge_case_clouds():
    """(scan (corner, surf), map corner, map surf) for the d^2 edges at EDGE_SQ: per type, scan points 10 m apart on the x axis
    and map points at float offsets from them: 0.5 along y (d2 == EDGE_SQ exactly), one float below and one above, a neighbour in
    the next cube (x = 25 is a cube boundary), one across a grid cell face (35.00035 m), and a scan point with no neighbour.  Every
    point is alone in its voxel, so neither the stack filter nor the map build moves it."""
    half = np.float32(0.5)
    below, above = np.nextafter(half, np.float32(0)), np.nextafter(half, np.float32(1))
    scan, maps = [], []
    for t in (0, 1):
        z = np.float32(3.0 * t)   # the two types at different heights
        q = [(3, 0, z), (13, 0, z), (23, 0, z), (24.9, 0, z), (35.0, 0, z), (45, 0, z), (-7, 0, z)]
        m = [(3, half, z), (13, below, z), (23, above, z), (25.2, 0, z), (35.3, 0, z), (-7, 0, z + np.float32(0.999))]
        scan.append(np.array([(x, y, zz, 1.0 + t) for x, y, zz in q], np.float32))
        maps.append(np.array([(x, y, zz, 7.0) for x, y, zz in m], np.float32))
    return scan, maps[0], maps[1]


# ---- crafted scenes of the relocaliser's edge cases (tests/test_gpu_reloc_edges.py, checked on the CPU by
# tests/test_oracle_reloc_edges.py).  Every scan point sits alone in its stack voxel, so the stack sizes are the cloud sizes.
MAP_CELL = np.float32(1.0) * (np.float32(1.0) + np.float32(1e-5))   # the prior map's hash-grid cell edge (kMapCell)
INV_CELL = np.float32(1.0) / MAP_CELL
IDENT7 = np.array([0, 0, 0, 1.0, 0, 0, 0])
FAR_POSE = np.array([0, 0, 0, 1.0, 1e4, 0, 0])   # a pose that moves every scene below 10 km away from its map


def cell_of(pts):
    """the grid cell of float32 points as the kernels compute it: floor(v * inv_cs) in float"""
    return np.floor(np.asarray(pts, np.float32)[..., :3] * INV_CELL).astype(np.int64)


def sq_d2(pts, q):
    """float32 ((dx*dx + dy*dy) + dz*dz) of every point to q, the scoring predicate's distance"""
    d = np.asarray(pts, np.float32).reshape(-1, 4)[:, :3] - np.asarray(q, np.float32).reshape(-1)[:3]
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def voxels_of(pts, leaf):
    """the voxel of every point in a grid of edge `leaf` (the stack filter's floor(p * (1 / leaf)) in float)"""
    return np.floor(np.asarray(pts, np.float32)[:, :3] * (np.float32(1.0) / np.float32(leaf))).astype(np.int64)


def alone_in_voxels(pts, leaf):
    v = voxels_of(pts, leaf)
    return len(np.unique(v, axis=0)) == len(v)


def voxel_cloud(ijk, leaf, intensity):
    """points at the centres of the voxels ijk of a grid of edge `leaf`: each alone in its voxel"""
    p = np.zeros((len(ijk), 4), np.float32)
    p[:, :3] = (np.asarray(ijk, np.float64) + 0.5) * float(np.float32(leaf))
    p[:, 3] = intensity
    return p


def random_voxels(rng, n, box, z0=0):
    """n distinct voxels of an x-y centred box of box[0] x box[1] x box[2] voxels starting at voxel height z0"""
    flat = rng.choice(int(np.prod(box)), n, replace=False)
    ijk = np.stack(np.unravel_index(flat, box), 1).astype(np.int64)
    return ijk - np.array([box[0] // 2, box[1] // 2, -z0])


def stage_pool(line_res=0.2, plane_res=0.4, n=5000, seed=3):
    """scan pools (corner, surf) of n points each, every point alone in its voxel, so that the first k points of a pool make a
    stack of exactly k points; and the map (corner, surf): a jittered 60 % of each pool plus clutter.  The corner points span
    40 x 40 x 4 m, the surf points 40 x 40 x 4 m, 6 m higher"""
    rng = np.random.default_rng(seed)
    scan, maps = [], []
    for t, leaf in enumerate((line_res, plane_res)):
        k = int(round(1 / leaf))
        ijk = random_voxels(rng, n, (40 * k, 40 * k, 4 * k), z0=6 * k * t)
        s = voxel_cloud(ijk, leaf, 1.0 + t)
        keep = s[rng.random(n) < 0.6].copy()
        keep[:, :3] += rng.normal(0, 0.25, (len(keep), 3)).astype(np.float32)
        clutter = np.zeros((1000, 4), np.float32)
        clutter[:, :3] = rng.uniform([-20, -20, 6 * t], [20, 20, 6 * t + 4], (1000, 3))
        clutter[:, 3] = 7.0
        scan.append(s)
        maps.append(np.concatenate([keep, clutter]))
    return scan, maps


def stage_hyps(seed=4, n_near=120, n_wide=120):
    """the identity, poses around it (the map's dense part: most points score) and poses anywhere over the pool's extent"""
    rng = np.random.default_rng(seed)
    out = [IDENT7]
    for n, yaw_sd, t_sd in ((n_near, 0.02, 0.3), (n_wide, np.pi, 12.0)):
        yaw = rng.normal(0, yaw_sd, n)
        t = rng.normal(0, t_sd, (n, 3)) * [1, 1, 0.1]
        out.append(np.concatenate([np.zeros((n, 2)), np.sin(yaw / 2)[:, None], np.cos(yaw / 2)[:, None], t], 1))
    return np.concatenate([np.asarray(out[0])[None]] + out[1:])


def subsample_index(n, m):
    """the stack index of every scoring point: floor(i n / m) in 64-bit integers"""
    return (np.arange(m, dtype=np.int64) * n) // m


def big_stack(n=60000, plane_res=0.4, seed=6):
    """a surf scan of n points, each alone in its voxel (a 40 x 40 x 16 m block), a 10-point corner scan, and the map (corner,
    surf): a jittered 60 % of the surf points and the corner points as they are"""
    rng = np.random.default_rng(seed)
    k = int(round(1 / plane_res))
    surf = voxel_cloud(random_voxels(rng, n, (40 * k, 40 * k, 16 * k)), plane_res, 2.0)
    corner = voxel_cloud(random_voxels(rng, 10, (40, 40, 4), z0=200), 0.2, 1.0)
    keep = surf[rng.random(n) < 0.6].copy()
    keep[:, :3] += rng.normal(0, 0.3, (len(keep), 3)).astype(np.float32)
    return (corner, surf), (corner.copy(), keep)


# the 27-cell walk of any_in_block27: lane L probes cell (L % 3 - 1, (L % 9) // 3 - 1, L // 9 - 1) around the query's cell, and
# candidate e of the walk lies in the lane whose inclusive count first exceeds e.  A point alone in its cell has the flat index
# of the counts of the lanes before it.
WALK_CELL = (5, 6, 4)   # the query's cell: every coordinate of the scene lies in [4, 8), where a float's ulp is 2^-21
WALK_LEAF = 0.02        # the leaves of the walk scenes' contexts: the near misses are voxel centres of this grid
WALK_SQ = 0.85          # inlier_sq: a cell's corner lies at d2 0.75 from the query, so every lane can hold the inlier
_LATTICE = {}


def walk_lane(off):
    """the lane that probes cell offset (dx, dy, dz)"""
    dx, dy, dz = off
    return (dz + 1) * 9 + (dy + 1) * 3 + (dx + 1)


def walk_query():
    q = np.zeros((1, 4), np.float32)
    q[0, :3] = (np.array(WALK_CELL, np.float64) + 0.5) * float(MAP_CELL)
    q[0, 3] = 1.0
    return q


def walk_lattice():
    """every WALK_LEAF voxel centre within 1.05 m of the query in each axis: (points, lane or -1, float d2 to the query)"""
    if "l" not in _LATTICE:
        q = walk_query()
        k = int(round(1 / WALK_LEAF))
        lo = np.floor((q[0, :3] - 1.05) * k).astype(np.int64)
        n = int(round(2.1 * k))
        ijk = np.stack(np.meshgrid(*[np.arange(lo[a], lo[a] + n) for a in range(3)], indexing="ij"), -1).reshape(-1, 3)
        p = voxel_cloud(ijk, WALK_LEAF, 7.0)
        off = cell_of(p) - np.array(WALK_CELL)
        ok = (np.abs(off) <= 1).all(axis=1)
        lane = np.where(ok, (off[:, 2] + 1) * 9 + (off[:, 1] + 1) * 3 + (off[:, 0] + 1), -1)
        _LATTICE["l"] = (p, lane, sq_d2(p, q[0]))
    return _LATTICE["l"]


def _spread(total, lanes):
    """total candidates over the lanes, as evenly as possible (earlier lanes take the remainder)"""
    if not lanes:
        assert total == 0, total
        return {}
    base, rem = divmod(total, len(lanes))
    return {L: base + (i < rem) for i, L in enumerate(lanes)}


def walk_scene(inlier_lane, flat, total, inlier_sq=WALK_SQ, seed=0, extra=None):
    """one query point and a map of `total` points around it in the 27 cells: near misses (inlier_sq <= float d2 < 1) and, when
    inlier_lane is not None, one inlier (d2 < inlier_sq) alone in the cell of that lane at flat walk index `flat`.  The near misses
    fill the lanes before the inlier's (flat of them) and after it; the centre cell (lane 13, d2 <= 0.75) holds none unless it
    is the inlier's.  extra: {lane: n} moves n near misses into that lane from the ones after it.  -> dict(query, map, lane,
    d2, counts[27], flat, inlier_sq)"""
    rng = np.random.default_rng(seed)
    p, lane, d2 = walk_lattice()
    thr = np.float32(inlier_sq)
    miss = (d2 >= thr) & (d2 < np.float32(1.0))
    if inlier_lane is None:
        counts = _spread(total, [L for L in range(27) if L != 13])
    else:
        counts = _spread(flat, [L for L in range(inlier_lane) if L != 13])
        after = [L for L in range(inlier_lane + 1, 27) if L != 13]
        counts.update(_spread(total - flat - 1 - sum((extra or {}).values()), after))
    for L, n in (extra or {}).items():
        counts[L] = counts.get(L, 0) + n
    pts = []
    for L, n in sorted(counts.items()):
        cand = np.flatnonzero(miss & (lane == L))
        assert len(cand) >= n, ("lane", L, "holds", len(cand), "near misses, not", n)
        pts.append(p[np.sort(rng.choice(cand, n, replace=False))])
    if inlier_lane is not None:
        cand = np.flatnonzero((d2 < thr) & (lane == inlier_lane))
        pts.append(p[[rng.choice(cand)]])
        counts[inlier_lane] = 1
    m = np.concatenate(pts)
    c = np.zeros(27, np.int64)
    for L, n in counts.items():
        c[L] = n
    off = cell_of(m) - np.array(WALK_CELL)
    return {"query": walk_query(), "map": m, "lane": walk_lane(off.T), "d2": sq_d2(m, walk_query()[0]), "counts": c, "flat": flat,
            "inlier_sq": inlier_sq}


EDGE_WALK_SQ = 0.5625   # 0.75^2, exact in float


def edge_walk_scene(below, seed=1):
    """a dense cell (lane 14, the +x face: 1500 near misses) holding a point at float d2 == EDGE_WALK_SQ exactly (not counted)
    and, when `below`, one at the float just below it (counted); 1000 more near misses in the other lanes.  Lattice points that
    share a voxel with either are dropped, so every point stays alone in its voxel."""
    s = walk_scene(None, 0, 1000, inlier_sq=EDGE_WALK_SQ, seed=seed, extra={14: 1500})
    q = s["query"][0]
    target = np.float32(EDGE_WALK_SQ)
    at = q.copy()
    at[0] = q[0] + np.float32(0.75)
    add = [at]
    if below:
        want = np.nextafter(target, np.float32(0))
        ulp = np.float32(2.0 ** -21)
        found = None
        for k in range(64):   # 0.1 m off the x axis (another voxel), x searched one ulp at a time
            y = q[1] + np.float32(0.1) + np.float32(k) * ulp
            dy = np.float64(y - q[1])
            x0 = q[0] + np.float32(np.sqrt(0.5625 - dy * dy))
            b = np.tile(np.array([x0, y, q[2], 7.0], np.float32), (257, 1))
            b[:, 0] = x0 + np.arange(-128, 129, dtype=np.float32) * ulp
            hit = np.flatnonzero(sq_d2(b, q) == want)
            if len(hit):
                found = b[hit[0]]
                break
        assert found is not None
        add.append(found)
    add = np.array(add, np.float32)
    add[:, 3] = 7.0
    keep = ~(voxels_of(s["map"], WALK_LEAF)[:, None, :] == voxels_of(add, WALK_LEAF)[None, :, :]).all(-1).any(1)
    m = np.concatenate([s["map"][keep], add])
    off = cell_of(m) - np.array(WALK_CELL)
    return {"query": s["query"], "map": m, "lane": walk_lane(off.T), "d2": sq_d2(m, q), "score": int(below), "inlier_sq": EDGE_WALK_SQ}


def line_scene(n=16, slope=0.05, x0=0.0):
    """scan (corner, surf): n points per type 3 m apart on the x axis (surf 5 m higher); map: point j of each type at x + x0 +
    slope * j.  A hypothesis that shifts the scan by s along x scores the points with |s - x0 - slope j| < sqrt(inlier_sq): the
    score grades with s.  The map is thin for a localising frame, so a refined pose is its hypothesis."""
    j = np.arange(n, dtype=np.float64)
    scan, maps = [], []
    for t in (0, 1):
        z = 5.0 * t
        scan.append(np.stack([3.0 * j, 0 * j, 0 * j + z, 0 * j + 1.0 + t], 1).astype(np.float32))
        maps.append(np.stack([3.0 * j + x0 + slope * j, 0 * j, 0 * j + z, 0 * j + 7.0], 1).astype(np.float32))
    return scan, maps


def shift(s):
    return np.array([0, 0, 0, 1.0, s, 0, 0])


def host_top(sc, k):
    """the first k of np.lexsort((index, -score)) for scores >= 0, without sorting the zeros"""
    sc = np.asarray(sc)
    assert (sc >= 0).all()
    nz = np.flatnonzero(sc)
    o = nz[np.lexsort((nz, -sc[nz]))][:k]
    if len(o) < k:
        o = np.concatenate([o, np.flatnonzero(sc == 0)[:k - len(o)]])
    return o


# (inlier lane, its flat walk index, candidates of the walk): the inlier first, at the chunk seams 31 / 32 / 33 and 63 / 64, last,
# behind 1500 near misses, and no inlier at all
WALK_SCENES = [(0, 0, 3000), (13, 31, 2000), (13, 32, 2000), (13, 33, 2000), (13, 63, 2000), (13, 64, 2000), (26, 2999, 3000),
               (13, 1500, 3000), (None, 0, 1200)]
# (corner stack, surf stack, max_score_points) of the staging tests: m = 31, 32, 33, 2047, 2048 (m_c = 2040: the type switch
# inside the last chunk of a stage), 2049, 4096 and 6145 (m_c = 3000: corner points over two stages), 4097
STAGE_CASES = [(13, 18, 1 << 20), (13, 19, 1 << 20), (13, 20, 1 << 20), (1001, 1046, 1 << 20), (2040, 8, 1 << 20), (5000, 1000, 1049),
               (3000, 1096, 1 << 20), (2040, 4000, 2057), (3000, 5000, 3145)]
