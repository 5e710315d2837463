"""Crafted cases for mapping trajectories that start on a copy of the prior map (aloam_lane_map_on_prior; cubemap.cu
store_import_body, k_store_seed_tables, k_store_seed_copy; the fit check of the arming): stores with given centre offsets, per-cube
counts and points written into a mapped lane snapshot; the crafted layouts (chunk boundaries of the 1024-thread table walk, cube
kinds, full slab pools, capacity-exact cubes, count-0 cubes); the adjacent doubles of the start position's slack bound; and a host
model of the arming rule.  TEST INFRASTRUCTURE."""
import numpy as np

import cube_edge_cases as E

NCUBE, DIMS = E.NCUBE, E.DIMS
F32 = np.float32
POOL = 1024                    # slabs per cloud type
SLACK = 16                     # cubes the start position may lie outside the buffer on an axis
THREADS = 1024
PER = (NCUBE + THREADS - 1) // THREADS   # cubes per thread of the seed's table walk: 5
LEAVES = (0.2, 0.4)            # line_res, plane_res of a 16-line context (aloam_default_config)
IDENT_Q = np.array(E.IDENT_Q)


def chunk_of(i):
    """the thread of the seed's table walk that holds cube i, and i's place in its chunk"""
    return i // PER, i % PER


def chunk_edges():
    """cubes 0 and NCUBE - 1 and both sides of every chunk boundary (5t - 1, 5t), ascending"""
    out = {0, NCUBE - 1}
    for t in range(1, (NCUBE + PER - 1) // PER):
        out |= {PER * t - 1, PER * t}
    return sorted(out)


def cube_box(idx, cen):
    """the map-frame box [lo, hi) per axis of cube idx under centre offsets cen"""
    ijk = E.ijk_of(idx)
    lo = np.array([50.0 * (ijk[a] - cen[a]) - 25.0 for a in range(3)])
    return lo, lo + 50.0


def cube_centre(ijk, cen):
    return np.array([50.0 * (ijk[a] - cen[a]) for a in range(3)])


def block(ijk):
    """the 5 x 5 x 3 cubes around centre cube ijk that lie inside the buffer (the valid block of a frame that does not shift)"""
    i, j, k = ijk
    return {E.cube_index(a, b, c) for a in range(i - 2, i + 3) for b in range(j - 2, j + 3) for c in range(k - 1, k + 2)
            if 0 <= a < DIMS[0] and 0 <= b < DIMS[1] and 0 <= c < DIMS[2]}


def points_in(rng, idx, cen, n, leaf, pairs=False):
    """n float32 points (with intensities) inside cube idx, 1 m clear of its faces, each in a voxel of its own at `leaf` -- or, with
    pairs, two points in each voxel (n even).  The voxel is the filters' float index floor(p * (1 / leaf))."""
    lo, hi = cube_box(idx, cen)
    inv = F32(1.0) / F32(leaf)
    vlo = np.ceil((lo + 1.0) / leaf).astype(np.int64)
    vhi = np.floor((hi - 1.0) / leaf).astype(np.int64) - 1
    m = n // 2 if pairs else n
    span = vhi - vlo + 1
    flat = rng.choice(int(np.prod(span)), m, replace=False)
    vox = np.stack(np.unravel_index(flat, tuple(int(s) for s in span)), -1) + vlo
    reps = 2 if pairs else 1
    out = np.zeros((m * reps, 4), F32)
    for r in range(reps):
        frac = rng.uniform(0.3, 0.7, (m, 3)) if r == 0 else rng.uniform(0.1, 0.9, (m, 3))
        out[r::reps, :3] = ((vox + frac) * leaf).astype(F32)
    out[:, 3] = rng.uniform(0, 16, len(out)).astype(F32)
    key = np.floor(out[:, :3] * inv).astype(np.int64)
    assert (key[::reps] == vox).all() and (key[reps - 1::reps] == vox).all(), "a point left its voxel"
    return out


class Scene:
    """a store to seed from: centre offsets, counts (2, NCUBE) (-1: no slab), the points of every cube and type, and the init
    T_wmap_wodom (q xyzw, t) of the START"""

    def __init__(self, cen, init_ijk, offset=(3.25, -4.5, 1.75)):
        self.cen = tuple(int(v) for v in cen)
        self.init_ijk = tuple(init_ijk)
        self.t = cube_centre(init_ijk, self.cen) + np.array(offset)
        self.q = IDENT_Q.copy()
        self.counts = np.full((2, NCUBE), -1, np.int32)
        self.cubes = {}

    def put(self, ty, idx, pts):
        self.counts[ty, idx] = len(pts)
        self.cubes[ty, idx] = np.asarray(pts, F32).reshape(-1, 4)

    def points(self):
        """the points in ALOAM_EXPORT_MAP order: cube-major, corner then surf"""
        out = [self.cubes[ty, i] for i in range(NCUBE) for ty in (0, 1) if self.counts[ty, i] > 0]
        return np.concatenate(out) if out else np.zeros((0, 4), F32)

    def clouds(self):
        """the corner and the surf cloud, each in cube order"""
        return [np.concatenate([self.cubes[ty, i] for i in range(NCUBE) if self.counts[ty, i] > 0] or [np.zeros((0, 4), F32)])
                for ty in (0, 1)]

    def block_sizes(self):
        """corner and surf points the START frame's submap holds (the init's valid block)"""
        b = block(self.init_ijk)
        return [int(sum(max(int(self.counts[ty, i]), 0) for i in b)) for ty in (0, 1)]

    def thin(self):
        """the START frame skips its optimisation (laserMapping.cpp:554): corner <= 10 or surf <= 50 in its submap"""
        c, s = self.block_sizes()
        return c <= 10 or s <= 50


def scene_layout(seed=5):
    """(a): cubes 0 and 4850 and both sides of every chunk boundary of the table walk, at centre offsets (7, 12, 4).  Pairs at even
    t hold corner points only, at odd t surf points only, every 97th pair and the two end cubes both; a quarter of the cubes hold one
    point.  Surf cubes in the START's valid block hold one point each, so the frame is thin."""
    rng = np.random.default_rng(seed)
    s = Scene((7, 12, 4), (10, 9, 5))
    b = block(s.init_ijk)
    for idx in chunk_edges():
        t = (idx + 1) // PER
        kinds = (0, 1) if idx in (0, NCUBE - 1) or t % 97 == 0 else ((0,) if t % 2 == 0 else (1,))
        for ty in kinds:
            n = 1 if (idx % 4 == 0 or (ty == 1 and idx in b)) else 2 + idx % 4
            s.put(ty, idx, points_in(rng, idx, s.cen, n, LEAVES[1]))
    return s


def scene_pool(n, seed=6):
    """(b): n cubes of each type hold one point each, spread over the buffer outside the START's valid block (a fixed order of the
    cubes, so the scene of n holds the scene of n - 1), at centre offsets (12, 9, 6)"""
    rng = np.random.default_rng(seed)
    s = Scene((12, 9, 6), (10, 10, 5))
    b = block(s.init_ijk)
    order = [i for i in np.random.default_rng(99).permutation(NCUBE) if i not in b]
    for idx in sorted(int(i) for i in order[:n]):
        for ty in (0, 1):
            s.put(ty, idx, points_in(rng, idx, s.cen, 1, LEAVES[1]))
    return s


def scene_capacity(ty, n, pairs, seed=7):
    """(c): one cube of type ty with n points in the START's own cube (pairs: two points in each voxel of the type's leaf, so the
    START's re-filter halves it), a few one-point cubes of the other type outside the valid block; the frame is thin because the
    block holds no points of the other type"""
    rng = np.random.default_rng(seed)
    s = Scene((10, 10, 5), (9, 11, 5))
    s.put(ty, E.cube_index(*s.init_ijk), points_in(rng, E.cube_index(*s.init_ijk), s.cen, n, LEAVES[ty], pairs))
    for idx in (E.cube_index(2, 3, 1), E.cube_index(18, 17, 9), E.cube_index(15, 4, 2)):
        s.put(1 - ty, idx, points_in(rng, idx, s.cen, 1, LEAVES[1 - ty]))
    return s


def scene_zero(seed=8):
    """(d): the layout of scene_layout with count-0 cubes (a slab, no points) of both types inside and outside the valid block"""
    s = scene_layout(seed)
    b = sorted(block(s.init_ijk))
    zeros = [(0, b[3]), (1, b[3]), (1, b[40]), (0, 17), (1, 2222), (0, 4000), (1, 4000)]
    for ty, idx in zeros:
        s.put(ty, idx, np.zeros((0, 4), F32))
    s.zeros = zeros
    return s


def scene_zero_pool(k, seed=6):
    """the scene_pool(1024) layout with k of its cubes of each type at count 0: a snapshot whose 1024 slabs of each type are all
    taken, k of them by empty cubes, so the seed (which gives a count-0 cube no slab) leaves k slabs of each type free"""
    s = scene_pool(1024, seed)
    held = [int(i) for i in np.flatnonzero(s.counts[0] >= 0)]
    s.zeros = [(ty, i) for i in held[:k] for ty in (0, 1)]
    for ty, i in s.zeros:
        s.put(ty, i, np.zeros((0, 4), F32))
    return s


# ---- the slack bound of the start position

def slack_pairs(axis, cen):
    """((refused, accepted), (accepted, refused)): the adjacent doubles between which the centre cube of a start position goes from
    -17 to -16 and from dims + 15 to dims + 16 on `axis` under centre offset cen"""
    lo = E.straddle(50.0 * (-SLACK - cen) - 25.0, cen)
    hi = E.straddle(50.0 * (DIMS[axis] + SLACK - cen) - 25.0, cen)
    assert [E.cube_coord(v, cen) for v in lo + hi] == [-SLACK - 1, -SLACK, DIMS[axis] + SLACK - 1, DIMS[axis] + SLACK]
    return lo, hi


def slack_inits(cen, base):
    """(axis, side, accepted t, refused t) for each axis and side: base with that coordinate on the slack bound"""
    out = []
    for a in range(3):
        (r0, a0), (a1, r1) = slack_pairs(a, cen[a])
        for side, acc, ref in (("low", a0, r0), ("high", a1, r1)):
            t, u = np.array(base, float), np.array(base, float)
            t[a], u[a] = acc, ref
            out.append((a, side, t, u))
    return out


# ---- the arming rule

def fits(counts, cen, t, max_points):
    """aloam_lane_map_on_prior's verdict on a prior map with per-cube counts (2, NCUBE) (0 and -1: no points), centre offsets cen
    and start position t: 'ok', 'capacity' or 'invalid'"""
    for a in range(3):
        c = E.cube_coord(float(t[a]), cen[a])
        if c < -SLACK or c >= DIMS[a] + SLACK:
            return "invalid"
    cap = (min(16384, max_points), min(65536, max_points))
    for ty in (0, 1):
        n = np.asarray(counts[ty])
        if n.max(initial=0) > cap[ty] or int((n > 0).sum()) > POOL:
            return "capacity"
    return "ok"


# ---- mapped snapshots holding a crafted store

def crafted_blob(base, cen, counts, points, q=E.IDENT_Q, t=(0.0, 0.0, 0.0)):
    """the mapped lane snapshot `base` (taken under the configuration the store is for) with its store replaced: centre offsets
    cen, counts (2, NCUBE) and the points in ALOAM_EXPORT_MAP order, T_wmap_wodom (q, t), frames = 0, an empty valid list, and the
    world pose of its last scan at the identity (so the map position the snapshot check tests is t)"""
    return E.with_store_fields(base, cen=cen, q_wmap=q, t_wmap=t, world=tuple(E.IDENT_Q) + (0.0, 0.0, 0.0), valid=[], frames=0,
                               counts=counts, points=points)


def scene_blob(base, scene, T=None):
    """scene's store as a mapped snapshot; T (7 doubles): its T_wmap_wodom (default the identity)"""
    if T is None:
        return crafted_blob(base, scene.cen, scene.counts, scene.points())
    return crafted_blob(base, scene.cen, scene.counts, scene.points(), T[:4], T[4:])


def split_store(blob):
    """a mapped snapshot's store as {(type, cube): points} for every cube with a slab, and its counts"""
    b, s = E.store_section(blob)
    counts = E.store_counts(blob)
    pts = np.frombuffer(b, F32, offset=s + E.TABLE).reshape(-1, 4)
    out, off = {}, 0
    for i in range(NCUBE):
        for ty in (0, 1):
            n = int(counts[ty, i])
            if n >= 0:
                out[ty, i] = pts[off:off + n]
                off += n
    assert off == len(pts)
    return out, counts


# ---- the seeded oracle

def normalised(q, t):
    """(q, t) as the library normalises an init: q / sqrt(q . q), summed in index order"""
    n2 = 0.0
    for v in q:
        n2 += float(v) * float(v)
    return np.concatenate([np.asarray(q, np.float64) / np.sqrt(n2), np.asarray(t, np.float64)])


def edge_scans(synth, n):
    """scans 0 .. n-1 of a VLP-16 trajectory whose returns end at 40 m: a START frame's features stay in its valid block"""
    return [synth.scan("VLP-16", k, seed=synth.BASE_SEED + 91, n_az=900, max_range=40.0) for k in range(n)]


def seeded_cubemap(orc, scene, T):
    """the oracle's CubeMap holding scene's store at T_wmap_wodom T (7 doubles)"""
    from map_on_prior_seed import seed_cubemap
    cm = orc.CubeMap()
    seed_cubemap(cm, scene.cen, T[:4], T[4:], scene.counts, scene.points())
    return cm


def oracle_frames(orc, synth, cm, scans, odom, leaves=LEAVES):
    """the frames of scans on cm with odometry poses odom, the oracle's features: (map poses, infos)"""
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    feats = []
    for raw in scans:
        f = orc.Features(raw, ns, mr)
        feats.append((f.less_sharp, f.less_flat))
    return oracle_steps(cm, feats, odom, leaves)


def oracle_steps(cm, feats, odom, leaves=LEAVES):
    """the frames of feats ((less_sharp, less_flat) per scan) on cm with odometry poses odom: (map poses, infos)"""
    poses, infos = [], []
    for k, (ls, lf) in enumerate(feats):
        p, info = cm.step(ls, lf, odom[k, :4], odom[k, 4:], *leaves)
        poses.append(p)
        infos.append(info)
    return np.array(poses), infos


def oracle_store(cm):
    """every cube of the oracle's store: {(type, cube): points} for the cubes that hold points"""
    out = {}
    for i in range(NCUBE):
        for ty in (0, 1):
            p = cm.cube(ty, i)
            if len(p):
                out[ty, i] = p
    return out


def start_model(scene, T):
    """the centre offsets and valid list a START frame at T_wmap_wodom T computes (cube_edge_cases.Model, an empty frame)"""
    m = E.Model(cen=scene.cen)
    m.T = (tuple(float(v) for v in T[:4]), tuple(float(v) for v in T[4:]))
    _, st = m.frame(np.zeros((0, 4), F32), np.zeros((0, 4), F32), E.IDENT_Q, (0.0, 0.0, 0.0))
    return st["centre"], st["valid"]
