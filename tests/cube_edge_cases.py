"""Crafted cases for the mapper's ring buffer (laserMapping.cpp:142-146, :309-529, :741-758; cubemap.cu cube_coord,
mapper_begin_body, rotate_line, cube_ids_body): a host restatement of the centre cube, the six shift loops, the valid list and
the cube of a stored point, with plausible mis-transcriptions of each; the decisions of the cube rule on each axis; poses and
body points crafted to land on them bit for bit; and a writer that relabels a saved lane snapshot's store by a whole number of
cubes.  TEST INFRASTRUCTURE."""
import functools
import struct

import numpy as np

CW, CH, CD = 21, 21, 11
DIMS = (CW, CH, CD)
NCUBE = CW * CH * CD
CEN0 = (10, 10, 5)
HEADER, TABLE = 256, 39424            # sizeof(SnapHeader), sizeof(SnapStore)
F32 = np.float32
IDENT_Q = (0.0, 0.0, 0.0, 1.0)

# the mis-transcriptions the restatement is checked against: each must change at least one crafted case
RULE_MUTATIONS = ("floor", "le_zero", "no_decrement", "float_sum")
MUTATIONS = RULE_MUTATIONS + ("trigger_le3", "axes_kji", "valid_kji")


# ---- Eigen-order quaternion arithmetic in double (quat.cuh; Eigen::Quaternion's operation order), xyzw

def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz)


def qinv(a):
    x, y, z, w = a
    n2 = x * x + y * y + z * z + w * w
    return (-x / n2, -y / n2, -z / n2, w / n2)


def qrot(q, v):
    x, y, z, w = q
    uv = [y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]]
    uv = [u + u for u in uv]
    c2 = [y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0]]
    return [v[k] + w * uv[k] + c2[k] for k in range(3)]


def associate(T, q, t):
    """transformAssociateToMap (:142-146): the map pose x (7 doubles) of odometry pose (q, t) under T = (q_wmap_wodom, t_wmap_wodom)"""
    qm, tm = T
    r = qrot(qm, [float(v) for v in t])
    return tuple(qmul(qm, tuple(float(v) for v in q))) + tuple(r[k] + tm[k] for k in range(3))


def transform_update(x, q, t):
    """transformUpdate (:148-152): T from the map pose x and the odometry pose"""
    qn = qmul(tuple(x[:4]), qinv(tuple(float(v) for v in q)))
    r = qrot(qn, [float(v) for v in t])
    return (qn, tuple(x[4 + k] - r[k] for k in range(3)))


def to_map(pts, x):
    """pointAssociateToMap (:154-163): body points (n, 4) float32 -> map points, the rotation in double, then the cast to float"""
    p = np.asarray(pts, F32)
    ux, uy, uz, w, tx, ty, tz = (float(v) for v in x)
    vx, vy, vz = (p[:, k].astype(np.float64) for k in range(3))
    uvx, uvy, uvz = uy * vz - uz * vy, uz * vx - ux * vz, ux * vy - uy * vx
    uvx, uvy, uvz = uvx + uvx, uvy + uvy, uvz + uvz
    cx, cy, cz = uy * uvz - uz * uvy, uz * uvx - ux * uvz, ux * uvy - uy * uvx
    out = p.copy()
    out[:, 0] = (((vx + w * uvx) + cx) + tx).astype(F32)
    out[:, 1] = (((vy + w * uvy) + cy) + ty).astype(F32)
    out[:, 2] = (((vz + w * uvz) + cz) + tz).astype(F32)
    return out


# ---- the cube rule and its mis-transcriptions

def cube_coord(v, centre, mut=None):
    """int((v + 25.0) / 50.0) + centre, minus one when v + 25.0 < 0 (:314-325, :741-750), v a double (a float point widened)"""
    v = float(v)
    if mut == "float_sum":
        s = float(F32(v) + F32(25.0))
    else:
        s = v + 25.0
    if mut == "floor":
        return int(np.floor(s / 50.0)) + centre
    c = int(s / 50.0) + centre
    neg = s <= 0 if mut == "le_zero" else s < 0
    if neg and mut != "no_decrement":
        c -= 1
    return c


def cube_index(i, j, k):
    return i + CW * j + CW * CH * k


def ijk_of(idx):
    return idx % CW, (idx // CW) % CH, idx // (CW * CH)


def straddle(f, centre, limit=16):
    """(a, b): the two adjacent doubles within `limit` steps of face f between which the cube rule changes (v + 25 is rounded:
    the double before a face can still round onto it, e.g. 125 - 1 ulp + 25 == 150)"""
    down = up = float(f)
    for _ in range(limit):
        b = float(np.nextafter(down, -np.inf))
        if cube_coord(b, centre) != cube_coord(down, centre):
            return b, down
        c = float(np.nextafter(up, np.inf))
        if cube_coord(c, centre) != cube_coord(up, centre):
            return up, c
        down, up = b, c
    raise AssertionError("no decision near %r" % (f,))


def decisions(axis, centre=None):
    """the pose coordinates where the cube rule decides on `axis` (doubles): for every face v + 25 = 50 k whose cubes touch the
    buffer, the face itself and the adjacent pair of doubles the rule's result changes between; then -25.0 and -0.0.  The faces
    where the centre cube becomes 2 / 3 and dims - 4 / dims - 3 are among them (trigger_pairs)"""
    centre = CEN0[axis] if centre is None else centre
    out = []
    for k in range(-centre - 1, DIMS[axis] - centre + 1):
        f = 50.0 * k - 25.0
        a, b = straddle(f, centre)
        out += sorted({a, b, f})
    return out + [-25.0, -0.0]


def trigger_pairs(axis, centre=None):
    """((v2, v3), (v17, v18)): the adjacent doubles between which the centre cube goes from 2 to 3, and from dims - 4 to dims - 3
    (the shift triggers ctr < 3 and ctr >= dims - 3)"""
    centre = CEN0[axis] if centre is None else centre
    lo = straddle(50.0 * (3 - centre) - 25.0, centre)
    hi = straddle(50.0 * (DIMS[axis] - 3 - centre) - 25.0, centre)
    assert [cube_coord(v, centre) for v in lo + hi] == [2, 3, DIMS[axis] - 4, DIMS[axis] - 3]
    return lo, hi


def face_values(axis, centre=None):
    """float32 faces of the stored-point rule on `axis` inside the buffer: x + 25 = 50 k (x = +-25, -75, 50 k - 25)"""
    centre = CEN0[axis] if centre is None else centre
    return [F32(50.0 * k - 25.0) for k in range(-centre + 1, DIMS[axis] - centre)]


# ---- the cube store: centre, shift, valid list, insertion (no re-filter: crafted points never share a voxel)

class Model:
    """laserMapping.cpp's store on thin frames (the pose is the hand-off pose): cubes hold their points as sets"""

    def __init__(self, mut=None, cen=CEN0):
        self.mut = mut
        self.cen = list(cen)
        self.T = (IDENT_Q, (0.0, 0.0, 0.0))
        self.cubes = {}            # (type, cube index) -> list of (n, 4) float32 arrays
        self.valid = []
        self.scrolled = 0          # points dropped by the shifts
        self.stored = []           # (type, map point) of every point a frame inserted

    def coord(self, v, a):
        return cube_coord(v, self.cen[a], self.mut if self.mut in RULE_MUTATIONS else None)

    def _shift(self, a, up):
        """one step of the ring buffer along axis a (:327-509): up -- every cube moves one index up, the top one wraps to 0 emptied"""
        new = {}
        for (ty, idx), pts in self.cubes.items():
            ijk = list(ijk_of(idx))
            ijk[a] += 1 if up else -1
            if 0 <= ijk[a] < DIMS[a]:
                new[(ty, cube_index(*ijk))] = pts
            else:
                self.scrolled += sum(p.shape[0] for p in pts)
        self.cubes = new

    def frame(self, corner, surf, q, t):
        x = associate(self.T, q, t)
        ctr = [self.coord(x[4 + a], a) for a in range(3)]
        lo = (lambda c: c <= 3) if self.mut == "trigger_le3" else (lambda c: c < 3)
        for a in ((2, 1, 0) if self.mut == "axes_kji" else (0, 1, 2)):
            while lo(ctr[a]):
                self._shift(a, True); ctr[a] += 1; self.cen[a] += 1
            while ctr[a] >= DIMS[a] - 3:
                self._shift(a, False); ctr[a] -= 1; self.cen[a] -= 1
        rng = [range(ctr[0] - 2, ctr[0] + 3), range(ctr[1] - 2, ctr[1] + 3), range(ctr[2] - 1, ctr[2] + 2)]
        if self.mut == "valid_kji":
            cubes = [(i, j, k) for k in rng[2] for j in rng[1] for i in rng[0]]
        else:
            cubes = [(i, j, k) for i in rng[0] for j in rng[1] for k in rng[2]]
        self.valid = [cube_index(*c) for c in cubes if all(0 <= c[a] < DIMS[a] for a in range(3))]
        n_sub = [sum(self.count(ty, v) for v in self.valid) for ty in (0, 1)]
        assert not (n_sub[0] > 10 and n_sub[1] > 50), "a crafted frame must be thin: the model does not optimise"
        self.T = transform_update(x, q, t)
        dropped = 0
        for ty, cloud in ((0, corner), (1, surf)):
            if len(cloud) == 0:
                continue
            w = to_map(cloud, x)
            for p in w:
                c = [self.coord(float(p[a]), a) for a in range(3)]
                if all(0 <= c[a] < DIMS[a] for a in range(3)):
                    self.cubes.setdefault((ty, cube_index(*c)), []).append(p[None])
                    self.stored.append((ty, p))
                else:
                    dropped += 1
        return np.array(x), {"centre": tuple(self.cen), "ctr": tuple(ctr), "valid": list(self.valid), "dropped": dropped}

    def count(self, ty, idx):
        return sum(p.shape[0] for p in self.cubes.get((ty, idx), []))

    def cube(self, ty, idx):
        parts = self.cubes.get((ty, idx), [])
        return np.concatenate(parts) if parts else np.zeros((0, 4), F32)

    def held(self):
        return sorted(k for k, v in self.cubes.items() if sum(p.shape[0] for p in v))


def as_set(a):
    """the rows of a cloud in a canonical order (the store's order inside a cube is the voxel filter's, not the model's)"""
    a = np.ascontiguousarray(a, F32).reshape(-1, 4)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


# ---- crafted poses and points

def pose_for(T, q, target, axis, start=None):
    """an odometry translation t such that the map pose of (q, t) under T has x[4 + axis] == target exactly and the other two
    coordinates near start (default 0): the inverse transform, then nextafter steps on t until the host arithmetic hits target"""
    want = [0.0, 0.0, 0.0] if start is None else [float(v) for v in start]
    want[axis] = float(target)
    qm, tm = T
    t = qrot(qinv(qm), [want[k] - tm[k] for k in range(3)])   # x_t = qm * t + tm
    for comp in [axis] + [k for k in range(3) if k != axis]:
        for direction in (np.inf, -np.inf):
            tt = list(t)
            for _ in range(400):
                if associate(T, q, tt)[4 + axis] == target:
                    return np.array(tt)
                tt[comp] = float(np.nextafter(tt[comp], direction))
    raise AssertionError("no odometry translation puts the map pose on %r" % (target,))


def point_on(x, axis, value, others, window=6):
    """a float32 body point whose map coordinate on `axis` is exactly the float `value` under the map pose x, the other two map
    coordinates near `others`; None when the float neighbourhood of the inverse transform holds none"""
    want = [float(v) for v in others]
    want.insert(axis, float(value))
    q = tuple(float(v) for v in x[:4])
    p0 = np.array(qrot(qinv(q), [want[k] - x[4 + k] for k in range(3)]), F32)
    steps = np.arange(-window, window + 1)
    grid = np.stack(np.meshgrid(steps, steps, steps, indexing="ij"), -1).reshape(-1, 3)
    grid = grid[np.argsort(np.abs(grid).sum(1), kind="stable")]
    cand = np.zeros((grid.shape[0], 4), F32)
    for k in range(3):
        vals = {0: p0[k]}
        for s in range(1, window + 1):
            vals[s] = np.nextafter(vals[s - 1], F32(np.inf))
            vals[-s] = np.nextafter(vals[-s + 1], F32(-np.inf))
        cand[:, k] = [vals[int(g)] for g in grid[:, k]]
    w = to_map(cand, x)
    hit = np.flatnonzero(w[:, axis] == F32(value))
    return None if hit.size == 0 else cand[hit[0]]


def quat(axis, angle):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    return tuple(np.concatenate([a * np.sin(angle / 2), [np.cos(angle / 2)]]))


def spread(rng, n, centre, half):
    """n float32 points with intensities, uniform in a box: crafted clouds never put two points in one voxel (checked by callers)"""
    out = np.zeros((n, 4), F32)
    out[:, :3] = rng.uniform(np.asarray(centre) - half, np.asarray(centre) + half, (n, 3))
    out[:, 3] = rng.uniform(0, 16, n)
    return out


def voxel_key(p, leaf=0.8):
    """the voxel of a point at the surf leaf, as the voxel filters compute it (float product, floor)"""
    inv = F32(1.0) / F32(leaf)
    return tuple(int(np.floor(F32(p[k]) * inv)) for k in range(3))


def distinct_voxels(pts, leaf):
    """every point of pts in its own voxel of size leaf (the float index of the voxel filters)"""
    if len(pts) < 2:
        return True
    key = np.floor(np.asarray(pts, F32)[:, :3] * (F32(1.0) / F32(leaf))).astype(np.int64)
    return np.unique(key, axis=0).shape[0] == key.shape[0]


def face_frame(rng, x, n_fill=60):
    """body-frame surf points for map pose x: on every face of every axis inside the buffer and one float either side, plus
    n_fill points spread around the pose.  Faces whose float neighbourhood holds no exact point are skipped; returns (cloud,
    placed faces as (axis, value))"""
    rows, placed = [], []
    for axis in range(3):
        for f in face_values(axis):
            for v in (np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))):
                others = [x[4 + k] + rng.uniform(-200, 200) * (0.25 if k == 2 else 1.0) for k in range(3) if k != axis]
                p = point_on(x, axis, v, others)
                if p is not None:
                    q = p.copy(); q[3] = F32(rng.uniform(0, 16))
                    rows.append(q); placed.append((axis, float(v)))
    fill = spread(rng, n_fill, [0, 0, 0], [150, 150, 20])
    cloud = np.concatenate([np.array(rows, F32).reshape(-1, 4), fill])
    return cloud[rng.permutation(cloud.shape[0])], placed


# ---- relabelled snapshots

def store_section(blob):
    b = np.asarray(blob, np.uint8).tobytes()
    nls, nlf = struct.unpack_from("<ii", b, 28)
    return b, HEADER + 16 * (nls + nlf)


def store_counts(blob):
    b, s = store_section(blob)
    return np.frombuffer(b, np.int32, 2 * NCUBE, s + 592).reshape(2, NCUBE).copy()


def store_centre(blob):
    b, s = store_section(blob)
    return struct.unpack_from("<3i", b, s)


def relabel_fits(counts, valid, d):
    """every cube holding a slab and every valid entry stays inside the buffer when moved by d"""
    idx = [i for i in range(NCUBE) if counts[0, i] >= 0 or counts[1, i] >= 0] + list(valid)
    return all(0 <= ijk_of(i)[a] + d[a] < DIMS[a] for i in idx for a in range(3))


def relabel(blob, d):
    """the mapped lane snapshot `blob` with its store relabelled by d cubes: cen' = cen + d, every cube (its count) and every valid
    entry moved by d, the payload bytes kept (moving every cube by the same d keeps their index order, the order of the payload).
    The same map in the same map frame, held d cubes further into the buffer."""
    b, s = store_section(blob)
    out = bytearray(b)
    cen = struct.unpack_from("<3i", b, s)
    nv = struct.unpack_from("<i", b, s + 12)[0]
    valid = struct.unpack_from("<%di" % nv, b, s + 16)
    counts = store_counts(blob)
    assert relabel_fits(counts, valid, d), "the relabelled store must stay inside the buffer"
    moved = np.full_like(counts, -1)
    off = d[0] + CW * d[1] + CW * CH * d[2]
    held = np.flatnonzero((counts >= 0).any(axis=0))
    moved[:, held + off] = counts[:, held]
    struct.pack_into("<3i", out, s, *(cen[a] + d[a] for a in range(3)))
    struct.pack_into("<%di" % nv, out, s + 16, *(v + off for v in valid))
    out[s + 592:s + 592 + moved.nbytes] = moved.tobytes()
    return np.frombuffer(bytes(out), np.uint8)


def with_store_fields(blob, cen=None, t_wmap=None, q_wmap=None, world=None, warm=None, valid=None, frames=None, counts=None,
                      points=None):
    """a copy of `blob` with header / store fields replaced (for the snapshot checks and crafted stores).  counts ((2, NCUBE), -1:
    no slab) and points (the ALOAM_EXPORT_MAP payload) go together: the point total and the snapshot's size follow them"""
    b, s = store_section(blob)
    out = bytearray(b)
    if counts is not None:
        counts = np.ascontiguousarray(counts, np.int32).reshape(2, NCUBE)
        pts = np.ascontiguousarray(points, F32).reshape(-1, 4)
        assert len(pts) == int(np.maximum(counts, 0).sum()), "points must hold the counted points"
        out = out[:s + TABLE] + bytearray(pts.tobytes())
        out[s + 592:s + 592 + counts.nbytes] = counts.tobytes()
        struct.pack_into("<q", out, s + 39408, len(pts))
        struct.pack_into("<q", out, 16, len(out))
    if valid is not None:
        out[s + 16:s + 528] = bytes(512)
        struct.pack_into("<i", out, s + 12, len(valid))
        struct.pack_into("<%di" % len(valid), out, s + 16, *valid)
    if frames is not None:
        struct.pack_into("<i", out, s + 528, frames)
    if cen is not None:
        struct.pack_into("<3i", out, s, *cen)
    if q_wmap is not None:
        struct.pack_into("<4d", out, s + 536, *q_wmap)
    if t_wmap is not None:
        struct.pack_into("<3d", out, s + 568, *t_wmap)
    if world is not None:
        struct.pack_into("<7d", out, 160, *world)
    if warm is not None:
        struct.pack_into("<7d", out, 104, *warm)
    return np.frombuffer(bytes(out), np.uint8)


# ---- crafted paths: lists of frames (q_odom, t_odom, surf cloud); the corner cloud is always empty, so every frame is thin

ROT = [quat([1.0, -0.4, 0.3], 0.35), quat([-0.2, 0.9, 0.5], -0.6), quat([0.1, 0.2, 1.0], 2.4), IDENT_Q]
LEAVES = (0.4, 0.8)


def _walk(rng, targets, axis, near=60.0, fill=6):
    """a path whose frame j puts map coordinate `axis` of the pose exactly on targets[j] (the other two near 0) under a rotated
    odometry pose, with surf points on every face of every axis that lies inside the buffer and within 110 m of the pose, and one
    float either side of each"""
    m = Model()
    frames, world = [], set()
    for j, v in enumerate(targets):
        q = ROT[j % len(ROT)]
        start = [rng.uniform(-20, 20), rng.uniform(-20, 20), rng.uniform(-5, 5)]
        t = pose_for(m.T, q, v, axis, start)
        x = associate(m.T, q, t)
        assert x[4 + axis] == v
        rows, body = [], set()
        for a in range(3):
            faces = [f for f in face_values(a, m.cen[a]) if abs(float(f) - x[4 + a]) < 110.0]
            for f in rng.permutation(faces):
                for w in (np.nextafter(F32(f), F32(-np.inf)), F32(f), np.nextafter(F32(f), F32(np.inf))):
                    others = [x[4 + k] + rng.uniform(-near, near) * (0.3 if k == 2 else 1.0) for k in range(3) if k != a]
                    p = point_on(x, a, w, others)
                    if p is not None:
                        p = p.copy(); p[3] = F32(rng.uniform(0, 16))
                        kb, kw = voxel_key(p), voxel_key(to_map(p[None], x)[0])
                        if kb not in body and kw not in world:   # no two points ever share a voxel of a filter
                            rows.append(p); body.add(kb); world.add(kw)
        for p in spread(rng, fill, [0, 0, 0], [near, near, 15]):
            kb, kw = voxel_key(p), voxel_key(to_map(p[None], x)[0])
            if kb not in body and kw not in world:
                rows.append(p); body.add(kb); world.add(kw)
        cloud = np.array(rows, F32).reshape(-1, 4)
        cloud = cloud[rng.permutation(cloud.shape[0])]
        m.frame(np.zeros((0, 4), F32), cloud, q, t)
        frames.append((np.array(q), t, cloud))
    return frames


DECISION_PATHS = tuple("%s_%d" % (kind, a) for a in range(3) for kind in ("decisions", "trigger_low", "trigger_high"))


@functools.lru_cache(maxsize=None)
def decision_paths():
    """name -> frames: per axis, every decision of decisions() in a shuffled order (the pose walks across the buffer, shifting
    where it must), and per axis and side the two trigger values in both orders from a fresh store.  Built once, on first use"""
    rng = np.random.default_rng(2024)
    paths = {}
    for a in range(3):
        vals = [v for v in decisions(a) if v != 0.0]
        # -0.0 first: a fresh store's T is the identity, so the map pose is the odometry pose (x = -0.0 + 0.0 = +0.0)
        paths["decisions_%d" % a] = _walk(rng, [-0.0] + [vals[i] for i in rng.permutation(len(vals))], a)
        (v2, v3), (v17, v18) = trigger_pairs(a)
        paths["trigger_low_%d" % a] = _walk(rng, [v3, v2, v3], a)
        paths["trigger_high_%d" % a] = _walk(rng, [v17, v18, v17], a)
    assert tuple(paths) == DECISION_PATHS
    return paths


def faces_missed(paths):
    """the (axis, float value) of every face of face_values() -- every face inside the fresh buffer -- and of the float either side
    of it that no point stored along the paths lies on"""
    want = {(a, float(v)) for a in range(3) for f in face_values(a)
            for v in (np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf)))}
    for frames in paths.values():
        m, _ = run_model(frames)
        for _, p in m.stored:
            want -= {(a, float(p[a])) for a in range(3)}
    return want


JUMPS = (1, 2, 17, 20, 21, 22, 40)
JUMP_PATHS = tuple("jump_%s_%d" % (name, n) for n in JUMPS for name in ("i", "j", "k", "diag"))


@functools.lru_cache(maxsize=None)
def jump_paths():
    """name -> frames: a store with points in the cubes around the start, then one frame that jumps n cubes along an axis or the
    diagonal (both signs), then a frame back near the start"""
    rng = np.random.default_rng(77)
    paths = {}
    for n in JUMPS:
        for name, d in (("i", (1, 0, 0)), ("j", (0, -1, 0)), ("k", (0, 0, 1)), ("diag", (-1, 1, -1))):
            t1 = np.array(d, float) * 50.0 * n + [3.25, -4.5, 1.75]
            q = ROT[n % 3]
            frames = [(np.array(IDENT_Q), np.array([0.5, 0.25, -0.5]), spread(rng, 40, [0, 0, 0], [120, 120, 60])),
                      (np.array(q), t1, spread(rng, 40, [0, 0, 0], [120, 120, 60])),
                      (np.array(ROT[1]), np.array([10.0, -5.0, 2.0]), spread(rng, 20, [0, 0, 0], [60, 60, 30]))]
            paths["jump_%s_%d" % (name, n)] = frames
    return paths


def run_model(frames, mut=None):
    m = Model(mut)
    out = []
    for q, t, surf in frames:
        pose, st = m.frame(np.zeros((0, 4), F32), surf, q, t)
        out.append((pose, st, {k: as_set(m.cube(*k)) for k in m.held()}))
    return m, out
