"""Crafted cases for cube growth's slab allocator (cubemap.cu take_run, cube_insert_body phases 1-4, rotate_line,
store_import_body): a host model of a growth-on lane store on thin frames -- the ring buffer of cube_edge_cases.Model, the run
allocator of test_oracle_cube_growth (Pool, run_order, max_order, pack) -- with plausible mis-transcriptions of each rule, and
scenarios whose pools are exactly tight: wraps that free runs of 2-256 slabs, four runs freed in one bitmap word by one shift
step, the whole-pool run, competing growths, the deferred free, a retry after a wrap, growth by two orders in one insert and
restarts on a fragmented pool.  Every scenario runs from a restored snapshot or from aloam_mapper_reset on lane 0 of the host
API (aloam_mapper_step).  TEST INFRASTRUCTURE."""
import functools
import hashlib
import struct

import numpy as np

import cube_edge_cases as E
import test_lane_snapshot_format as F
from test_oracle_cube_growth import POOL, Pool, max_order, pack, run_order

F32 = np.float32
LEAF = 1e-4                 # every stack filter passes its input through unchanged (see passes_through)
EMPTY = np.zeros((0, 4), F32)
IDENT = np.array(E.IDENT_Q)

# the mis-transcriptions the model is checked against: each must change the outcome of at least one scenario
MUTATIONS = ("no_free_on_wrap", "free_first_word", "eager_free", "cube_index_order", "unaligned_first_fit", "grow_one_order",
             "fail_frees_run", "restart_keeps_pool")


def passes_through(cloud, leaf=LEAF):
    """the stack filter returns `cloud` unchanged and in its order: PCL's "leaf size is too small" exit (voxel.cu seg_keys_body:
    the float32 extent of the cloud over the leaf plus one, per axis, multiplied in 64 bits past INT_MAX).  A single point is its
    own voxel.  A product past 2^63 would wrap (and the device refuses the frame), so crafted frames stay below it"""
    if len(cloud) < 2:
        return True
    p = np.asarray(cloud, F32)[:, :3]
    inv = F32(1.0) / F32(leaf)
    d = [int(F32(p[:, a].max() - p[:, a].min()) * inv) + 1 for a in range(3)]
    assert d[0] * d[1] * d[2] < 2 ** 63, "the extent product of a crafted frame must not wrap"
    return d[0] * d[1] * d[2] > 2 ** 31 - 1


class _Pool(Pool):
    """Pool with a vectorised take (the same block) and the unaligned take of a mutation"""

    def take(self, o):
        n = 1 << o
        free = np.flatnonzero(~self.used.reshape(-1, n).any(axis=1))
        if free.size == 0:
            return -1
        s = int(free[0]) * n
        self.used[s:s + n] = True
        return s

    def take_any(self, o):
        """unaligned_first_fit: the first free block of 2^o slabs at any offset"""
        n = 1 << o
        for s in range(POOL - n + 1):
            if not self.used[s:s + n].any():
                self.used[s:s + n] = True
                return s
        return -1


class Model(E.Model):
    """a lane store with growth on or off on thin frames: cube_edge_cases.Model's poses, shifts and cubes, plus per type a slab
    pool and the run (first slab, order) of every cube that holds one"""

    def __init__(self, caps, growth, mut=None, strict=True):
        self.gmut = mut
        self.strict = strict     # the scenario rules: stack filters that pass through, no point in a valid cube
        self.caps = tuple(caps)
        self.reset(growth)

    def reset(self, growth):
        """a fresh START (aloam_mapper_reset): centre, T and cubes of a new trajectory, every slab free, runs of up to the largest
        order of the setting `growth`"""
        keep = self.gmut == "restart_keeps_pool" and hasattr(self, "pools")
        E.Model.__init__(self)
        self.top = [max_order(c) if growth else 0 for c in self.caps]
        if not keep:
            self.pools = [_Pool(), _Pool()]
        self.runs = {}          # (type, cube index) -> (first slab, order)

    def restore(self, counts, cubes, growth):
        """a restored snapshot (store_import_body): counts (2, NCUBE) with -1 for no run, cubes {(type, index): points}; the runs
        as pack() lays them out, the state of a fresh trajectory otherwise"""
        mut, self.gmut = self.gmut, None
        self.reset(growth)
        self.gmut = mut
        for ty in (0, 1):
            runs, used = pack(counts[ty], self.caps[ty])
            assert used <= POOL and all(counts[ty][i] <= self.caps[ty] << self.top[ty] for i in runs)
            self.pools[ty].used[:used] = True
            for i, r in runs.items():
                self.runs[(ty, i)] = r
                if counts[ty][i] > 0:
                    self.cubes[(ty, i)] = [np.asarray(cubes[(ty, i)], F32)]

    def _shift(self, a, up):
        """rotate_line: the wrapped cube's run goes back to the pool"""
        moved = {}
        for (ty, idx), (s, o) in self.runs.items():
            ijk = list(E.ijk_of(idx))
            ijk[a] += 1 if up else -1
            if 0 <= ijk[a] < E.DIMS[a]:
                moved[(ty, E.cube_index(*ijk))] = (s, o)
            elif self.gmut != "no_free_on_wrap":
                n = 1 << o
                if self.gmut == "free_first_word":
                    n = min(n, 32 - s % 32)
                self.pools[ty].used[s:s + n] = False
        self.runs = moved
        E.Model._shift(self, a, up)

    def frame(self, corner, surf, q, t):
        """one thin frame: the pose, shifts and valid list of cube_edge_cases.Model, then the insert of both clouds.  Returns (map
        pose, overflow flag)"""
        x, st = E.Model.frame(self, EMPTY, EMPTY, q, t)
        valid = set(st["valid"])
        assert not self.strict or not any(i in valid for _, i in self.held()), "a valid cube with points would be re-filtered"
        flag = False
        for ty, cloud in ((0, corner), (1, surf)):
            flag |= self._insert(ty, np.asarray(cloud, F32).reshape(-1, 4), x, valid)
        return x, flag

    def _insert(self, ty, cloud, x, valid):
        """cube_insert_body: count, list the cubes that need a run in the order of their first stack point, serve each from the
        lowest aligned free block (a cube that is not served keeps its old run), free the old runs, append in stack order up to
        each run's capacity"""
        if len(cloud) == 0:
            return False
        assert not self.strict or passes_through(cloud), "a crafted frame must span more than the stack filter's index range on every axis"
        cap, pool = self.caps[ty], self.pools[ty]
        ceiling = cap << self.top[ty]
        w = E.to_map(cloud, x)
        cube = []
        for p in w:
            c = [self.coord(float(p[a]), a) for a in range(3)]
            if not all(0 <= c[a] < E.DIMS[a] for a in range(3)):
                assert not self.strict, "crafted points stay inside the buffer"
                cube.append(-1)              # outside the buffer: dropped by the cube rule, not flagged
                continue
            cube.append(E.cube_index(*c))
            assert not self.strict or cube[-1] not in valid, "a crafted point never lands in a valid cube"
        gets, first = {}, {}
        for i, c in enumerate(cube):
            if c < 0:
                continue
            gets[c] = gets.get(c, 0) + 1
            first.setdefault(c, i)
        want = {c: run_order(min(self.count(ty, c) + gets[c], ceiling), cap) for c in gets}
        need = [c for c in gets if (ty, c) not in self.runs or want[c] > self.runs[(ty, c)][1]]
        need.sort(key=(lambda c: c) if self.gmut == "cube_index_order" else (lambda c: first[c]))
        flag, old_runs = False, []
        for c in need:
            old = self.runs.get((ty, c))
            o = want[c]
            if self.gmut == "grow_one_order":
                o = 0 if old is None else min(o, old[1] + 1)
            s = pool.take_any(o) if self.gmut == "unaligned_first_fit" else pool.take(o)
            if s < 0:
                flag = True
                if self.gmut == "fail_frees_run" and old is not None:
                    pool.free(*old)
                    del self.runs[(ty, c)]
                    self.cubes.pop((ty, c), None)
                continue
            self.runs[(ty, c)] = (s, o)
            if old is not None:
                if self.gmut == "eager_free":
                    pool.free(*old)
                else:
                    old_runs.append(old)
        for r in old_runs:
            pool.free(*r)
        cube = np.asarray(cube)
        for c in gets:                       # each cube's points in stack order, up to its run's capacity
            r = self.runs.get((ty, c))
            room = 0 if r is None else max(0, (cap << r[1]) - self.count(ty, c))
            mine = w[cube == c]
            flag |= room < len(mine)
            if room:
                self.cubes.setdefault((ty, c), []).append(mine[:room])
        return flag

    def totals(self):
        return tuple(sum(self.count(ty, i) for t, i in self.held() if t == ty) for ty in (0, 1))

    def payload(self):
        """the ALOAM_EXPORT_MAP export: cube by cube, corner before surf, each cube's points in store order"""
        parts = [self.cube(ty, i) for i in range(E.NCUBE) for ty in (0, 1) if self.count(ty, i)]
        return np.concatenate(parts) if parts else EMPTY


# ---- crafted stores and frames

def at(ijk, rng, n=1, cen=E.CEN0):
    """n float32 map points inside cube (i, j, k) of a store with centre offsets cen, on a 1/64 m grid (exact in float and after
    adding a translation that is a multiple of 50 m), within 10 m of the cube's centre in x and y.  In z they hug the face that
    planes 7 | 8 and 9 | 10 share (3 m either side), so a frame that opens cubes on both planes of a pair spans 6 m in z and its
    extent product at the 1e-4 m leaf stays far below 2^63"""
    g = rng.integers(-640, 641, (n, 3))
    if ijk[2] in (7, 9):
        g[:, 2] = rng.integers(1408, 1599, n)
    elif ijk[2] in (8, 10):
        g[:, 2] = rng.integers(-1600, -1407, n)
    out = np.zeros((n, 4), F32)
    for a in range(3):
        out[:, a] = (ijk[a] - cen[a]) * 50.0 + g[:, a] / 64.0
    out[:, 3] = rng.integers(0, 1024, n) / 64.0
    return out


def cubes_of(ks, i_range=range(1, 20)):
    """the cube coordinates (relative to the first centre CEN0) of planes k in ks, i in i_range: never in the valid window of a
    pose at height 0 (k = 4 .. 6), never on the planes i = 0 and 20 that a one-step shift along i wraps"""
    return [(i, j, k) for k in ks for j in range(E.CH) for i in i_range]


FILL = cubes_of((1, 2, 3))          # one-slab fillers of restored stores (1197 cubes)
NEW = cubes_of((7, 8, 9, 10))       # cubes the frames open (1596 cubes): a frame takes them from one pair, 7 | 8 or 9 | 10
NEW78, NEW910 = NEW[:798], NEW[798:]


class Store:
    """a crafted store: counts (2, NCUBE) and the points of every cube, cubes given by their CEN0 coordinates"""

    def __init__(self):
        self.counts = np.full((2, E.NCUBE), -1, np.int32)
        self.pts = {}

    def put(self, ty, ijk, pts):
        i = E.cube_index(*ijk)
        assert self.counts[ty, i] < 0
        self.counts[ty, i] = len(pts)
        self.pts[(ty, i)] = np.asarray(pts, F32)

    def payload(self):
        parts = [self.pts[(ty, i)] for i in range(E.NCUBE) for ty in (0, 1) if self.counts[ty, i] > 0]
        return np.concatenate(parts) if parts else EMPTY

    def slabs(self, ty, cap):
        return pack(self.counts[ty], cap)[1]


def config(max_points):
    """the context of every scenario: leaves of 1e-4 m, max_points = the slab capacity of both types up to 16384"""
    return dict(n_scans=16, max_points=max_points, max_map_points=200000, line_res=LEAF, plane_res=LEAF)


def template(cfg):
    """a mapped snapshot with an empty store, written from the documented layout with the fingerprint of a context created with
    config(...) = cfg (the other fields at aloam_default_config's values for 16 rings): identity poses, centre (10, 10, 5), no
    "last" clouds"""
    blob = bytearray(F._blob(nls=0, nlf=0, counts=np.full((2, E.NCUBE), -1, np.int32), valid=()))
    struct.pack_into("<iiiiifff", blob, 36, cfg["n_scans"], 0, 1, 2, 4, 0.3, cfg["line_res"], cfg["plane_res"])
    struct.pack_into("<iii", blob, 68, min(16384, cfg["max_points"]), min(65536, cfg["max_points"]), cfg["max_map_points"])
    struct.pack_into("<7d", blob, 104, 0, 0, 0, 1, 0, 0, 0)
    struct.pack_into("<7d", blob, 160, 0, 0, 0, 1, 0, 0, 0)
    return np.frombuffer(bytes(blob), np.uint8)


def snapshot(cfg, store, growth):
    """the template with the store's counts and points, T_wmap_wodom the identity, header byte 220 = growth"""
    b = E.with_store_fields(template(cfg), counts=store.counts, points=store.payload(), q_wmap=E.IDENT_Q, t_wmap=(0.0, 0.0, 0.0))
    out = bytearray(b.tobytes())
    struct.pack_into("<i", out, 220, growth)
    return np.frombuffer(bytes(out), np.uint8)


class Scenario:
    """steps: ("restore", store, growth) | ("reset", growth) | ("frame", t, corner, surf) with identity rotations; `fresh`: the
    steps start from aloam_mapper_reset under growth `growth` (no restore), so the oracle's CubeMap can follow them"""

    def __init__(self, name, max_points, growth=1):
        self.name, self.max_points, self.growth = name, max_points, growth
        self.steps = []

    def restore(self, store, growth=1):
        self.steps.append(("restore", store, growth))
        return self

    def reset(self, growth):
        self.steps.append(("reset", growth))
        return self

    def frame(self, t=(0.0, 0.0, 0.0), corner=EMPTY, surf=EMPTY):
        t = np.asarray(t, float)
        body = [np.asarray(c, F32).reshape(-1, 4).copy() for c in (corner, surf)]
        for b in body:
            b[:, :3] -= t.astype(F32)        # map points given; the pose's translation is exact (multiples of 50 m)
        self.steps.append(("frame", t, body[0], body[1]))
        return self

    @property
    def fresh(self):
        return not any(s[0] == "restore" for s in self.steps)

    @property
    def caps(self):
        return (min(16384, self.max_points), min(65536, self.max_points))


def walk(sc, mut=None):
    """the model over the scenario's steps: yields (step, model, map pose, overflow flag) after every step (pose and flag None for
    a restore or a reset)"""
    m = Model(sc.caps, sc.growth, mut)
    for step in sc.steps:
        if step[0] == "restore":
            m.restore(step[1].counts, step[1].pts, step[2])
            yield step, m, None, None
        elif step[0] == "reset":
            m.reset(step[1])
            yield step, m, None, None
        else:
            _, t, corner, surf = step
            pose, flag = m.frame(corner, surf, IDENT, t)
            yield step, m, pose, flag


def outcome(sc, mut=None):
    """what a scenario predicts, comparable between mutations: per frame the flag, every cube's count and the store's points in
    export order"""
    return [(flag, tuple((k, m.count(*k)) for k in m.held()), hashlib.sha1(m.payload().tobytes()).hexdigest())
            for step, m, _, flag in walk(sc, mut) if step[0] == "frame"]


# ---- the scenarios (cap = the slab capacity; runs of 2^o slabs hold cap << o points)

JUMP = 400.0     # a pose 8 cubes along +x: the centre cube 18 -> one shift towards low indices, plane i = 0 wraps


def _fillers(s, ty, n, rng, skip=()):
    for ijk in [c for c in FILL if c not in skip][:n]:
        s.put(ty, ijk, at(ijk, rng))


def wrap_single_word(extra=False):
    """plane i = 0 (k = 0) holds runs of 16, 8, 4 and 2 slabs; growers on plane i = 5 hold full runs of 8, 4, 2 and 1 slabs; one-slab
    fillers make the pool exactly full.  The jump wraps plane 0; the next frame gives every grower one point, in the stack order 8,
    4, 2, 1 slabs, so each needs twice its run and finds it only in the hole of the same size, at its aligned position.  Their old
    runs come free: 15 new cubes fit and the 16th is flagged.  extra: the jump frame opens one more cube, which takes the lowest
    free slab and splits the 16-slab hole"""
    rng = np.random.default_rng(1)
    cap = 1024
    s = Store()
    for j, o in enumerate((4, 3, 2, 1)):
        s.put(1, (0, j, 0), at((0, j, 0), rng, cap << o))
    growers = [(5, j, 0) for j in range(4)]
    for g, o in zip(growers, (3, 2, 1, 0)):
        s.put(1, g, at(g, rng, cap << o))
    _fillers(s, 1, POOL - 30 - 15, rng)
    assert s.slabs(1, cap) == POOL
    sc = Scenario("wrap_single_word" + ("_extra" if extra else ""), cap).restore(s)
    sc.frame((JUMP, 0, 0), surf=at(NEW[0], rng) if extra else EMPTY)
    sc.frame((JUMP, 0, 0), surf=np.concatenate([at(g, rng) for g in growers]))
    sc.frame((JUMP, 0, 0), surf=np.concatenate([at(c, rng) for c in NEW[1:17]]))
    return sc


def one_word(towards_high, extra=False):
    """four cubes on lines j = 0 .. 3 of the wrapped plane, 8-slab runs, packed after two 16-slab growers into slabs 32 .. 63: one
    bitmap word, freed by four lines of one shift step.  A grower then needs 32 slabs, which only that word holds.  extra: one
    new cube first, in the jump frame"""
    rng = np.random.default_rng(2 + towards_high)
    cap = 1024
    i = 20 if towards_high else 0
    s = Store()
    growers = [(5, 0, 0), (5, 1, 0)]
    for g in growers:
        s.put(1, g, at(g, rng, cap << 4))
    for j in range(4):
        s.put(1, (i, j, 0), at((i, j, 0), rng, cap << 3))
    _fillers(s, 1, POOL - 64, rng)
    assert s.slabs(1, cap) == POOL
    t = (-JUMP if towards_high else JUMP, 0, 0)
    sc = Scenario("one_word_%s%s" % ("high" if towards_high else "low", "_extra" if extra else ""), cap).restore(s)
    sc.frame(t, surf=at(NEW[0], rng) if extra else EMPTY)
    sc.frame(t, surf=at(growers[1], rng))
    return sc


def multi_word(extra=False):
    """runs of 256 and 64 slabs (2^18 and 65536 points) on the wrapped plane, 704 fillers: the wrap frees 320 slabs over 10 words.
    The next frame opens 320 new cubes in a shuffled order (321 with extra): exactly 320 are stored, the first in the stack"""
    rng = np.random.default_rng(4)
    cap = 1024
    s = Store()
    s.put(1, (0, 0, 0), at((0, 0, 0), rng, cap << 8))
    s.put(1, (0, 3, 0), at((0, 3, 0), rng, cap << 6))
    _fillers(s, 1, POOL - 320, rng)
    assert s.slabs(1, cap) == POOL
    sc = Scenario("multi_word" + ("_extra" if extra else ""), cap).restore(s)
    sc.frame((JUMP, 0, 0))
    new = [NEW[k] for k in rng.permutation(400)[:321 if extra else 320]]
    sc.frame((JUMP, 0, 0), surf=np.concatenate([at(c, rng) for c in new]))
    return sc


def whole_pool(extra=False):
    """max_points = 256: the largest run is the whole pool (1024 slabs, 2^18 points).  1. a full 512-slab cube (131072 points)
    takes one more point: its 1024-slab run cannot be taken while it holds half the pool -- flagged, the point dropped;  2. a cube
    of 2^18 points restored on the whole pool: new cubes and the cube itself are flagged;  3. the jump wraps it: 1024 new
    one-slab cubes fit in five frames.  extra: the jump frame opens one more cube, and the last of the 1024 is flagged"""
    rng = np.random.default_rng(5)
    cap = 256
    s1 = Store()
    s1.put(1, (5, 0, 0), at((5, 0, 0), rng, cap << 9))
    s2 = Store()
    s2.put(1, (0, 0, 0), at((0, 0, 0), rng, cap << 10))
    assert s2.slabs(1, cap) == POOL
    sc = Scenario("whole_pool" + ("_extra" if extra else ""), cap).restore(s1)
    sc.frame(surf=at((5, 0, 0), rng))
    sc.restore(s2)
    sc.frame(surf=np.concatenate([at((0, 0, 0), rng), at(NEW[0], rng), at(NEW[1], rng)]))
    sc.frame((JUMP, 0, 0), surf=at(NEW910[-1], rng) if extra else EMPTY)
    for cubes in (NEW78[:256], NEW78[256:512], NEW78[512:768], NEW78[768:], NEW910[:POOL - len(NEW78)]):   # 798 + 226
        sc.frame((JUMP, 0, 0), surf=np.concatenate([at(c, rng) for c in cubes]))
    return sc


def competing(growth, extra=False):
    """two cubes need the last aligned block in one insert.  Growth on: a restored pool with slabs 1022 and 1023 free, cubes A and
    B (B of the higher index) full at one slab, B's point first in the stack: B grows, A is flagged and keeps its 1024 points.
    Growth off, from aloam_mapper_reset: 1023 new cubes in two frames, then A and B new, B first: B takes the last slab.  extra: one more new
    cube takes the free slab a frame earlier"""
    rng = np.random.default_rng(6 + growth)
    cap = 1024
    A, B = (4, 0, 0), (6, 0, 0)
    sc = Scenario("competing_%s%s" % ("on" if growth else "off", "_extra" if extra else ""), cap, growth)
    if growth:
        s = Store()
        s.put(1, A, at(A, rng, cap))
        s.put(1, B, at(B, rng, cap))
        _fillers(s, 1, POOL - 4, rng)
        assert s.slabs(1, cap) == POOL - 2
        sc.restore(s)
    else:
        sc.frame(surf=np.concatenate([at(c, rng) for c in NEW78]))
        sc.frame(surf=np.concatenate([at(c, rng) for c in NEW910[:POOL - 1 - len(NEW78)]]))
    if extra:
        sc.frame(surf=at(NEW910[-1], rng))
    sc.frame(surf=np.concatenate([at(B, rng), at(A, rng)]))
    sc.frame(surf=np.concatenate([at(B, rng), at(A, rng)]))
    return sc


def deferred(extra=False):
    """cube A (full at one slab) grows into the only free block (slabs 1022, 1023) while new cube B, later in the stack, needs one
    slab: B is flagged, as A's old slab is freed only once every cube is served.  The next frame gives B that slab.  extra: that
    frame opens cube C before B, and C takes it"""
    rng = np.random.default_rng(8)
    cap = 1024
    A, B = (4, 0, 0), NEW[5]
    s = Store()
    s.put(1, A, at(A, rng, cap))
    _fillers(s, 1, POOL - 3, rng)
    assert s.slabs(1, cap) == POOL - 2
    sc = Scenario("deferred" + ("_extra" if extra else ""), cap).restore(s)
    sc.frame(surf=np.concatenate([at(A, rng), at(B, rng)]))
    sc.frame(surf=np.concatenate(([at(NEW[0], rng)] if extra else []) + [at(B, rng)]))
    return sc


def retry(extra=False):
    """a full pool: cube A (one full slab) gets 512 points and cannot grow -- flagged, its 1024 points kept.  The jump wraps a
    2-slab cube on plane 0; A's next points grow it into that block, after its first 1024.  extra: one new cube in the jump frame"""
    rng = np.random.default_rng(9)
    cap = 1024
    A = (5, 0, 0)
    s = Store()
    s.put(1, (0, 0, 0), at((0, 0, 0), rng, cap << 1))
    s.put(1, A, at(A, rng, cap))
    _fillers(s, 1, POOL - 3, rng)
    assert s.slabs(1, cap) == POOL
    sc = Scenario("retry" + ("_extra" if extra else ""), cap).restore(s)
    sc.frame(surf=at(A, rng, 512))
    sc.frame((JUMP, 0, 0), surf=at(NEW[0], rng) if extra else EMPTY)
    sc.frame((JUMP, 0, 0), surf=at(A, rng, 512))
    return sc


def two_orders(extra=False):
    """max_points = 20000: corner slabs of 16384 points, frames of 20000, a corner pool with slabs 1018 .. 1023 free.  A full
    one-slab corner cube gets 20000 points and moves straight to a 4-slab run (36384 points, slabs 1020 .. 1023); a new corner cube
    gets 20000 and takes 2 slabs (1018, 1019).  Nothing is dropped.  extra: one more filler holds slab 1018, so the new cube finds
    no aligned block of two"""
    rng = np.random.default_rng(10)
    cap = 16384
    A = (5, 0, 0)
    s = Store()
    s.put(0, A, at(A, rng, cap))
    _fillers(s, 0, POOL - 6 - (0 if extra else 1), rng)
    assert s.slabs(0, cap) == POOL - 6 + extra
    sc = Scenario("two_orders" + ("_extra" if extra else ""), 20000).restore(s)
    sc.frame(corner=at(A, rng, 20000))
    sc.frame(corner=at(NEW[0], rng, 20000))
    return sc


def unaligned_holes(extra=False):
    """a full pool whose wrap frees slabs 1 and 2: two free slabs but no aligned block of two.  Cube A (one full slab) gets a point:
    flagged, its 1024 points kept; the next frame's two new cubes take slabs 1 and 2.  extra: the jump frame opens one more cube"""
    rng = np.random.default_rng(13)
    cap = 1024
    A = (5, 20, 3)
    s = Store()
    for ijk in ((1, 0, 0), (0, 1, 0), (0, 2, 0), (1, 3, 0)):   # slabs 0 .. 3 in cube order; plane 0 holds slabs 1 and 2
        s.put(1, ijk, at(ijk, rng))
    s.put(1, A, at(A, rng, cap))
    _fillers(s, 1, POOL - 5, rng, skip=(A,))
    assert s.slabs(1, cap) == POOL
    sc = Scenario("unaligned_holes" + ("_extra" if extra else ""), cap).restore(s)
    sc.frame((JUMP, 0, 0), surf=at(NEW[5], rng) if extra else EMPTY)
    sc.frame((JUMP, 0, 0), surf=at(A, rng))
    sc.frame((JUMP, 0, 0), surf=np.concatenate([at(c, rng) for c in NEW[:2]]))
    return sc


def restart_store():
    """a fragmented growth-on store: cubes of plane i = 0 and i = 1 alternate on slabs 0 .. 125 (one-slab runs in cube order),
    so the wrap of plane 0 leaves every other slab free"""
    rng = np.random.default_rng(11)
    s = Store()
    for k in (1, 2, 3):
        for j in range(E.CH):
            for i in (0, 1):
                s.put(1, (i, j, k), at((i, j, k), rng))
    return s, rng


def restart(growth, fresh=False):
    """the fragmented store after the wrap, then aloam_mapper_reset under `growth` (fresh: a new context, nothing before): 798
    new one-slab cubes, then 227 more, of which the last is flagged: exactly 1024 fit"""
    s, rng = restart_store()
    sc = Scenario("restart_%s%s" % ("on" if growth else "off", "_fresh" if fresh else ""), 1024, growth)
    if not fresh:
        sc.restore(s)
        sc.frame((JUMP, 0, 0))
        sc.reset(growth)
    rng = np.random.default_rng(12)
    sc.frame(surf=np.concatenate([at(c, rng) for c in NEW78]))
    sc.frame(surf=np.concatenate([at(c, rng) for c in NEW910[:POOL + 1 - len(NEW78)]]))
    return sc


@functools.lru_cache(maxsize=None)
def scenarios():
    out = [wrap_single_word(), wrap_single_word(True), one_word(False), one_word(True), one_word(False, True), one_word(True, True),
           multi_word(), multi_word(True), whole_pool(), whole_pool(True), competing(1), competing(1, True), competing(0),
           competing(0, True), deferred(), deferred(True), retry(), retry(True), unaligned_holes(), unaligned_holes(True),
           two_orders(), two_orders(True), restart(1), restart(0), restart(1, True), restart(0, True)]
    return {sc.name: sc for sc in out}
