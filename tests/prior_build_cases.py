"""Shared by the CPU and GPU tests of the prior-map build (aloam_prior_map_build): the oracle's build (binning, then the oracle's
VoxelGrid per cube), an independent numpy model of it, clouds that sit on the cube rule's edges, and a writer that puts a built map
into a snapshot of format v1."""
import struct

import numpy as np

W, H, D = 21, 21, 11
NCUBE = W * H * D
STORE = 39424


def cube_of(v, centre):
    """the cube coordinate of the reference's insertion (laserMapping.cpp:741-750) in double, or None where the point is dropped:
    (v + 25) / 50 not finite or beyond int.  Note int() truncates: v + 25 = -50 k lands in cube -k - 1 + centre, not floor's -k"""
    s = float(np.float32(v)) + 25.0
    q = s / 50.0
    if not (-2147483649.0 < q < 2147483648.0):
        return None
    return int(q) + centre - (1 if s < 0 else 0)


def voxel_model(cloud, leaf):
    """pcl::VoxelGrid over one cube with the canonical ties (stable sort by voxel index), float32 sums in sorted order"""
    p = np.ascontiguousarray(cloud, np.float32)
    if len(p) == 0:
        return p.reshape(0, 4)
    inv = np.float32(1.0) / np.float32(leaf)
    mn, mx = p[:, :3].min(axis=0), p[:, :3].max(axis=0)
    d = ((mx - mn) * inv).astype(np.int64) + 1
    if int(d[0]) * int(d[1]) * int(d[2]) > 2**31 - 1:
        return p.copy()
    min_b = np.floor(mn * inv).astype(np.int64)
    div_b = np.floor(mx * inv).astype(np.int64) - min_b + 1
    ijk = (np.floor(p[:, :3] * inv) - min_b.astype(np.float32)).astype(np.int64)
    idx = (ijk[:, 0] + ijk[:, 1] * div_b[0] + ijk[:, 2] * div_b[0] * div_b[1]) & 0xFFFFFFFF
    order = np.argsort(idx, kind="stable")
    out = []
    k = 0
    while k < len(order):
        e = k
        acc = np.zeros(4, np.float32)
        while e < len(order) and idx[order[e]] == idx[order[k]]:
            acc = (acc + p[order[e]]).astype(np.float32)
            e += 1
        out.append(acc / np.float32(e - k))
        k = e
    return np.array(out, np.float32).reshape(-1, 4)


def build_model(corner, surf, line_res, plane_res, centre=(10, 10, 5)):
    """-> ({"corner", "surf", "cube_start"} as OracleBuild.packed, (dropped corner, dropped surf))"""
    out, cs, dropped = {}, np.zeros((2, NCUBE + 1), np.int32), []
    for t, (name, cloud, leaf) in enumerate((("corner", corner, line_res), ("surf", surf, plane_res))):
        cubes = [[] for _ in range(NCUBE)]
        drop = 0
        for p in np.asarray(cloud, np.float32).reshape(-1, 4):
            c = [cube_of(p[a], centre[a]) for a in range(3)]
            if any(v is None for v in c) or not (0 <= c[0] < W and 0 <= c[1] < H and 0 <= c[2] < D):
                drop += 1
                continue
            cubes[c[0] + W * c[1] + W * H * c[2]].append(p)
        parts = [voxel_model(np.array(q, np.float32).reshape(-1, 4), leaf) for q in cubes]
        cs[t, 1:] = np.cumsum([len(q) for q in parts])
        out[name] = np.concatenate(parts)
        dropped.append(drop)
    out["cube_start"] = cs
    return out, tuple(dropped)


def cube_index_of(cloud, centre):
    """the cube of every point, vectorised (-1 where it is dropped): the rule of cube_of, computed with numpy in double"""
    p = np.asarray(cloud, np.float32).reshape(-1, 4)
    ok = np.ones(len(p), bool)
    ijk = np.zeros((len(p), 3), np.int64)
    with np.errstate(invalid="ignore", over="ignore"):
        for a in range(3):
            s = p[:, a].astype(np.float64) + 25.0
            q = s / 50.0
            fin = (q > -2147483649.0) & (q < 2147483648.0)
            ijk[fin, a] = np.trunc(q[fin]).astype(np.int64) + centre[a] - (s[fin] < 0)
            ok &= fin
    ok &= (ijk[:, 0] >= 0) & (ijk[:, 0] < W) & (ijk[:, 1] >= 0) & (ijk[:, 1] < H) & (ijk[:, 2] >= 0) & (ijk[:, 2] < D)
    return np.where(ok, ijk[:, 0] + W * ijk[:, 1] + W * H * ijk[:, 2], -1)


class OracleBuild:
    """the oracle's prior-map build: every point binned into its cube (cube_index_of), each cube of each type filtered by the
    oracle's own VoxelGrid (pyoracle.voxel_grid, canonical ties) over its points in input order"""

    def __init__(self, corner, surf, line_res, plane_res, centre=(10, 10, 5)):
        import pyoracle
        self.centre = tuple(int(v) for v in centre)
        self.cubes, self.dropped = {}, []
        for t, (cloud, leaf) in enumerate(((corner, line_res), (surf, plane_res))):
            p = np.ascontiguousarray(cloud, np.float32).reshape(-1, 4)
            cube = cube_index_of(p, self.centre)
            self.dropped.append(int((cube < 0).sum()))
            order = np.argsort(cube, kind="stable")   # input order inside every cube
            cube_sorted = cube[order]
            for c in np.unique(cube_sorted[cube_sorted >= 0]):
                lo, hi = np.searchsorted(cube_sorted, [c, c + 1])
                self.cubes[(t, int(c))] = pyoracle.voxel_grid(p[order[lo:hi]], leaf, pyoracle.SORT_CANONICAL)
        self.dropped = tuple(self.dropped)

    def cube(self, t, i):
        return self.cubes.get((t, i), np.zeros((0, 4), np.float32))

    def packed(self):
        """{"corner", "surf"}: each type's cubes packed in cube order; "cube_start": (2, NCUBE + 1) int32, cube i of type t at
        [cube_start[t, i], cube_start[t, i + 1])"""
        out, cs = {}, np.zeros((2, NCUBE + 1), np.int32)
        for t, name in ((0, "corner"), (1, "surf")):
            parts = [self.cube(t, i) for i in range(NCUBE)]
            cs[t, 1:] = np.cumsum([len(q) for q in parts])
            out[name] = np.concatenate(parts).astype(np.float32).reshape(-1, 4)
        out["cube_start"] = cs
        return out

    def export(self):
        """the ALOAM_EXPORT_MAP order: corner cube i, then surf cube i, for i = 0 .. NCUBE - 1"""
        return np.concatenate([self.cube(t, i) for i in range(NCUBE) for t in (0, 1)]).astype(np.float32).reshape(-1, 4)

    def frozen(self):
        """the map as a pyfrozen.FrozenMap, for the oracle's localising frames"""
        import pyfrozen
        return pyfrozen.FrozenMap.from_cubes(self.centre, self.cubes)


def oracle_build(corner, surf, line_res, plane_res, centre=(10, 10, 5)):
    """-> (OracleBuild, (dropped corner, dropped surf))"""
    m = OracleBuild(corner, surf, line_res, plane_res, centre)
    return m, m.dropped


def edge_clouds(seed=7):
    """points on the cube rule's edges for centre (10, 10, 5): x + 25 exactly 0 and a float below, +-50 (faces), -50 (the int()
    edge), the buffer's outer faces, non-finite coordinates, and values beyond int; plus a few random points inside"""
    rng = np.random.default_rng(seed)
    xs = [-25.0, np.nextafter(np.float32(-25.0), np.float32(-1e9)), 25.0, -75.0, np.nextafter(np.float32(-75.0), np.float32(0)), 475.0,
          np.nextafter(np.float32(525.0), np.float32(0)), 525.0, -525.0, np.nextafter(np.float32(-525.0), np.float32(0)), 1e12, -1e12,
          np.nan, np.inf, -np.inf]
    pts = []
    for x in xs:
        for y in (0.0, -25.0, 25.0):
            pts.append([x, y, 0.0, 1.5])
            pts.append([0.0, x, y, 2.5])
            pts.append([y, 0.0, x, 3.5])
    inside = rng.uniform(-200, 200, (300, 4)).astype(np.float32)
    inside[:, 2] = rng.uniform(-120, 120, 300)
    cloud = np.concatenate([np.array(pts, np.float32), inside])
    return cloud, cloud[::-1].copy()


def far_clouds():
    """points at x + 25 = +-50 000 exactly and around them, with the centres that put them inside the buffer"""
    pts = []
    for x in (49975.0, -50025.0, 49974.0, -50024.0, 50024.0, -50026.0):
        for y in (-0.5, 0.0, 0.5):
            pts.append([x, y, y, 1.0])
    return np.array(pts, np.float32)


def store_counts(packed):
    """(2, NCUBE) counts of a snapshot's store from a packed map: -1 for a cube without points"""
    cs = np.asarray(packed["cube_start"], np.int64)
    n = (cs[:, 1:] - cs[:, :-1]).astype(np.int32)
    return np.where(n > 0, n, -1).astype(np.int32)


def snapshot_with_store(blob, centre, counts, export):
    """a copy of the mapped snapshot `blob` whose store section holds the given centre offsets, counts and points (ALOAM_EXPORT_MAP
    order); the header's total size follows"""
    b = bytearray(bytes(np.asarray(blob, np.uint8).tobytes()))
    nls, nlf = struct.unpack_from("<ii", b, 28)
    s = 256 + 16 * (nls + nlf)
    head = bytearray(b[s:s + STORE])
    struct.pack_into("<3i", head, 0, *centre)
    head[592:592 + 2 * NCUBE * 4] = np.ascontiguousarray(counts, np.int32).tobytes()
    export = np.ascontiguousarray(export, np.float32).reshape(-1, 4)
    struct.pack_into("<q", head, 39408, export.shape[0])
    out = bytearray(b[:s]) + head + export.tobytes()
    struct.pack_into("<q", out, 16, len(out))
    return np.frombuffer(bytes(out), np.uint8)
