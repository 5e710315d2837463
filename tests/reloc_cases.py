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


def brute_score(map_corner, map_surf, pts, hyps, inlier_sq):
    """independent model: numpy float32 ((dx^2 + dy^2) + dz^2) against every map point of the type, the transform restated in
    numpy (Eigen's operation order, double, stored as float)"""
    H = normalised(hyps)
    out = np.zeros(len(H), np.int64)
    thr = np.float32(inlier_sq)
    for cloud, p in ((map_corner, pts[0]), (map_surf, pts[1])):
        if len(cloud) == 0 or len(p) == 0:
            continue
        m = np.asarray(cloud, np.float32)[:, :3]
        for h, x in enumerate(H):
            q = transform(x, p)
            d = q[:, None, :] - m[None, :, :]
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
