"""Scenes of the per-row records' edge-case tests (tests/test_gpu_track_edges.py, checked on the CPU by
tests/test_oracle_track_edges.py): the stack sizes of synthetic scans that steer k_track_score's staging, the crafted thin-map
scenes that put one stack point of a real scan on the query of a walk scene of tests/reloc_cases.py, the schedules of the row-table
calls and the scan whose less-flat stack filter overflows its key.

Every scan here is a raw scan of trajectory 0 (the world of tests/track_cases.py) or that scan with a few returns moved along their
rays.  Stack sizes come from the oracle's features and voxel filter; the GPU tests hold the device's n_stack to them."""
import numpy as np

import pyoracle
import reloc_cases as RC

SEED_OFF = 50   # trajectory 0 of lane_refs.traj
BIG = 1 << 20   # max_score_points above every stack
_SCANS, _STACKS = {}, {}


def raw_scan(synth, sensor, n_az, index):
    key = (sensor, n_az, index)
    if key not in _SCANS:
        _SCANS[key] = synth.scan(sensor, index, seed=synth.BASE_SEED + SEED_OFF, n_az=n_az)
    return _SCANS[key]


def stacks(synth, sensor, n_az, index, leaves):
    """(n_c, n_s): the oracle's stack sizes of the scan at (line_res, plane_res)"""
    key = (sensor, n_az, index, tuple(leaves))
    if key not in _STACKS:
        ns, _, mr = synth.SENSORS[sensor][:3]
        f = pyoracle.Features(raw_scan(synth, sensor, n_az, index), ns, mr)
        _STACKS[key] = (len(pyoracle.voxel_grid(f.less_sharp, leaves[0])), len(pyoracle.voxel_grid(f.less_flat, leaves[1])))
    return _STACKS[key]


def resolve_mp(spec, n_c, n_s):
    """max_score_points of a case: an int, or n_c - 1 / n_c / n_c + 1 / above both stacks"""
    return {"nc-1": n_c - 1, "nc": n_c, "nc+1": n_c + 1, "big": BIG}.get(spec, spec)


def staging(n_c, n_s, mp):
    """(m_c, m): scoring points of the corner stack and in all"""
    m_c = min(n_c, mp)
    return m_c, m_c + min(n_s, mp)


# ------------------------------------------------------------------------------------------------------- A. staging and records
# (sensor, n_az, scan index, max_score_points).  VLP-16 at 60 azimuth steps has an empty surf stack, so m = m_c = max_score_points
# walks m through 1, 31 .. 513; at 900 steps both stacks are larger than 257, so m_c = max_score_points = 255 / 256 / 257 puts the
# type switch at lane 31 / 0 / 1 of a warp with surf points after it; HDL-32 at 100 steps has a surf stack of 84 points.
DEFAULT_LEAVES = (0.2, 0.4)
STAGE_CASES = [("VLP-16", 60, 3, mp) for mp in (1, 31, 32, 33, 255, 256, 257, 513)] + \
              [("VLP-16", 900, 3, mp) for mp in (1, 255, 256, 257, "nc-1", "nc", "nc+1", "big")] + \
              [("HDL-32", 100, 3, mp) for mp in (31, 33, 83, 84, 85, "big")]
STAGE_M = (1, 31, 32, 33, 255, 256, 257, 513)
STAGE_MC_RES = (0, 1, 31)
# the largest stack the synthetic sensors reach: an HDL-64 scan at 4000 azimuth steps with a 5 cm plane leaf (the less-flat cloud
# is already thinned to one point per 0.2 m voxel per ring, so its size is bounded by the rings' length), scored subsampled
LARGE_CASE = ("HDL-64", 4000, 3, (0.4, 0.05), 30000)
LARGE_MIN = 30000
# the 16-lane localising step: lane -> (n_az, scan index, arming).  Lane 0 holds the smallest stacks and lane 15 the largest (the
# grid is sized from host bounds, not from any record); lane 3 is armed off the map, the others at the scan's map pose
WIDE_LANES = [(60, 1), (60, 4), (100, 2), (100, 5), (200, 0), (200, 6), (400, 1), (400, 8), (900, 2), (900, 7), (1800, 3),
              (1800, 9), (4000, 3), (4000, 5), (4000, 6), (4000, 0)]
WIDE_OFF = 3


# ------------------------------------------------------------------------------------------------ B. crafted thin-map scenes
SCENE_SCAN = ("VLP-16", 900, 3)
TINY_SQ = float(np.nextafter(np.float32(0), np.float32(1)))   # the smallest positive float


def scan_stacks(synth, leaves=(RC.WALK_LEAF, RC.WALK_LEAF), scan=SCENE_SCAN):
    """the oracle's (corner, surf) stacks of the scene scan at the walk leaves"""
    sensor, n_az, index = scan
    ns, _, mr = synth.SENSORS[sensor][:3]
    f = pyoracle.Features(raw_scan(synth, *scan), ns, mr)
    return pyoracle.voxel_grid(f.less_sharp, leaves[0]), pyoracle.voxel_grid(f.less_flat, leaves[1])


def pick(n_c, t, lane, n):
    """the index in stack t (n points) of a point whose scoring position (i, or n_c + i for surf) falls on `lane` of its warp,
    past the first two warps of its type"""
    off = 0 if t == 0 else n_c
    i = 64 + (lane - (off + 64)) % 32
    assert i < n, (i, n)
    return i


def arming(query, p, offset=(0.0, 0.0, 0.0)):
    """identity rotation and t = query - p (+ offset), in double: p moved by it lands on query exactly when the offset is 0"""
    t = np.asarray(query, np.float32)[:3].astype(np.float64) - np.asarray(p, np.float32)[:3].astype(np.float64) + np.asarray(offset)
    return np.r_[0.0, 0.0, 0.0, 1.0, t]


def exact_scene(seed=2):
    """a walk scene without an inlier at WALK_SQ plus a map point exactly on the query (d2 = 0): an inlier at the smallest
    positive inlier_sq, where the nearest other point (at float d2 >= 0.75) is not"""
    s = RC.walk_scene(None, 0, 1200, seed=seed)
    q = s["query"]
    keep = ~(RC.voxels_of(s["map"], RC.WALK_LEAF) == RC.voxels_of(q, RC.WALK_LEAF)[0]).all(1)
    m = np.concatenate([s["map"][keep], q.copy()])
    m[:, 3] = 7.0
    return {"query": q, "map": m, "d2": RC.sq_d2(m, q[0])}


# (name, scene, inlier_sq, offset, whether the chosen point is an inlier)
def thin_scenes():
    out = []
    for sc in RC.WALK_SCENES:
        s = RC.walk_scene(*sc)
        out.append(("walk-lane%s-flat%d" % (sc[0], sc[1]), s, s["inlier_sq"], (0, 0, 0), sc[0] is not None))
    for below in (False, True):
        s = RC.edge_walk_scene(below)
        out.append(("edge-%s" % ("below" if below else "at"), s, RC.EDGE_WALK_SQ, (0, 0, 0), below))
    s = RC.walk_scene(*RC.WALK_SCENES[-2])
    out.append(("isq-1.0", s, 1.0, (0, 0, 0), True))
    e = exact_scene()
    out.append(("isq-tiny-exact", e, TINY_SQ, (0, 0, 0), True))
    s = RC.walk_scene(*RC.WALK_SCENES[0])
    out.append(("isq-tiny-miss", s, TINY_SQ, (0, 0, 0), False))
    cs = float(RC.MAP_CELL)
    far = [(1e4, 0, 0), (-1e4, 0, 0), (0, 0, 1e30), (-1e30, -1e30, -1e30), (2.0**20 * cs, 0, 0), (0, 2.0**20 * cs, 0),
           (0, 0, 2.0**20 * cs), (0, -cs, 2.0**21 * cs)]
    for off in far:
        out.append(("far-%g-%g-%g" % off, s, s["inlier_sq"], off, False))
    return out


OTHER_MAP = np.array([[30.0, 30.0, 30.0, 7.0]], np.float32)   # the other type's map: one far point, so the frame is thin


# ------------------------------------------------------------------------------------------------------------ C. row tables
def schedule(steps, lanes, n_scans, armed, seed=11):
    """ops (steps, lanes) and scan indices: every lane alternates idle gaps and trajectories of 3 .. 12 scans (a START then SCANs
    over consecutive scans); lanes in `armed` ({lane: scan}) start at step 0 or 1 with a trajectory from that scan to the last.  Lane 0 idles first, so records and lanes
    differ in every frame."""
    rng = np.random.default_rng(seed)
    ops = np.zeros((steps, lanes), np.int32)
    idx = np.zeros((steps, lanes), np.int64)
    for l in range(lanes):
        k = 3 if l == 0 else (int(rng.integers(0, 2)) if l in armed else int(rng.integers(0, 4)))
        while k < steps:
            n = int(rng.integers(3, 13))
            first = l in armed and k <= 1
            s0 = armed[l] if first else int(rng.integers(0, n_scans - n + 1))
            n = min(n_scans - s0 if first else n, steps - k, n_scans - s0)
            ops[k, l] = 2
            ops[k + 1:k + n, l] = 1
            idx[k:k + n, l] = np.arange(s0, s0 + n)
            k += n + int(rng.integers(0, 3))
    return ops, idx


def expected_kinds(ops, armed, skip, IDLE=0, MAPPED=1, LOCALISED=2, SKIPPED=3):
    """the row kind of every entry: a START consumes its lane's arming; scan j of a trajectory is mapped when j % skip == 0"""
    kinds = np.zeros(ops.shape, np.int32)
    for l in range(ops.shape[1]):
        arm, loc, j = l in armed, False, 0
        for k in range(ops.shape[0]):
            op = ops[k, l]
            if op == 0:
                continue
            if op == 2:
                loc, arm, j = arm, False, 0
            kinds[k, l] = (LOCALISED if loc else MAPPED) if j % skip == 0 else SKIPPED
            j += 1
    return kinds


# ------------------------------------------------------------------------------------------------------ C5. key overflow
def seg_box(pts, leaf):
    """the segmented filter's two box tests in float (voxel.cu): (PCL's overflow, the key's) of one cloud"""
    p = np.asarray(pts, np.float32)[:, :3]
    mn, mx = p.min(0), p.max(0)
    inv = np.float32(1.0) / np.float32(leaf)
    d = [int(np.float32((mx[a] - mn[a]) * inv)) + 1 for a in range(3)]
    div = [int(np.floor(np.float32(mx[a] * inv))) - int(np.floor(np.float32(mn[a] * inv))) + 1 for a in range(3)]
    pcl = d[0] * d[1] * d[2] > 2**31 - 1
    return pcl, (not pcl) and div[0] * div[1] * div[2] > 2**31


def overflow_scan(synth, index=4, leaf=0.2):
    """scan `index` of the VLP-16 world (900 azimuth steps) with two returns moved out along their rays -- one of the top ring, one
    of the bottom ring at about the opposite heading; far from their neighbours they become less-sharp points -- until the
    less-sharp cloud's box at `leaf` needs more than 31 key bits while PCL's own test passes.  -> (raw, the two indices)"""
    raw = raw_scan(synth, "VLP-16", 900, index).copy()
    el = np.degrees(np.arctan2(raw[:, 2], np.hypot(raw[:, 0], raw[:, 1])))
    ring = np.round((el + 15.0) / 2.0).astype(int)
    az = np.arctan2(raw[:, 1], raw[:, 0])
    mid = np.arange(len(raw)) > len(raw) // 3
    i = int(np.flatnonzero(mid & (ring == 15))[0])
    opp = np.angle(np.exp(1j * (az - az[i] - np.pi)))
    cand = np.flatnonzero(mid & (ring == 0))
    j = int(cand[np.argmin(np.abs(opp[cand]))])
    ns, _, mr = synth.SENSORS["VLP-16"][:3]

    def moved(r):
        out = raw.copy()
        for k in (i, j):
            out[k, :3] = (raw[k, :3].astype(np.float64) * (r / np.linalg.norm(raw[k, :3].astype(np.float64)))).astype(np.float32)
        return out

    far = moved(250.0)
    rest = pyoracle.Features(far, ns, mr).less_sharp[:, :3]
    rest = rest[~(rest[:, None, :] == far[None, [i, j], :3]).all(-1).any(1)]
    for r in np.arange(200.0, 330.0, 0.002):
        out = moved(r)
        if not seg_box(np.r_[rest, out[[i, j], :3]], leaf)[1]:
            continue
        if seg_box(pyoracle.Features(out, ns, mr).less_sharp, leaf)[1]:
            return out, (i, j)
    raise AssertionError("no range puts the less-sharp box in the key-overflow window")
