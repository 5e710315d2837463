"""The lost-track scenario of the per-row records (aloam_map_rows): localising lanes on the oracle world of tests/reloc_cases.py, one
armed at a scan's true map pose, one armed with a gross error, one armed off the map, and the prior-map inlier score of every frame.

The oracle side runs pyfrozen.Localiser (the frozen-map frame) on the oracle's own odometry from the START scan, and scores every
frame's map pose with reloc_cases.FrozenScorer -- the score aloam_map_rows gives a localising row.  tests/test_oracle_track_score.py
fixes the thresholds below on the oracle alone; tests/test_gpu_map_rows.py holds the device to them."""
import numpy as np

import pyoracle
import reloc_cases as RC

# scoring of the tracking rows: the relocalisation scenario's radius and points per type
ISQ, PTS = RC.INLIER_SQ, RC.MAX_PTS
# the lane that keeps track starts at this scan of the mapped stretch and runs to the end of the oracle world
START = 2
# a gross arming error that two outer x four inner iterations cannot pull in: the heading turned by 45 degrees and the position
# moved 3 m sideways
LOST_YAW, LOST_OFF = np.radians(45.0), (0.0, 3.0, 0.0)
# a frame whose score is below LOST_RATIO of its scoring points has lost track; a tracking frame scores above TRACK_RATIO (every
# point on the mapped stretch, above 0.8 on the six scans past it)
LOST_RATIO, TRACK_RATIO = 0.5, 0.75
# an arming off the map: every window cube is empty
OFF_MAP_T = (400.0, 0.0, 0.0)


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw, aw * bw - ax * bx - ay * by - az * bz])


def mis_armed(pose):
    """the pose turned by LOST_YAW about z and moved by LOST_OFF"""
    dq = np.array([0, 0, np.sin(LOST_YAW / 2), np.cos(LOST_YAW / 2)])
    out = np.array(pose, np.float64, copy=True)
    out[:4] = qmul(dq, out[:4])
    out[4:] = out[4:] + np.asarray(LOST_OFF)
    return out


def off_map(pose):
    out = np.array(pose, np.float64, copy=True)
    out[4:] = OFF_MAP_T
    return out


def odometry(feats, start, stop):
    """the oracle's odometry poses (q xyzw, t) of scans start .. stop-1 for a trajectory STARTed at `start` (identity there)"""
    od = pyoracle.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    out = []
    for k in range(start, stop):
        f = feats[k]
        if k > start:
            q, t, _ = od.register(f.sharp, f.flat, q, t)
            qw, tw = pyoracle.integrate_pose(qw, tw, q, t)
        od.set_last(f.less_sharp, f.less_flat)
        out.append(np.concatenate([qw, tw]))
    return np.array(out)


def track(frozen, scorer, feats, init, start, stop, res, isq=ISQ, pts=PTS):
    """a lane armed with `init` (7) and STARTed at scan `start`, run to `stop`: (map poses, infos, scores, scoring points per frame)"""
    import pyfrozen
    odo = odometry(feats, start, stop)
    loc = pyfrozen.Localiser(frozen, init[:4], init[4:])
    poses, infos, scores, n_score = [], [], [], []
    for j, k in enumerate(range(start, stop)):
        f = feats[k]
        pose, info = loc.step(f.less_sharp, f.less_flat, odo[j, :4], odo[j, 4:], *res)
        poses.append(pose)
        infos.append(info)
        scores.append(int(scorer.score(f.less_sharp, f.less_flat, pose[None], isq, pts, *res, normalise=False)[0]))
        sp = RC.scoring_points(f.less_sharp, f.less_flat, pts, *res)
        n_score.append(len(sp[0]) + len(sp[1]))
    return np.array(poses), infos, np.array(scores), np.array(n_score)
