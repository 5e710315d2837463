"""The host model of the recovery of localising lanes (aloam_set_recovery): the candidates around a row's map pose in the device's
operation order, the trigger and accept tests in float32, transformUpdate in Eigen's order, and the oracle's recovery loop -- the
frozen-map frames of pyfrozen.Localiser on the oracle odometry of tests/track_cases.py, every triggered frame's candidates scored by
reloc_cases.FrozenScorer and the localiser's T_wmap_wodom replaced on adoption.

tests/test_oracle_recovery.py fixes the scenario's constants below on the oracle alone; tests/test_gpu_recovery.py holds the device
to them and to this model bit for bit."""
import numpy as np

import reloc_cases as RC
import track_cases as TC

# a row triggers below half its scoring points (LOST_RATIO of the lost-track scenario) and adopts a candidate that holds
# TRACK_RATIO of them
TRIGGER, ACCEPT = TC.LOST_RATIO, TC.TRACK_RATIO
# the candidates: +-4 m at 1 m and 24 headings (15 degrees) about the sensor -- the scenario's 45 degree, 3 m arming error is on
# the lattice
HALF, STEP, N_YAW = 4.0, 1.0, 24
# the mis-armed lane adopts on its START row; its frames from FRAMES_TO_TRACK after the START on stay within 0.1 m / 0.02 rad of
# the truly armed lane
FRAMES_TO_TRACK = 1


def deltas(aloam, half=HALF, step=STEP, n_yaw=N_YAW):
    """the relative poses: pose_grid around the identity"""
    return aloam.pose_grid(np.array([0, 0, 0, 1.0]), np.zeros(3), half, step, np.arange(n_yaw) * (2 * np.pi / n_yaw))


def qmul(a, b):
    """cubemap.cu's qmul (Eigen's operator*), q = (x, y, z, w), term for term"""
    ax, ay, az, aw = (float(v) for v in a)
    bx, by, bz, bw = (float(v) for v in b)
    w = aw * bw - ax * bx - ay * by - az * bz
    x = aw * bx + ax * bw + ay * bz - az * by
    y = aw * by + ay * bw + az * bx - ax * bz
    z = aw * bz + az * bw + ax * by - ay * bx
    return np.array([x, y, z, w])


def qinv(a):
    x, y, z, w = (float(v) for v in a)
    n2 = x * x + y * y + z * z + w * w
    return np.array([-x / n2, -y / n2, -z / n2, w / n2])


def qrot(q, v):
    x, y, z, w = (float(c) for c in q)
    v = [float(c) for c in v]
    uv = [y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]]
    uv = [u + u for u in uv]
    c2 = [y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0]]
    return np.array([v[k] + w * uv[k] + c2[k] for k in range(3)])


def normalise(q):
    """aloam_lane_localise's normalisation: q / sqrt(q . q), the squares summed in index order"""
    n2 = 0.0
    for v in q:
        n2 += float(v) * float(v)
    n = np.sqrt(n2)
    return np.array([float(v) / n for v in q])


def products(P, D):
    """the candidates before normalisation: (q_d * q_P, t_P + t_d) for every delta row d of D"""
    out = np.empty((len(D), 7))
    for h, d in enumerate(np.asarray(D, np.float64)):
        out[h, :4] = qmul(d[:4], P[:4])
        out[h, 4:] = [float(P[4 + k]) + float(d[4 + k]) for k in range(3)]
    return out


def candidates(P, D):
    """the candidates the device scores: D normalised as aloam_set_recovery normalises it, then q_h = normalise(q_d * q_P)"""
    out = products(P, RC.normalised(D))
    for h in range(len(out)):
        out[h, :4] = normalise(out[h, :4])
    return out


def triggers(score, n_score, frac=TRIGGER):
    return int(n_score) > 0 and np.float32(score) < np.float32(frac) * np.float32(n_score)


def accepts(best_score, score, n_score, frac=ACCEPT):
    return int(best_score) > int(score) and np.float32(best_score) >= np.float32(frac) * np.float32(n_score)


def best_of(scores):
    """(score descending, h ascending)"""
    h = int(np.argmax(scores))
    return h, int(scores[h])


def transform_update(x, odom):
    """laserMapping.cpp:148-152: T_wmap_wodom = x * odom^-1, in cubemap.cu's order"""
    qn = qmul(x[:4], qinv(odom[:4]))
    r = qrot(qn, odom[4:])
    return np.concatenate([qn, [float(x[4 + k]) - r[k] for k in range(3)]])


def recover_track(frozen, scorer, feats, init, start, stop, res, D, trigger=TRIGGER, accept=ACCEPT, isq=TC.ISQ, pts=TC.PTS):
    """a lane armed with `init` and STARTed at scan `start`, run to `stop` with recovery: per frame (map pose, score, n_score,
    triggered, best, best_score, adopted)"""
    import pyfrozen
    odo = TC.odometry(feats, start, stop)
    loc = pyfrozen.Localiser(frozen, init[:4], init[4:])
    out = []
    for j, k in enumerate(range(start, stop)):
        f = feats[k]
        pose, _ = loc.step(f.less_sharp, f.less_flat, odo[j, :4], odo[j, 4:], *res)
        sp = RC.scoring_points(f.less_sharp, f.less_flat, pts, *res)
        n = len(sp[0]) + len(sp[1])
        s = int(scorer.score_points(sp, pose[None], isq, normalise=False)[0])
        row = {"pose": pose, "score": s, "n_score": n, "triggered": False, "best": -1, "best_score": -1, "adopted": False}
        if triggers(s, n, trigger):
            cand = candidates(pose, D)
            h, bs = best_of(scorer.score_points(sp, cand, isq, normalise=False))
            row.update(triggered=True, best=h, best_score=bs, adopted=accepts(bs, s, n, accept), cand=cand[h])
            if row["adopted"]:
                T = transform_update(cand[h], odo[j])
                loc.q, loc.t = T[:4], T[4:]
        out.append(row)
    return out
