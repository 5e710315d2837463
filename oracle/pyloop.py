"""The oracle of loop verification (aloam_set_loops, aloam_loop_verify): the keyframe-cloud subsample, the window and the submap
gather, the initial heading, the inlier score by brute force and the constraint in Eigen's operation order.  The registration
itself is the oracle's map registration (pyoracle.Mapping: set_map + register).  ORACLE = test infrastructure, like pyplace."""
import math

import numpy as np

import pyclouds

SECTORS = 60


def subsample(stack, cloud_points):
    """stored point i of a keyframe's stack of n points: stack point floor(i n / m), m = min(n, cloud_points) (64-bit integers)"""
    s = np.ascontiguousarray(stack, np.float32).reshape(-1, 4)
    n = s.shape[0]
    m = min(n, int(cloud_points))
    return s[(np.arange(m, dtype=np.int64) * n) // max(m, 1)].copy() if m else s[:0].copy()


def window(query, cand, half, exclude):
    """the keyframes [lo, hi] of the candidate's submap: max(0, c - half) .. min(c + half, q - 1 - exclude)"""
    return max(0, cand - half), min(cand + half, query - 1 - exclude)


def gather(clouds, poses, lo, hi):
    """the submap of keyframes lo .. hi: per type the concatenation of their stored clouds (clouds[k] = (corner, surf)), each point
    moved by pointAssociateToMap at keyframe k's pose (poses[k], q xyzw, t) -> (corner, surf) float32"""
    out = [[], []]
    for k in range(lo, hi + 1):
        for t in range(2):
            out[t].append(pyclouds.associate_to_map(poses[k], clouds[k][t]))
    return tuple(np.concatenate(o) if o else np.zeros((0, 4), np.float32) for o in out)


def qmul(a, b):
    """Eigen's quaternion product a * b, (x, y, z, w), term for term"""
    ax, ay, az, aw = (float(v) for v in a)
    bx, by, bz, bw = (float(v) for v in b)
    return np.array([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz])


def qrot(q, v):
    """Eigen's q * v: uv = 2 (q.vec x v), v + w uv + q.vec x uv"""
    x, y, z, w = (float(c) for c in q)
    v = [float(c) for c in v]
    uv = [y * v[2] - z * v[1], z * v[0] - x * v[2], x * v[1] - y * v[0]]
    uv = [u + u for u in uv]
    c2 = [y * uv[2] - z * uv[1], z * uv[0] - x * uv[2], x * uv[1] - y * uv[0]]
    return np.array([v[k] + w * uv[k] + c2[k] for k in range(3)])


def normalised(x):
    """q / |q| with |q|^2 summed in index order (aloam_lane_localise), t unchanged"""
    x = np.array(x, np.float64)
    n2 = 0.0
    for k in range(4):
        n2 += float(x[k]) * float(x[k])
    n = math.sqrt(n2)
    x[:4] = [float(x[k]) / n for k in range(4)]
    return x


def init_pose(pose_c, shift):
    """q_c * Rz(shift * 2 pi / 60) written as place_hypotheses writes it, normalised; t_c"""
    a = float(shift) * 2.0 * math.pi / SECTORS
    sz, cz = math.sin(a / 2), math.cos(a / 2)
    x, y, z, w = (float(v) for v in pose_c[:4])
    out = np.zeros(7)
    out[:4] = [x * cz + y * sz, y * cz - x * sz, z * cz + w * sz, w * cz - z * sz]
    out[4:] = pose_c[4:]
    return normalised(out)


def rel(pose_c, pose):
    """T_c^-1 * pose in Eigen's order: (q_c.conjugate() * q, q_c.conjugate() * (t - t_c))"""
    cc = np.array([-pose_c[0], -pose_c[1], -pose_c[2], pose_c[3]], np.float64)
    out = np.zeros(7)
    out[:4] = qmul(cc, pose[:4])
    out[4:] = qrot(cc, [float(pose[4 + k]) - float(pose_c[4 + k]) for k in range(3)])
    return out


def inliers(points, sub, inlier_sq, chunk=256):
    """how many of the (already moved) points have a point of sub at float ((dx*dx + dy*dy) + dz*dz) < inlier_sq (brute force)"""
    p = np.ascontiguousarray(points, np.float32)[:, :3]
    s = np.ascontiguousarray(sub, np.float32)[:, :3]
    if p.shape[0] == 0 or s.shape[0] == 0:
        return 0
    lim = np.float32(inlier_sq)
    n = 0
    for i in range(0, p.shape[0], chunk):
        d = p[i:i + chunk, None, :] - s[None, :, :]
        d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        n += int(np.count_nonzero((d2 < lim).any(axis=1)))
    return n


def score(corner, surf, pose, sub_corner, sub_surf, inlier_sq):
    """the loop row's score: the query keyframe's stored points moved by pose, inliers per type against the submap"""
    return (inliers(pyclouds.associate_to_map(pose, corner), sub_corner, inlier_sq) +
            inliers(pyclouds.associate_to_map(pose, surf), sub_surf, inlier_sq))
