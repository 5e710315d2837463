"""CPU: the oracle of loop verification (oracle/pyloop.py) on crafted inputs -- the keyframe-cloud subsample around n = m, the
window clipped at 0 and at q - 1 - exclude_recent, the gather at identity poses, the score against a plain brute force and the
constraint's round trip with the pose."""
import math

import numpy as np
import pytest

import pyloop as L

IDENT = np.array([0, 0, 0, 1.0, 0, 0, 0])


def _cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(n, 4)).astype(np.float32) * 5
    c[:, 3] = np.arange(n)
    return c


@pytest.mark.parametrize("n, m", [(5, 8), (8, 8), (9, 8), (1000, 7), (0, 4), (7, 1)])
def test_subsample_picks_floor_i_n_over_m(n, m):
    s = _cloud(n)
    got = L.subsample(s, m)
    k = min(n, m)
    assert got.shape == (k, 4)
    for i in range(k):
        assert np.array_equal(got[i], s[(i * n) // k])
    if n <= m:
        assert np.array_equal(got, s)


def test_window_clips_at_both_ends():
    assert L.window(30, 2, 5, 10) == (0, 7)              # clipped at 0
    assert L.window(30, 17, 5, 10) == (12, 19)           # clipped at q - 1 - e
    assert L.window(30, 19, 0, 10) == (19, 19)
    assert L.window(100, 40, 5, 10) == (35, 45)


def test_gather_at_identity_poses_is_a_concatenation():
    clouds = [(_cloud(3 + k, k), _cloud(5 + 2 * k, 10 + k)) for k in range(6)]
    poses = np.tile(IDENT, (6, 1))
    c, s = L.gather(clouds, poses, 1, 4)
    assert np.array_equal(c, np.concatenate([clouds[k][0] for k in range(1, 5)]))
    assert np.array_equal(s, np.concatenate([clouds[k][1] for k in range(1, 5)]))


def test_gather_moves_each_keyframe_by_its_own_pose():
    clouds = [(_cloud(4, 1), _cloud(6, 2)), (_cloud(4, 3), _cloud(6, 4))]
    poses = np.array([IDENT, [0, 0, math.sin(0.3), math.cos(0.3), 5.0, -2.0, 1.0]])
    c, _ = L.gather(clouds, poses, 0, 1)
    assert np.array_equal(c[:4], clouds[0][0])
    th = 0.6
    p = clouds[1][0][:, :3].astype(np.float64)
    want = np.column_stack([math.cos(th) * p[:, 0] - math.sin(th) * p[:, 1] + 5, math.sin(th) * p[:, 0] + math.cos(th) * p[:, 1] - 2, p[:, 2] + 1])
    assert np.abs(c[4:, :3] - want).max() < 1e-4
    assert np.array_equal(c[4:, 3], clouds[1][0][:, 3])


def test_score_equals_a_brute_force():
    rng = np.random.default_rng(3)
    sub = (rng.uniform(-10, 10, (3000, 4))).astype(np.float32)
    pts = (rng.uniform(-10, 10, (500, 4))).astype(np.float32)
    pts[:100, :3] = sub[:100, :3] + np.float32(0.3)   # inliers for 0.3^2 * 3 < 1
    for r2 in (0.25, 1.0):
        want = sum(1 for p in pts if min(float(np.float32(np.float32((p[0] - q[0]) * (p[0] - q[0]) + (p[1] - q[1]) * (p[1] - q[1])) + (p[2] - q[2]) * (p[2] - q[2])))
                                         for q in sub) < r2)
        assert L.inliers(pts, sub, r2) == want
    assert L.score(pts, pts[:0], IDENT, sub, sub[:0], 1.0) == L.inliers(pts, sub, 1.0)


def test_rel_round_trips_with_the_pose():
    rng = np.random.default_rng(7)
    for _ in range(20):
        pc = L.normalised(np.concatenate([rng.normal(size=4), rng.normal(size=3) * 10]))
        p = L.normalised(np.concatenate([rng.normal(size=4), rng.normal(size=3) * 10]))
        r = L.rel(pc, p)
        back = np.concatenate([L.qmul(pc[:4], r[:4]), L.qrot(pc[:4], r[4:]) + pc[4:]])
        assert np.abs(back - p).max() < 1e-12
    assert np.array_equal(L.rel(IDENT, IDENT), IDENT)


def test_init_pose_turns_by_the_shift():
    pc = np.array([0, 0, 0, 1.0, 1, 2, 3])
    for s in (0, 1, 15, 30, 59):
        x = L.init_pose(pc, s)
        yaw = 2 * math.atan2(x[2], x[3])
        assert abs((yaw - s * 2 * math.pi / 60 + math.pi) % (2 * math.pi) - math.pi) < 1e-12
        assert np.array_equal(x[4:], pc[4:])
