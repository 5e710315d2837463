"""CPU: the frozen-map frame of the oracle (oracle/frozen.cc), the restatement behind localisation against a prior map: the
mapper's frame without the ring-buffer shift and without insertion / re-filter.  From the same store and T_wmap_wodom it returns the
ordinary oracle frame's pose bit for bit; it never writes the store; a vehicle that leaves the buffer gets a clipped, then empty
window and no optimisation instead of a shift; skipped scans get the high-frequency pose."""
import numpy as np
import pytest

import pyfrozen

N_BUILD = 5


@pytest.fixture(scope="module")
def world(orc, synth):
    """features and oracle odometry of a short VLP-16 trajectory, and the oracle store after mapping its first N_BUILD scans"""
    ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
    od = orc.Odometry()
    cm = orc.CubeMap()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    feats, odom = [], []
    for k in range(N_BUILD + 3):
        f = orc.Features(synth.scan("VLP-16", k, n_az=600), ns, mr)
        if k > 0:
            q, t, _ = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
        od.set_last(f.less_sharp, f.less_flat)
        feats.append((np.array(f.less_sharp), np.array(f.less_flat)))
        odom.append((qw.copy(), tw.copy()))
        if k < N_BUILD:
            cm.step(f.less_sharp, f.less_flat, qw, tw, line_res, plane_res)
    return {"cm": cm, "feats": feats, "odom": odom, "leaves": (line_res, plane_res)}


def _freeze(cm):
    st = cm.state()
    cubes = {}
    for index in range(pyfrozen.NCUBE):
        for which in (0, 1):
            c = cm.cube(which, index)
            if c.shape[0]:
                cubes[(which, index)] = c
    assert cubes
    return pyfrozen.FrozenMap.from_cubes(st["centre"], cubes), cubes, st


def test_first_frozen_frame_equals_the_ordinary_frame_and_the_store_stays_as_it_is(world):
    cm = world["cm"]
    frozen, cubes, st = _freeze(cm)
    loc = pyfrozen.Localiser(frozen, st["q_wmap_wodom"], st["t_wmap_wodom"], normalise=False)
    (c, s), (qo, to) = world["feats"][N_BUILD], world["odom"][N_BUILD]
    pose, info = loc.step(c, s, qo, to, *world["leaves"])
    ref, rinfo = cm.step(c, s, qo, to, *world["leaves"])   # the ordinary frame from the same store and T (it does not shift here)
    assert cm.state()["centre"] == st["centre"]
    assert info["optimised"] == rinfo["optimised"] == 1 and np.array_equal(pose, ref)
    assert loc.valid == cm.state()["valid"] and info["corner_from_map"] == rinfo["corner_from_map"] and info["surf_from_map"] == rinfo["surf_from_map"]
    assert np.array_equal(loc.q, cm.state()["q_wmap_wodom"]) and np.array_equal(loc.t, cm.state()["t_wmap_wodom"])
    # 20 more frozen frames: every cube of the prior map keeps its bytes, and no cube appears
    for k in range(20):
        (c, s), (qo, to) = world["feats"][N_BUILD + k % 3], world["odom"][N_BUILD + k % 3]
        loc.step(c, s, qo, to, *world["leaves"])
    for index in range(pyfrozen.NCUBE):
        for which in (0, 1):
            got = frozen.cube(which, index)
            assert got.tobytes() == (cubes[(which, index)].tobytes() if (which, index) in cubes else b""), (which, index)


def test_leaving_the_buffer_clips_then_empties_the_window_instead_of_shifting(world):
    frozen, cubes, st = _freeze(world["cm"])
    assert st["centre"] == (10, 10, 5)
    (c, s), (qo, _) = world["feats"][N_BUILD], world["odom"][N_BUILD]
    ident = np.array([0, 0, 0, 1.0])
    n_valid = []
    for x in (0.0, 400.0, 460.0, 520.0, 700.0):   # centre cube i = 10, 18, 19, 20, 24 of 0 .. 20
        loc = pyfrozen.Localiser(frozen, ident, np.array([x, 0, 0]))
        pose, info = loc.step(c, s, qo, np.zeros(3), *world["leaves"])
        n_valid.append(info["n_valid"])
        assert loc.valid == sorted(loc.valid, key=lambda v: (v % 21, (v // 21) % 21, v // 441))   # loop order: i, then j, then k
        if x > 0:   # outside the mapped cubes: too thin, the pose is the hand-off pose and T_wmap_wodom what it was
            assert info["optimised"] == 0 and info["corner_from_map"] == 0
            assert np.array_equal(pose[4:], [x, 0, 0]) and np.array_equal(loc.t, [x, 0, 0])
    assert n_valid == [75, 75, 60, 45, 0]


def test_skipped_scans_get_the_high_frequency_pose(world, orc):
    frozen, cubes, st = _freeze(world["cm"])
    loc = pyfrozen.Localiser(frozen, st["q_wmap_wodom"], st["t_wmap_wodom"], skip=3, normalise=False)
    poses = []
    for k in range(4):
        (c, s), (qo, to) = world["feats"][N_BUILD + k % 3], world["odom"][N_BUILD + k % 3]
        T = (loc.q.copy(), loc.t.copy())
        pose, info = loc.step(c, s, qo, to, *world["leaves"])
        poses.append(pose)
        if k % 3:
            assert info is None and np.array_equal(loc.q, T[0]) and np.array_equal(loc.t, T[1])   # nothing registered
            qw, tw = orc.integrate_pose(T[0], T[1], qo, to)   # q = q_wmap_wodom * q_wodom, t = q_wmap_wodom * t_wodom + t_wmap_wodom
            assert np.allclose(pose[:4], qw, atol=1e-15) and np.allclose(pose[4:], tw, atol=1e-12)
        else:
            assert info["optimised"] == 1
