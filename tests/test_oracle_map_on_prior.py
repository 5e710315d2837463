"""CPU: a mapping trajectory on a copy of a prior map (aloam_lane_map_on_prior) in the oracle and in the reference.  The oracle's
CubeMap seeded with a map's cubes, centre offsets and T_wmap_wodom equals, frame by frame and bit for bit, the reference's own
laserMapping.cpp whose globals were set the same way before its first frame (both seeded by tests/map_on_prior_seed.py): pose,
T_wmap_wodom, centre offsets and every cube of both arrays.  Cases: a second trajectory that starts inside a VLP-16 map and drives on, an init that shifts the ring buffer in the first frame until the seeded cubes wrap
out, centre offsets other than {10, 10, 5}, and an empty seed, which is the unseeded run."""
import numpy as np
import pytest

import lane_refs as R
from map_on_prior_seed import seed_cubemap, seed_ref

NCUBE = 21 * 21 * 11
N_MAP = 10


def _ref(orc, tag, leaves):
    from refsource import RefMapping, private_copy
    try:
        ref = RefMapping(private_copy("libref_mapping.so", "seed_" + tag), *leaves, orc.SORT_CANONICAL)
    except OSError as e:
        pytest.skip("oracle/_ref is not usable here: %r" % (e,))
    return ref


def _store(cm):
    """an oracle store as (centre, counts (2, NCUBE), points in ALOAM_EXPORT_MAP order)"""
    counts, pts = np.full((2, NCUBE), -1, np.int32), []
    for i in range(NCUBE):
        for ty in range(2):
            p = cm.cube(ty, i)
            if len(p):
                counts[ty, i] = len(p)
                pts.append(p)
    return cm.state()["centre"], counts, (np.concatenate(pts) if pts else np.zeros((0, 4), np.float32))


def _relabelled(store, dx):
    """the store with every cube moved dx cubes down in i and the centre offset with it: the same points over the same ground"""
    centre, counts, pts = store
    off = np.concatenate([[0], np.cumsum(np.maximum(counts.T.reshape(-1), 0))])   # export order: cube-major, corner then surf
    new, out = np.full((2, NCUBE), -1, np.int32), []
    for i in range(NCUBE):
        for ty in range(2):
            if i % 21 + dx <= 20 and counts[ty, i + dx] > 0:
                s = 2 * (i + dx) + ty
                new[ty, i] = counts[ty, i + dx]
                out.append(pts[off[s]:off[s + 1]])
    assert sum(len(p) for p in out) == len(pts)
    return (centre[0] - dx, centre[1], centre[2]), new, np.concatenate(out)


_MAPS = {}


def _session1(orc, synth):
    """the oracle's store after mapping scans 0 .. N_MAP-1 of trajectory 0, and its map poses"""
    if "vlp" not in _MAPS:
        scans = R.traj(synth, 0, N_MAP)
        odom, _ = R.oracle(orc, synth, scans, ("seed-s1",), False)
        ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
        cm, poses = orc.CubeMap(), []
        for k, raw in enumerate(scans):
            f = orc.Features(raw, ns, mr)
            poses.append(cm.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], line_res, plane_res)[0])
        _MAPS["vlp"] = (_store(cm), np.array(poses))
    return _MAPS["vlp"]


def _run_both(orc, synth, tag, store, q0, t0, s0, n, seeded=True):
    """scans s0 .. s0+n-1 of trajectory 0 as a new session (its own odometry from the identity) on the oracle and the reference,
    both seeded with `store` at T_wmap_wodom (q0, t0) (unseeded when seeded=False); every frame compared bit for bit"""
    ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
    scans = R.traj(synth, 0, s0 + n)[s0:]
    odom, _ = R.oracle(orc, synth, scans, ("seed-s2", s0, n), False)
    cm, ref = orc.CubeMap(), _ref(orc, tag, (line_res, plane_res))
    if seeded:
        seed_cubemap(cm, store[0], q0, t0, store[1], store[2])
        seed_ref(ref, store[0], q0, t0, store[1], store[2])
    poses, states = [], []
    for k, raw in enumerate(scans):
        f = orc.Features(raw, ns, mr)
        po, _ = cm.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], line_res, plane_res)
        r = ref.process(f.less_sharp, f.less_flat, f.less_flat, odom[k, :4], odom[k, 4:], stamp=0.1 * (k + 1))
        so = cm.state()
        assert np.array_equal(po, r["pose"]), (tag, k)
        assert so["centre"] == r["centre"], (tag, k)
        assert np.array_equal(so["q_wmap_wodom"], r["q_wmap_wodom"]) and np.array_equal(so["t_wmap_wodom"], r["t_wmap_wodom"]), (tag, k)
        for ty in range(2):
            sizes = ref.sizes(ty)
            assert int(sizes.sum()) == so["total_corner" if ty == 0 else "total_surf"], (tag, k, ty)
            for i in np.flatnonzero(sizes):
                assert np.array_equal(cm.cube(ty, int(i)), ref.cube(ty, int(i), int(sizes[i]))), (tag, k, ty, int(i))
        poses.append(po)
        states.append(so)
    return np.array(poses), states


def test_a_second_session_inside_the_map(orc, synth):
    store, poses = _session1(orc, synth)
    q0, t0 = poses[5][:4], poses[5][4:] + np.array([0.15, -0.1, 0.05])
    got, states = _run_both(orc, synth, "inside", store, q0, t0, 5, 12)
    assert states[-1]["total_surf"] > int(np.maximum(store[1][1], 0).sum())   # the session added points
    dt, dr = R.deviation(got[:N_MAP - 5], poses[5:])                           # and found session 1's poses again
    assert dt < 0.1 and dr < 0.02, (dt, dr)


def test_a_first_frame_shift_wraps_seeded_cubes_out(orc, synth):
    """a map position 400 m above the map: the first frame shifts the buffer down in k six times, and the map's plane of cubes
    wraps out"""
    store, _ = _session1(orc, synth)
    _, states = _run_both(orc, synth, "wrap", store, np.array([0, 0, 0, 1.0]), np.array([0, 0, 400.0]), 0, 3)
    assert states[0]["centre"][2] == store[0][2] - 6
    assert states[0]["total_corner"] + states[0]["total_surf"] < int(np.maximum(store[1], 0).sum())


def test_centre_offsets_other_than_the_default(orc, synth):
    """the map re-labelled 8 cubes down in i with centre (2, 10, 5): the vehicle starts in cube 2, so the first frame shifts up"""
    store, poses = _session1(orc, synth)
    moved = _relabelled(store, 8)
    assert moved[0] == (2, 10, 5)
    got, states = _run_both(orc, synth, "centre", moved, poses[3][:4], poses[3][4:], 3, 8)
    assert states[0]["centre"] == (3, 10, 5)
    dt, dr = R.deviation(got[:N_MAP - 3], poses[3:])
    assert dt < 0.1 and dr < 0.02, (dt, dr)


def test_an_empty_seed_is_the_unseeded_run(orc, synth):
    empty = ((10, 10, 5), np.full((2, NCUBE), -1, np.int32), np.zeros((0, 4), np.float32))
    a, _ = _run_both(orc, synth, "empty", empty, np.array([0, 0, 0, 1.0]), np.zeros(3), 0, 6)
    b, _ = _run_both(orc, synth, "unseeded", None, None, None, 0, 6, seeded=False)
    assert np.array_equal(a, b)
    _, poses = _session1(orc, synth)
    assert np.array_equal(a, poses[:6])
