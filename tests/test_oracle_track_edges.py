"""CPU: the scenes of the per-row records' edge-case tests (tests/track_edge_cases.py, used by tests/test_gpu_track_edges.py) have
the properties the GPU tests rely on: the staging cases reach every m, m_c residue and max_score_points they claim, the largest
stack is subsampled, the 16 lanes' stacks are ordered as claimed, every thin-map scene puts its chosen stack point on the query
and makes it an inlier (or not) exactly as claimed -- the oracle's score equal to the float32 brute force --, the row-table
schedules mix every kind, and the overflow scan's less-sharp box lies in the key-overflow window."""
import numpy as np
import pytest

import prior_build_cases as PB
import pyoracle
import reloc_cases as RC
import track_edge_cases as TE

EMPTY = np.zeros((0, 4), np.float32)


def test_staging_cases_reach_every_residue(synth):
    ms, res, specs = set(), set(), set()
    for sensor, n_az, index, spec in TE.STAGE_CASES:
        n_c, n_s = TE.stacks(synth, sensor, n_az, index, TE.DEFAULT_LEAVES)
        mp = TE.resolve_mp(spec, n_c, n_s)
        m_c, m = TE.staging(n_c, n_s, mp)
        ms.add(m)
        if m > m_c:   # surf points after the switch: in the same warp unless m_c is a multiple of 32
            res.add(m_c % 32)
        specs.add(spec if isinstance(spec, str) else ("1" if spec == 1 else "int"))
        if spec == "big":
            assert mp > max(n_c, n_s)
    assert set(TE.STAGE_M) <= ms, sorted(ms)
    assert set(TE.STAGE_MC_RES) <= res, res
    assert {"1", "nc-1", "nc", "nc+1", "big"} <= specs


def test_the_largest_stack_is_subsampled(synth):
    sensor, n_az, index, leaves, mp = TE.LARGE_CASE
    n_c, n_s = TE.stacks(synth, sensor, n_az, index, leaves)
    assert n_s >= TE.LARGE_MIN and mp < n_s
    # no synthetic scan reaches 46 341 points, where i * n of the subsample first needs 64 bits
    assert (mp - 1) * n_s < 2**31


def test_the_sixteen_lanes_order_their_stacks(synth):
    m = [sum(TE.stacks(synth, "VLP-16", n_az, k, TE.DEFAULT_LEAVES)) for n_az, k in TE.WIDE_LANES]
    assert len(set(m)) == 16 and m[0] == min(m) and m[15] == max(m), m
    assert len({(n, k) for n, k in TE.WIDE_LANES}) == 16 and max(k for _, k in TE.WIDE_LANES) < RC.N_MAP


_SCENES = TE.thin_scenes()


@pytest.mark.parametrize("t", [0, 1], ids=["corner", "surf"])
@pytest.mark.parametrize("k", range(len(_SCENES)), ids=[s[0] for s in _SCENES])
def test_thin_scenes_reach_their_edge(synth, k, t):
    name, s, isq, off, expect = _SCENES[k]
    leaves = (RC.WALK_LEAF, RC.WALK_LEAF)
    stk = TE.scan_stacks(synth)
    i = TE.pick(len(stk[0]), t, (7 * k + 31 * t) % 32, len(stk[t]))
    pos = i if t == 0 else len(stk[0]) + i
    assert pos % 32 == (7 * k + 31 * t) % 32
    p = stk[t][i]
    pose = TE.arming(s["query"][0], p, off)
    assert RC.normalised(pose)[0].tobytes() == pose.tobytes()
    moved = RC.transform(pose, p[None])[0]
    if not any(off):
        assert moved.tobytes() == s["query"][0, :3].tobytes()
    maps = (s["map"], TE.OTHER_MAP) if t == 0 else (TE.OTHER_MAP, s["map"])
    assert len(maps[1 - t]) <= 10   # the other type's window holds at most one point: the frame is thin
    assert RC.alone_in_voxels(s["map"], RC.WALK_LEAF)
    own = [EMPTY, EMPTY]
    own[t] = p[None]
    assert RC.brute_score(maps[0], maps[1], own, pose[None], isq)[0] == int(expect), name
    if name.startswith("walk") and expect:   # the inlier sits at its flat walk index
        assert s["counts"][:s["lane"][s["d2"] < np.float32(isq)][0]].sum() == s["flat"]
    if name == "isq-tiny-exact":
        assert (s["d2"] == 0).sum() == 1 and (s["d2"][s["d2"] > 0] >= 0.75).all()
    S = RC.FrozenScorer(PB.oracle_build(maps[0], maps[1], *leaves)[0].frozen())
    assert len(S.clouds[t]) == len(s["map"])
    pts = (stk[0], stk[1])
    ref = S.score_points(pts, pose[None], isq, normalise=False)
    assert ref.tolist() == RC.brute_score(maps[0], maps[1], pts, pose[None], isq).tolist()
    assert ref[0] >= int(expect)


def test_row_table_schedules_mix_every_kind():
    armed = {1: 2, 4: 0, 6: 5, 9: 1, 12: 3, 14: 6}
    for steps in (64, 256):
        ops, idx = TE.schedule(steps, 16, RC.N_MAP + 6, armed)
        assert ops[0, 0] == 0 and (ops[:2, list(armed)] == 2).any(axis=0).all()
        kinds = TE.expected_kinds(ops, armed, 2)
        assert set(np.unique(kinds)) == {0, 1, 2, 3}
        assert any(len(set(r)) == 4 for r in kinds)
        assert (kinds == 2).sum() >= 20
        assert ((ops == 2) | (ops == 1))[idx >= RC.N_MAP + 6].sum() == 0
    ops, idx = TE.schedule(14, 4, RC.N_MAP + 6, {2: 1}, seed=5)
    kinds = TE.expected_kinds(ops, {2: 1}, 2)
    assert (kinds == 2).sum() >= 3 and (kinds == 1).sum() >= 8


def test_the_overflow_scan_overflows_one_key(synth):
    raw, (i, j) = TE.overflow_scan(synth)
    base = TE.raw_scan(synth, "VLP-16", 900, 4)
    assert (np.flatnonzero((raw != base).any(1)) == sorted((i, j))).all()
    f = pyoracle.Features(raw, 16, synth.SENSORS["VLP-16"][2])
    line_res, plane_res = synth.SENSORS["VLP-16"][3:5]
    assert TE.seg_box(f.less_sharp, line_res) == (False, True)
    assert TE.seg_box(f.less_flat, plane_res) == (False, False)
    far = raw[[i, j], :3]
    assert (f.less_sharp[:, None, :3] == far[None]).all(-1).any(0).all()   # both moved returns are less-sharp points
    for k in (3, 5, 6):
        g = pyoracle.Features(TE.raw_scan(synth, "VLP-16", 900, k), 16, synth.SENSORS["VLP-16"][2])
        assert TE.seg_box(g.less_sharp, line_res) == (False, False) and TE.seg_box(g.less_flat, plane_res) == (False, False)
