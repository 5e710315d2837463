"""GPU parity on sweeps cut anywhere (tests/seam_cases.py): feature extraction against the oracle on the seam grid, the
scan-to-scan association on "last" clouds whose int(intensity) descends by one (relTime < 0 returns), and whole chains.
The association's break tables (odometry.cu) must reproduce the reference's loops (laserOdometry.cpp:310-361,400-455)
exactly where the clouds are not ascending in int(intensity)."""
import math

import numpy as np
import pytest

import edge_scenes as es
import lane_refs as R
import seam_cases as S
import test_gpu_lm_edges as LE
from conftest import rot_angle

pytestmark = pytest.mark.gpu

SENSORS = ["VLP-16", "HDL-32", "HDL-64"]


@pytest.fixture(scope="module")
def ctxs(aloam, synth):
    out = {s: aloam.Aloam(n_scans=synth.SENSORS[s][0], max_points=200000) for s in SENSORS}
    yield out
    for c in out.values():
        c.close()


def check_features(got, ref, ctx, tag):
    """the bars of tests/test_gpu_features.py"""
    assert got["full"].shape == ref.full.shape, tag
    assert np.array_equal(got["full"][:, :3], ref.full[:, :3]), tag
    assert np.array_equal(got["full"][:, 3].astype(np.int32), ref.full[:, 3].astype(np.int32)), tag
    assert np.all(np.abs(got["full"][:, 3] - ref.full[:, 3]) <= 1e-6 + np.spacing(np.abs(ref.full[:, 3]))), tag
    curv, label, s, e = ctx.debug_features(ref.full.shape[0])
    ns = len(ref.scan_start)
    assert np.array_equal(s[:ns], ref.scan_start) and np.array_equal(e[:ns], ref.scan_end), tag
    for r in range(ns):
        a, b = ref.scan_start[r], ref.scan_end[r]
        if b - a < 6:
            continue
        assert np.array_equal(curv[a:b + 1], ref.curvature[a:b + 1]), (tag, r)
        assert np.array_equal(label[a:b], ref.label[a:b]), (tag, r)
    for name in ["sharp", "less_sharp", "flat", "less_flat"]:
        g, r_ = got[name], getattr(ref, name)
        assert g.shape == r_.shape, (tag, name)
        assert np.array_equal(g[:, :3], r_[:, :3]), (tag, name)
        assert np.array_equal(g[:, 3].astype(np.int32), r_[:, 3].astype(np.int32)), (tag, name)
        assert np.all(np.abs(g[:, 3] - r_[:, 3]) <= 1e-5), (tag, name)


@pytest.mark.parametrize("sensor", SENSORS)
@pytest.mark.parametrize("cut", S.CUTS, ids=["q1", "q2", "q3", "q4", "zero", "pi_2", "minus_pi_2", "pi"])
def test_features_on_the_seam_grid(ctxs, orc, synth, sensor, cut):
    ns, _, mr = synth.SENSORS[sensor][:3]
    for k, (cov, off, lm, ccw) in enumerate(S.layouts(ns)):
        raw = S.seam_scan(synth, sensor, k % 4, cut, cov, off, lm, ccw)
        ref = orc.Features(raw, ns, mr, orc.SORT_CANONICAL)
        check_features(ctxs[sensor].extract_features(raw), ref, ctxs[sensor], (sensor, cut, cov, off is not None, lm, ccw))


@pytest.mark.parametrize("name", S.HAND_BUILT)
def test_features_of_hand_built_first_returns(ctxs, orc, synth, name):
    _, sensor, raw = next(c for c in S.hand_built(synth) if c[0] == name)
    ns, _, mr = synth.SENSORS[sensor][:3]
    check_features(ctxs[sensor].extract_features(raw), orc.Features(raw, ns, mr, orc.SORT_CANONICAL), ctxs[sensor], name)


def _assoc_pair(orc, synth, sensor, distortion):
    ns, _, mr = synth.SENSORS[sensor][:3]
    f0 = orc.Features(S.trajectory_scan(synth, sensor, 0), ns, mr)
    f1 = orc.Features(S.trajectory_scan(synth, sensor, 1), ns, mr)
    assert S.descents(f0.less_sharp) + S.descents(f0.less_flat) > 0   # the last clouds are not ascending in int(intensity)
    return f0, f1


@pytest.mark.parametrize("sensor", ["HDL-64", "VLP-16"])
@pytest.mark.parametrize("distortion", [0, 1])
@pytest.mark.parametrize("moved", [False, True])
def test_association_on_seam_clouds(aloam, orc, synth, sensor, distortion, moved):
    """aloam_odometry_set_last accepts the clouds the extraction produced, and the association equals the oracle's literal
    loops query by query: (closest, 2nd, 3rd, valid)"""
    f0, f1 = _assoc_pair(orc, synth, sensor, distortion)
    ctx = aloam.Aloam(n_scans=synth.SENSORS[sensor][0], max_points=200000, distortion=distortion)
    try:
        q = np.array([0.001, -0.002, 0.008, 0.99996] if moved else [0, 0, 0, 1.0]); q /= np.linalg.norm(q)
        t = np.array([0.7, 0.02, -0.01] if moved else [0, 0, 0.0])
        od = orc.Odometry(distortion=bool(distortion))
        od.set_last(f0.less_sharp, f0.less_flat)
        cc, pc, _ = od.associate(f1.sharp, f1.flat, q, t)
        ctx.odometry_set_last(f0.less_sharp, f0.less_flat)
        gcc, gpc = ctx.odometry_associate(f1.sharp, f1.flat, q, t)
        got_c = [(i, a, b) for i, (a, b, v) in enumerate(gcc) if v]
        got_p = [(i, a, b, c) for i, (a, b, c, v) in enumerate(gpc) if v]
        want_c = [tuple(int(v) for v in r) for r in cc]
        want_p = [tuple(int(v) for v in r) for r in pc]
        for got, want, kind in ((got_c, want_c, "corner"), (got_p, want_p, "surf")):
            if got != want:
                diff = [(g, w) for g, w in zip(got, want) if g != w][:5]
                pytest.fail("%s: %d of %d %s correspondences differ, first (got, expected): %s" % (sensor, len(diff), len(want), kind, diff))
        assert len(got_c) > 100 and len(got_p) > 200
    finally:
        ctx.close()


def _tie_cloud():
    """a hand-built last cloud: rings 3..7, int(intensity) dipping by one after every ring change, exact copies of points
    at forward and backward positions with int = rc +- 1 and entries right after each break index"""
    pts = []
    for ring in range(3, 8):
        for j in range(12):
            ang = 0.05 * j
            r = 10.0 + ring
            x, y, z = r * math.cos(ang), r * math.sin(ang), -1.0 + 0.2 * ring
            intensity = ring - 0.02 if j >= 9 and ring > 3 else ring + 0.01 * j   # last returns of a ring: relTime < 0
            pts.append([x, y, z, intensity])
    c = np.array(pts, np.float32)
    # exact copies: a ring-4 point repeated where int = 5 (forward, before the ring-6 block) and where int = 3 (backward)
    c[14, :3] = c[30, :3]
    c[26, :3] = c[30, :3]
    c[40, :3] = c[5, :3]
    # past the break indices: index 45 (int 5) follows the first int >= 6 (index 36), so for a query whose closest point
    # is index 0 (rc = 3) the forward loops stop before it; index 28 (int 5) precedes the last int <= 4 (index 35), so for
    # a query whose closest point is index 50 (rc = 7) the backward loops stop before it.  Both sit 1 cm from the query,
    # nearer than any candidate inside the window: an association that ignored the breaks would pick them.
    c[45, :3] = c[0, :3] + np.float32([0.0, 0.0, 0.01])
    c[28, :3] = c[50, :3] + np.float32([0.0, 0.0, 0.01])
    return c


PLANTED = ((0, 45), (50, 28))   # (query index = closest point, post-break entry beside it)


def test_association_ties_and_break_indices(aloam, orc):
    """exact-copy ties at forward and backward positions with int = rc +- 1 and entries right after break indices, on a
    cloud that descends by one at every ring change: the device equals the literal loops"""
    last = _tie_cloud()
    r = last[:, 3].astype(np.int32)
    assert np.any(np.diff(r) < 0) and np.all(r >= np.maximum.accumulate(r) - 1)
    rng = np.random.default_rng(4)
    queries = np.concatenate([last + np.float32([0, 0, 0, 0]), last + rng.normal(0, 0.05, last.shape).astype(np.float32) * [1, 1, 1, 0]])
    queries = np.ascontiguousarray(queries, np.float32)
    ctx = aloam.Aloam(n_scans=16, max_points=10000)
    try:
        for q, t in (([0, 0, 0, 1.0], [0, 0, 0.0]), ([0, 0, 0.01, 0.99995], [0.05, 0.0, 0.0])):
            q = np.array(q); q /= np.linalg.norm(q); t = np.array(t)
            od = orc.Odometry()
            od.set_last(last, last)
            cc, pc, _ = od.associate(queries, queries, q, t)
            ctx.odometry_set_last(last, last)
            gcc, gpc = ctx.odometry_associate(queries, queries, q, t)
            assert [(i, a, b) for i, (a, b, v) in enumerate(gcc) if v] == [tuple(int(v) for v in x) for x in cc]
            assert [(i, a, b, c) for i, (a, b, c, v) in enumerate(gpc) if v] == [tuple(int(v) for v in x) for x in pc]
            assert len(cc) > 20 and len(pc) > 20
            if not np.any(t):
                # the planted entries are the nearest other points of their queries, and the literal loops do not pick them
                for qi, planted in PLANTED:
                    d = np.sum((last[:, :3] - queries[qi, :3]) ** 2, axis=1)
                    d[qi] = np.inf
                    assert np.argmin(d) == planted
                    row_c = [x for x in cc if x[0] == qi]
                    row_p = [x for x in pc if x[0] == qi]
                    assert row_c and row_c[0][1] == qi and row_c[0][2] != planted, row_c
                    assert row_p and row_p[0][1] == qi and planted not in tuple(row_p[0][2:]), row_p
    finally:
        ctx.close()


def _unsupported(cloud):
    """clouds no scanRegistration output can be: int(intensity) two below its predecessor; a run of single steps down
    (5, 4, 3) that ends two below the running maximum; an int(intensity) of -1 and of 64"""
    i = len(cloud) // 2
    r0 = int(cloud[i - 1, 3])
    assert r0 >= 3
    out = []
    c = cloud.copy(); c[i, 3] = r0 - 2 + 0.05; out.append(("two_below_predecessor", c))
    c = cloud.copy(); c[i:i + 2, 3] = [r0 - 1 + 0.05, r0 - 2 + 0.05]; out.append(("run_of_single_steps", c))
    c = cloud.copy(); c[0, 3] = -1.5; out.append(("ring_minus_one", c))
    c = cloud.copy(); c[-1, 3] = 64.02; out.append(("ring_64", c))
    for name, c in out[:2]:
        r = c[:, 3].astype(np.int32)
        assert np.all(r[1:] >= r[:-1] - 1) == (name == "run_of_single_steps")   # only the running maximum catches this one
        assert not np.all(r >= np.maximum.accumulate(r) - 1)
    return out


def test_unsupported_cloud_is_refused_and_leaves_no_trace(aloam, orc, synth):
    """clouds outside the invariant int_i >= max_{j<i} int_j - 1, or with an int(intensity) outside 0..63, are refused with
    -8 (as corner or surf cloud); the next calls of the context equal a fresh context's"""
    f0, f1 = _assoc_pair(orc, synth, "VLP-16", 0)
    used = aloam.Aloam(n_scans=16, max_points=60000)
    fresh = aloam.Aloam(n_scans=16, max_points=60000)
    try:
        for name, bad in _unsupported(f0.less_flat):
            with pytest.raises(aloam.AloamError) as e:
                used.odometry_set_last(f0.less_sharp, bad)
            assert e.value.code == -8, name
        for name, bad in _unsupported(f0.less_sharp):
            with pytest.raises(aloam.AloamError) as e:
                used.odometry_set_last(bad, f0.less_flat)
            assert e.value.code == -8, name
        q = np.array([0, 0, 0.004, 1.0]); q /= np.linalg.norm(q); t = np.array([0.5, 0, 0.0])
        for c in (used, fresh):
            c.odometry_set_last(f0.less_sharp, f0.less_flat)
        a, b = used.odometry_associate(f1.sharp, f1.flat, q, t), fresh.odometry_associate(f1.sharp, f1.flat, q, t)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    finally:
        used.close(); fresh.close()


@pytest.mark.parametrize("name,distortion", [("HDL-64", 0), ("HDL-64", 1), ("VLP-16", 0), ("VLP-16", 1), ("VLP-16-ccw", 1)])
def test_scan_to_pose_and_stream_on_seam_trajectories(aloam, orc, synth, name, distortion):
    """scan_to_pose along a seam trajectory: correspondence counts equal the oracle chain's, poses within 1e-4; the scan
    stream gives the per-scan poses bit for bit.  With DISTORTION the HDL-64 chain carries queries with s up to ~9.998 and
    the counter-clockwise VLP-16 chain queries with s < 0 (asserted), so the LM's slerp path runs at those ratios."""
    sensor = S.TRAJECTORIES[name]["sensor"]
    ns, _, mr = synth.SENSORS[sensor][:3]
    raws = [S.trajectory_scan(synth, name, k) for k in range(5)]
    s_lo, s_hi = 0.0, 1.0
    ctx = aloam.Aloam(n_scans=ns, max_points=200000, distortion=distortion)
    od = orc.Odometry(distortion=bool(distortion))
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    per_scan, worst = [], 0.0
    try:
        for k, raw in enumerate(raws):
            f = orc.Features(raw, ns, mr)
            if k > 0:
                q, t, info = od.register(f.sharp, f.flat, q, t)
                qw, tw = orc.integrate_pose(qw, tw, q, t)
                s = S.ratios(np.concatenate([f.sharp, f.flat]))
                s_lo, s_hi = min(s_lo, float(s.min())), max(s_hi, float(s.max()))
            od.set_last(f.less_sharp, f.less_flat)
            gq, gt, st = ctx.scan_to_pose(raw)
            per_scan.append(np.concatenate([gq, gt]))
            worst = max(worst, float(np.abs(gt - tw).max()), rot_angle(gq, qw))
            if k > 0:
                assert (st["n_corner_corr"], st["n_plane_corr"]) == (info["corner_corr"], info["plane_corr"]), (k, st, info)
        assert worst < 1e-4, worst
        assert float(np.abs(tw).max()) > 0.05   # the chain moves (with DISTORTION the ccw sweep registers only ~0.3 m, on both sides)
        if name == "HDL-64":
            assert s_hi > 9.99, s_hi
        if name == "VLP-16-ccw":
            assert s_lo < -0.01, s_lo
        ctx.reset_odometry()
        keep = [np.ascontiguousarray(r) for r in raws]
        poses, _ = ctx.scan_stream([r.ctypes.data for r in keep], [len(r) for r in keep], False)
        assert np.array_equal(poses, np.array(per_scan)), np.abs(poses - np.array(per_scan)).max()
    finally:
        ctx.close()
    print("%s distortion=%d: query ratios s in [%.4f, %.4f], worst pose deviation from the oracle chain %.2e" % (name, distortion, s_lo, s_hi, worst))


def _lane_layout(b):
    """16 different seams: every cut of the grid, both directions, laser- and column-major, offsets on half the lanes"""
    return S.CUTS[b % 8], (b // 8) % 2 == 1, b % 3 == 0, b % 2 == 0


def test_batch_lanes_with_different_seams(aloam, orc, synth):
    """16 lanes, each a trajectory with its own seam, through the batched feature kernel (k_ring_features_batch) and the
    batched odometry: every lane equals its solo scan_stream bit for bit and the oracle chain within 1e-4"""
    ns, n_scans, lanes = 16, 3, 16
    off = S.ring_offsets(ns)
    raws = []
    for k in range(n_scans):
        row = []
        for b in range(lanes):
            cut, ccw, lm, with_off = _lane_layout(b)
            row.append(np.ascontiguousarray(synth.scan_seam("VLP-16", k, cut, 1.0, off if with_off else None, lm, ccw, n_az=901)))
        raws.append(row)
    ctx = aloam.Aloam(n_scans=ns, max_points=40000, max_batch=lanes)
    worst = 0.0
    try:
        ptrs = np.array([[r.ctypes.data for r in row] for row in raws], np.uint64)
        cnts = np.array([[len(r) for r in row] for row in raws], np.int32)
        got = ctx.scan_stream_batch(ptrs, cnts, False)
        for b in range(lanes):
            solo = aloam.Aloam(n_scans=ns, max_points=40000)
            try:
                want, _ = solo.scan_stream([raws[k][b].ctypes.data for k in range(n_scans)], [len(raws[k][b]) for k in range(n_scans)], False)
            finally:
                solo.close()
            assert np.array_equal(got[:, b], want), b
            ref, _ = R.oracle(orc, synth, [raws[k][b] for k in range(n_scans)], ("seam-lane", b), False)
            worst = max(worst, *R.assert_near(got[:, b], ref, "lane %d" % b))
    finally:
        ctx.close()
    print("16 seam lanes: worst pose deviation from the oracle chain %.2e" % worst)


def test_scan_stream_mapped_on_a_seam_trajectory(aloam, orc, synth):
    """scan_stream_mapped along the VLP-16 seam trajectory: the odometry rows equal scan_stream's bit for bit, and odometry
    and map poses are within 1e-4 of the oracle chain (scanRegistration | laserOdometry | laserMapping)"""
    raws = [np.ascontiguousarray(S.trajectory_scan(synth, "VLP-16", k)) for k in range(6)]
    mapped = R.solo(aloam, raws, "seam-VLP-16", True)
    plain = R.solo(aloam, raws, "seam-VLP-16", False)
    assert np.array_equal(mapped["odom"], plain["odom"])
    o, m = R.oracle(orc, synth, raws, "seam-VLP-16", True)
    R.assert_near(mapped["odom"], o, "odometry")
    dt, dr = R.assert_near(mapped["map"], m, "map")
    print("seam mapped stream: map poses within %.2e m / %.2e rad of the oracle chain" % (dt, dr))


def test_transform_to_end_on_seam_less_flat(aloam, orc, synth):
    """TransformToEnd on a counter-clockwise seam's less_flat, which holds ring-0 returns with negative intensity: the
    integer part is int() truncation (0 there, not floor's -1) on both sides, and the coordinates agree"""
    ctx = aloam.Aloam(n_scans=16, max_points=60000, distortion=1)
    try:
        f = ctx.extract_features(S.trajectory_scan(synth, "VLP-16-ccw", 2))
        lf = f["less_flat"]
        neg = lf[:, 3] < 0
        assert np.any(neg)
        q = np.array([0.004, -0.003, 0.02, 1.0]); q /= np.linalg.norm(q)
        t = np.array([0.8, -0.02, 0.01])
        for dist in (True, False):
            got = ctx.transform_to_end(lf, q, t, dist)
            ref = orc.transform_to_end(lf, q, t, dist)
            assert got.shape == ref.shape
            assert np.array_equal(got[:, 3], ref[:, 3])
            assert np.array_equal(got[:, 3], lf[:, 3].astype(np.int32).astype(np.float32))
            assert np.all(got[neg, 3] == 0.0)
            assert np.abs(got[:, :3] - ref[:, :3]).max() < 2e-6      # acos / sin differ in the last bits between libm and CUDA
    finally:
        ctx.close()


SEAM_S = (-0.05, -1e-7, 1.5, 9.998)
SEAM_X0 = dict(LE.X0_Q, near_identity=np.concatenate([es.quat([0.3, 1.0, -0.2], 1e-4), [0.01, -0.02, 0.0]]))


@pytest.fixture(scope="module")
def lm_ctx(aloam):
    c = aloam.Aloam(n_scans=64, max_points=20000)
    yield c
    c.close()


@pytest.mark.parametrize("q0", list(SEAM_X0))
def test_normal_equations_and_solve_at_seam_ratios(lm_ctx, orc, q0):
    """edge and plane blocks with the interpolation ratios a seam sweep gives the DISTORTION build (s < 0 on ring 0, s near
    10 where int(intensity) = ring - 1): normal equations and the trust-region solve against the oracle's Jet autodiff, at
    the bars of tests/test_gpu_lm_edges.py, at q = identity, near identity, with w < 0 and generic"""
    blocks = es.blocks(orc, np.random.default_rng(17), LE.X_TRUE, 600, noise=0.05, kinds=(0, 1), s_values=SEAM_S)
    assert set(SEAM_S) <= set(blocks[blocks[:, 0] != orc.PLANE_NORM, 10])
    x0 = SEAM_X0[q0]
    LE._compare_normal_equations(lm_ctx, orc, blocks, x0)
    LE._compare_solve(lm_ctx, orc, blocks, x0)
