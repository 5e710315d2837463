"""GPU: rings from the sensor driver (cfg.ring_source = ALOAM_RING_FIELD).  With float 3 set to the elevation formula's ring the
field mode gives exactly what the elevation mode gives; on other beam tables (tests: synth.RING_SENSORS) the device follows the
oracle's field mode (tests/ring_field_oracle.py) bit for bit in the features, and the oracle chain in odometry and mapping."""
import numpy as np
import pytest

import ring_field_oracle as RF
from conftest import rot_angle

pytestmark = pytest.mark.gpu

NAMES = ("full", "sharp", "less_sharp", "flat", "less_flat")
ERR_INVALID_ARG, ERR_UNSUPPORTED_SCANS, ERR_RING_TOO_LARGE, ERR_SNAPSHOT = -1, -2, -7, -11
IDLE, SCAN, START = 0, 1, 2


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _field(aloam, ns, max_points, **kw):
    mr, lr, pr = 0.3, 0.2, 0.4   # synth.RING_RANGES
    return aloam.Aloam(n_scans=ns, max_points=max_points, ring_source=aloam.RING_FIELD, minimum_range=mr, line_res=lr, plane_res=pr, **kw)


def _ns(synth, sensor):
    return len(synth.RING_SENSORS[sensor][0])


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, e.value.code


# ------------------------------------------------------------------------------------------------ 1. equivalence with elevation mode
def test_formula_ring_in_field_mode_equals_elevation_mode(aloam, synth):
    """every elevation case: extract_features and debug_features of the field mode with w = the formula's ring are the elevation
    mode's, bit for bit"""
    ctx = {}
    for tag, raw, ns, mr in RF.elevation_cases(synth):
        if ns not in ctx:
            ctx[ns] = tuple(aloam.Aloam(n_scans=ns, max_points=200000, minimum_range=mr, ring_source=rs) for rs in (aloam.RING_ELEVATION, aloam.RING_FIELD))
        e, f = ctx[ns]
        want = e.extract_features(raw)
        dwant = e.debug_features(len(want["full"]))
        got = f.extract_features(RF.formula_rings(raw, ns))
        dgot = f.debug_features(len(got["full"]))
        for n in NAMES:
            assert np.array_equal(_bits(got[n]), _bits(want[n])), (tag, n)
        for a, b in zip(dgot, dwant):
            assert np.array_equal(a, b), tag
    for pair in ctx.values():
        for c in pair:
            c.close()


def test_formula_ring_in_field_mode_equals_the_reference_source(aloam, orc, synth):
    """the same field-mode outputs against the reference's own scanRegistration.cpp (oracle/_ref, where it is built)"""
    import refsource
    for tag, raw, ns, mr in RF.elevation_cases(synth):
        if not tag.endswith(("/0", "/seam")):
            continue
        ref = refsource.ref_registration(ns, mr).run(raw, orc.SORT_CANONICAL)
        f = aloam.Aloam(n_scans=ns, max_points=200000, minimum_range=mr, ring_source=aloam.RING_FIELD)
        got = f.extract_features(RF.formula_rings(raw, ns))
        f.close()
        for n in NAMES:   # the bars of test_gpu_vs_reference_source.py
            g, r = got[n], ref[n]
            assert g.shape == r.shape and np.array_equal(g[:, :3], r[:, :3]), (tag, n)
            assert np.array_equal(g[:, 3].astype(np.int32), r[:, 3].astype(np.int32)) and np.abs(g[:, 3] - r[:, 3]).max() <= 1e-5, (tag, n)


# ------------------------------------------------------------------------------------------------ 2. features against the oracle
def _mix_invalid(raw, ns, seed):
    """one return in 40 gets a ring that drops it: NaN, +-inf, -1, n_scans, 2.5 or 1e9; one in 40 others gets -0.0 (ring 0)"""
    out = raw.copy()
    rng = np.random.default_rng(seed)
    pick = rng.permutation(len(out))[: len(out) // 20]
    bad, zero = pick[::2], pick[1::2]
    vals = np.array([np.nan, np.inf, -np.inf, -1.0, ns, 2.5, 1e9], np.float32)
    out[bad, 3] = vals[np.arange(len(bad)) % len(vals)]
    out[zero, 3] = np.float32(-0.0)
    return out


FEATURE_CASES = [  # sensor, reverse, laser_major, stride, invalid
    ("OS64", False, False, 4, False), ("OS64", True, True, 8, True), ("V32C", False, False, 8, False), ("V32C", True, False, 4, True),
    ("V32C", False, True, 4, False), ("L40", False, False, 4, True), ("L40", True, True, 8, False), ("R1", False, False, 4, False),
    ("R1", False, True, 8, True), ("R2", True, False, 4, False), ("R2", False, True, 8, True),
]


@pytest.mark.parametrize("sensor,reverse,laser_major,stride,invalid", FEATURE_CASES)
def test_features_equal_the_field_oracle(aloam, synth, sensor, reverse, laser_major, stride, invalid):
    ns = _ns(synth, sensor)
    # laser-major: 0.6 turn from 45 deg, so that the sweep's last return is not on an azimuth threshold
    raw = synth.scan_rings(sensor, 2, reverse=reverse, laser_major=laser_major, cut=0.785 if laser_major else None,
                           coverage=0.6 if laser_major else 1.0)
    if invalid:
        raw = _mix_invalid(raw, ns, ns)
    if stride == 8:   # ring in float 3, junk in floats 4-7
        raw = np.concatenate([raw, np.random.default_rng(1).normal(0, 1e6, (len(raw), 4)).astype(np.float32)], axis=1)
        raw[::7, 4:] = np.nan
    want = RF.Features(raw, ns, synth.RING_RANGES[0])
    c = _field(aloam, ns, len(raw) + 1024)
    got = c.extract_features(raw)
    curv, label, s, e = c.debug_features(len(got["full"]))
    c.close()
    assert_matches_oracle(got, curv, label, s, e, want, ns)
    assert len(want.sharp) > 0 and len(want.less_flat) > 0


def assert_matches_oracle(got, curv, label, s, e, ref, ns):
    """the bars of test_gpu_features.py: coordinates, ring ids, scanStart / End, curvature and labels exact; intensity = ring +
    0.1 relTime within the atan2f rounding of the device and the host libm"""
    for n in NAMES:
        g, r = got[n], getattr(ref, n)
        assert g.shape == r.shape, n
        assert np.array_equal(_bits(g[:, :3]), _bits(r[:, :3])), n
        assert np.array_equal(g[:, 3].astype(np.int32), r[:, 3].astype(np.int32)), n
        assert len(g) == 0 or np.abs(g[:, 3] - r[:, 3]).max() <= 1e-5, n
    assert np.array_equal(s, ref.scan_start) and np.array_equal(e, ref.scan_end)
    for r in range(ns):   # curvature and labels are defined inside [scanStart, scanEnd]
        a, b = ref.scan_start[r], ref.scan_end[r]
        if b - a < 6:
            continue
        assert np.array_equal(curv[a:b + 1], ref.curvature[a:b + 1]), r
        assert np.array_equal(label[a:b], ref.label[a:b]), r


# ------------------------------------------------------------------------------------------------ 3. odometry
def _oracle_chain(orc, synth, sensor, frames, reverse=False, distortion=False):
    ns = _ns(synth, sensor)
    od = orc.Odometry(distortion=distortion)
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    poses, counts = [], []
    for k in range(frames):
        f = RF.Features(synth.scan_rings(sensor, k, reverse=reverse), ns, synth.RING_RANGES[0])
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
            counts.append((info["corner_corr"], info["plane_corr"]))
        else:
            counts.append(None)
        od.set_last(f.less_sharp, f.less_flat)
        poses.append(np.concatenate([qw, tw]))
    return np.array(poses), counts


def _close(got, want):
    for k in range(len(want)):
        assert np.abs(got[k, 4:] - want[k, 4:]).max() < 1e-4 and rot_angle(got[k, :4], want[k, :4]) < 1e-4, k
        assert np.abs(got[k, 4:] - want[k, 4:]).max() < 1e-7, (k, got[k, 4:] - want[k, 4:])


@pytest.mark.parametrize("sensor,reverse,distortion", [("OS64", False, 0), ("V32C", False, 0), ("V32C", True, 0), ("OS64", False, 1)])
def test_odometry_follows_the_oracle_chain(aloam, orc, synth, sensor, reverse, distortion):
    """scan_to_pose, scan_stream and scan_stream_batch over a trajectory: world poses within the tolerances of
    test_gpu_odometry.py and the oracle's correspondence counts"""
    import torch
    frames = 5
    ns = _ns(synth, sensor)
    want, counts = _oracle_chain(orc, synth, sensor, frames, reverse, bool(distortion))
    raws = [synth.scan_rings(sensor, k, reverse=reverse) for k in range(frames)]
    mp = max(len(r) for r in raws) + 1024
    c = _field(aloam, ns, mp, distortion=distortion, max_batch=2)
    got = []
    for k, r in enumerate(raws):
        q, t, st = c.scan_to_pose(r)
        got.append(np.concatenate([q, t]))
        if k > 0:
            assert (st["n_corner_corr"], st["n_plane_corr"]) == counts[k], k
    got = np.array(got)
    _close(got, want)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    c.reset_odometry()
    p, _ = c.scan_stream([d.data_ptr() for d in dev], [len(r) for r in raws], True)
    assert np.array_equal(p, got)
    c.reset_odometry()
    ptrs = np.array([[d.data_ptr()] * 2 for d in dev], np.uint64)
    cnt = np.array([[len(r)] * 2 for r in raws], np.int64)
    pb = c.scan_stream_batch(ptrs, cnt, True)
    assert np.array_equal(pb[:, 0], got) and np.array_equal(pb[:, 1], got)
    c.close()


# ------------------------------------------------------------------------------------------------ 4. mapping, lanes, snapshots, prior maps


def test_mapped_stream_follows_the_oracle_mapper(aloam, orc, synth):
    """aloam_scan_stream_mapped on an OS64 trajectory == scan_to_pose + mapper_step per scan, bit for bit; the device mapper
    against the oracle's mapper fed the same clouds and odometry poses, with the bars of test_gpu_cubemap.py's mapping loop, up
    to the frame whose insert overflows a cube slab (16384 corner points: ALOAM_FLAG_CUBE_OVERFLOW, the device drops the
    overflow and the oracle has no limit; this dense 64-ring trajectory reaches it in a few frames)"""
    import torch
    sensor, frames = "OS64", 6
    ns = _ns(synth, sensor)
    raws = [synth.scan_rings(sensor, k) for k in range(frames)]
    mp = max(len(r) for r in raws) + 1024
    c = _field(aloam, ns, mp, max_map_points=400000)
    dev = [torch.from_numpy(r).cuda() for r in raws]
    odom, mapped = c.scan_stream_mapped([d.data_ptr() for d in dev], [len(r) for r in raws], True)
    c.close()
    want, _ = _oracle_chain(orc, synth, sensor, frames)
    _close(odom, want)
    c = _field(aloam, ns, mp, max_map_points=400000)
    c.mapper_reset()
    cm = orc.CubeMap()
    compared = 0
    for k, raw in enumerate(raws):
        gq, gt, _ = c.scan_to_pose(raw)
        assert np.array_equal(np.concatenate([gq, gt]), odom[k]), k
        f = c.extract_features(raw)
        mq, mt, st = c.mapper_step(f["less_sharp"], f["less_flat"], gq, gt)
        assert np.array_equal(np.concatenate([mq, mt]), mapped[k]), k
        if st["flags"] & aloam.FLAG_CUBE_OVERFLOW or compared < k:
            continue
        compared += 1
        pose, info = cm.step(f["less_sharp"], f["less_flat"], gq, gt, 0.2, 0.4)
        assert bool(info["optimised"]) == (not (st["flags"] & aloam.FLAG_MAP_TOO_THIN))
        assert np.abs(mt - pose[4:]).max() < 1e-4 and rot_angle(mq, pose[:4]) < 1e-4, (k, mt - pose[4:])
        so, sg = cm.state(), c.mapper_state()
        assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
        assert abs(sg["total_corner"] - so["total_corner"]) <= 5 and abs(sg["total_surf"] - so["total_surf"]) <= 20
        same = differ = 0
        for idx in so["valid"]:
            for which in (0, 1):
                a, b = c.mapper_cube(which, idx), cm.cube(which, idx)
                if a.shape != b.shape:
                    differ += 1
                    continue
                same += 1
                if len(a):
                    assert np.abs(a[:, :3] - b[:, :3]).max() < 2e-5 and np.abs(a[:, 3] - b[:, 3]).max() < 1e-4, (k, idx, which)
        assert same >= 1 and differ <= 4
    assert compared >= 3
    c.close()


def _lane_runs(synth):
    """three OS64 trajectories: from scan 0, ring ids reversed, and from scan 3"""
    return [[synth.scan_rings("OS64", k) for k in range(0, 5)], [synth.scan_rings("OS64", k, reverse=True) for k in range(0, 5)],
            [synth.scan_rings("OS64", k) for k in range(3, 8)]]


def _run_lanes(c, scans, ops, mapped=True):
    import torch
    dev = [[torch.from_numpy(s).cuda() for s in col] for col in scans]
    n, b = len(scans[0]), len(scans)
    ptrs = np.array([[dev[j][k].data_ptr() for j in range(b)] for k in range(n)], np.uint64)
    cnt = np.array([[len(scans[j][k]) for j in range(b)] for k in range(n)], np.int64)
    return c.scan_stream_lanes(ptrs, cnt, np.asarray(ops, np.int32), True, mapped=mapped)


def test_lanes_equal_their_solo_runs_and_snapshots_resume(aloam, synth):
    runs = _lane_runs(synth)
    mp = max(len(s) for r in runs for s in r) + 1024
    n = len(runs[0])
    ops = [[START] * 3] + [[SCAN] * 3] * (n - 1)
    c = _field(aloam, 64, mp, max_map_points=200000, max_batch=3)
    odom, mapped = _run_lanes(c, runs, ops)
    for j, r in enumerate(runs):
        s = _field(aloam, 64, mp, max_map_points=200000)
        so, sm = _run_lanes(s, [r], [[START]] + [[SCAN]] * (n - 1))
        assert np.array_equal(odom[:, j], so[:, 0]) and np.array_equal(mapped[:, j], sm[:, 0]), j
        s.close()
    # suspend lane 1 after three scans, resume it in lane 0 of another context: the uninterrupted run
    c.reset_odometry()
    _run_lanes(c, [runs[1][:3]], [[START], [SCAN], [SCAN]])
    blob = c.lane_save(0)
    assert aloam.snapshot_info(blob)["n_scans"] == 64 and int(np.frombuffer(blob[216:220].tobytes(), np.int32)[0]) == aloam.RING_FIELD
    r = _field(aloam, 64, mp, max_map_points=200000)
    r.lane_restore(0, blob)
    ro, rm = _run_lanes(r, [runs[1][3:]], [[SCAN]] * (n - 3))
    assert np.array_equal(ro[:, 0], odom[3:, 1]) and np.array_equal(rm[:, 0], mapped[3:, 1])
    r.close()
    # a context of the other ring source refuses it
    e = aloam.Aloam(n_scans=64, max_points=mp, max_map_points=200000, minimum_range=0.3, line_res=0.2, plane_res=0.4)
    _expect(aloam, ERR_SNAPSHOT, lambda: e.lane_restore(0, blob))
    _expect(aloam, ERR_SNAPSHOT, lambda: e.prior_map_load(blob))
    e.close()
    c.close()


def test_prior_map_built_from_an_os64_map_localises_os64_scans(aloam, synth):
    """a mapped OS64 lane's store, built into a prior map from its two clouds, localises a lane on the same scans exactly as the
    loaded snapshot does"""
    runs = _lane_runs(synth)[0]
    mp = max(len(s) for s in runs) + 1024
    m = _field(aloam, 64, mp, max_map_points=200000)
    _, mapped = _run_lanes(m, [runs], [[START]] + [[SCAN]] * (len(runs) - 1))
    blob = m.lane_save(0)
    m.close()
    split = aloam.snapshot_store_clouds(blob)
    out = []
    for how in ("load", "build"):
        c = _field(aloam, 64, mp, max_map_points=200000)
        if how == "load":
            c.prior_map_load(blob)
        else:
            assert c.prior_map_build(split["corner"], split["surf"], split["centre"]) == (0, 0)
        c.lane_localise(0, mapped[2, 0, :4], mapped[2, 0, 4:])
        out.append(_run_lanes(c, [runs[2:]], [[START]] + [[SCAN]] * (len(runs) - 3))[1])
        c.close()
    assert np.array_equal(out[0], out[1])
    assert np.abs(out[1][:, 0, 4:] - mapped[2:, 0, 4:]).max() < 0.05


# ------------------------------------------------------------------------------------------------ 5. errors and cost
def test_configuration_errors(aloam):
    _expect(aloam, ERR_INVALID_ARG, lambda: aloam.Aloam(n_scans=16, ring_source=2))
    for ns in (0, 65):
        _expect(aloam, ERR_UNSUPPORTED_SCANS, lambda: aloam.Aloam(n_scans=ns, ring_source=aloam.RING_FIELD))
    _expect(aloam, ERR_UNSUPPORTED_SCANS, lambda: aloam.Aloam(n_scans=48))
    for ns in (1, 48, 64):
        aloam.Aloam(n_scans=ns, ring_source=aloam.RING_FIELD, max_points=4096).close()


def test_a_ring_over_max_ring_points_is_refused(aloam, synth):
    raw = synth.scan_rings("R2", 0)
    c = _field(aloam, 2, len(raw) + 1024, max_ring_points=1024)
    assert np.bincount(raw[:, 3].astype(int)).min() > 1024
    _expect(aloam, ERR_RING_TOO_LARGE, lambda: c.extract_features(raw))
    c.extract_features(raw[: len(raw) // 4])   # two rings of ~450 returns
    c.close()


def test_launch_count_per_stream_step_is_the_same_in_both_modes(aloam, synth):
    import torch
    raws = [synth.scan("HDL-64", k) for k in range(4)]
    counts = []
    for rs in (aloam.RING_ELEVATION, aloam.RING_FIELD):
        c = aloam.Aloam(n_scans=64, max_points=140000, ring_source=rs, max_map_points=400000)
        dev = [torch.from_numpy(RF.formula_rings(r, 64)).cuda() for r in raws]
        ptr, cnt = [d.data_ptr() for d in dev], [len(r) for r in raws]
        c.scan_stream(ptr[:1], cnt[:1], True)
        n0 = c.launch_count()
        p, _ = c.scan_stream(ptr[1:], cnt[1:], True)
        n1 = c.launch_count()
        c.reset_odometry()
        o, m = c.scan_stream_mapped(ptr, cnt, True)
        counts.append((n1 - n0, c.launch_count() - n1, p.tobytes(), o.tobytes(), m.tobytes()))
        c.close()
    assert counts[0] == counts[1]
