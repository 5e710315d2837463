"""GPU: driver rings up to 128 (aloam_create_wide).  Up to 64 rings a wide-created context is the context of aloam_create, bit
for bit; on 65..128-ring tables (synth.WIDE_RING_SENSORS) the device follows the wide oracle (tests/wide_ring_oracle.py) in the
features at the bars of test_gpu_ring_field.py, and the oracle chain in odometry and mapping; lanes, snapshots, prior maps,
relocalisation and recovery run unchanged on an OS1-128-shaped trajectory."""
import numpy as np
import pytest

import wide_ring_oracle as WR
from conftest import rot_angle
from test_gpu_ring_field import NAMES, _bits, _expect, _mix_invalid, _run_lanes, assert_matches_oracle

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_RING_TOO_LARGE, ERR_NOT_RING_MAJOR, ERR_SNAPSHOT = -1, -7, -8, -11
IDLE, SCAN, START = 0, 1, 2


def _wide(aloam, ns, max_points, **kw):
    mr, lr, pr = 0.3, 0.2, 0.4   # synth.RING_RANGES
    return aloam.Aloam(n_scans=ns, max_points=max_points, ring_source=aloam.RING_FIELD, minimum_range=mr, line_res=lr, plane_res=pr,
                       wide=True, **kw)


def _dev(raws):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(r)).cuda() for r in raws]


# ------------------------------------------------------------------------------------------------ 1. up to 64 rings: the same context
@pytest.mark.parametrize("ns,field", [(16, False), (32, False), (64, False), (40, True), (64, True)])
def test_wide_entry_point_equals_aloam_create_up_to_64_rings(aloam, synth, ns, field):
    if field:
        sensor = "L40" if ns == 40 else "OS64"
        raws = [synth.scan_rings(sensor, k) for k in range(4)]
        kw = dict(ring_source=aloam.RING_FIELD, minimum_range=0.3, line_res=0.2, plane_res=0.4)
    else:
        sensor = {16: "VLP-16", 32: "HDL-32", 64: "HDL-64"}[ns]
        raws = [synth.scan(sensor, k) for k in range(4)]
        kw = dict(minimum_range=synth.SENSORS[sensor][2], line_res=synth.SENSORS[sensor][3], plane_res=synth.SENSORS[sensor][4])
    mp = max(len(r) for r in raws) + 1024
    dev = _dev(raws)
    ptr, cnt = [d.data_ptr() for d in dev], [len(r) for r in raws]
    out = []
    for wide in (False, True):
        c = aloam.Aloam(n_scans=ns, max_points=mp, max_map_points=400000, wide=wide, **kw)
        f = c.extract_features(raws[1])
        dbg = c.debug_features(len(f["full"]))
        n0 = c.launch_count()
        o, m = c.scan_stream_mapped(ptr, cnt, True)
        n1 = c.launch_count()
        store = (c.mapper_export(aloam.EXPORT_MAP), c.mapper_export(aloam.EXPORT_SURROUND))
        c.reset_odometry()
        p = np.array([np.concatenate(c.scan_to_pose(r)[:2]) for r in raws])
        out.append((f, dbg, o, m, n1 - n0, store, p))
        c.close()
    (fa, da, oa, ma, na, sa, pa), (fb, db, ob, mb, nb, sb, pb) = out
    for n in NAMES:
        assert np.array_equal(_bits(fa[n]), _bits(fb[n])), n
    for a, b in zip(da, db):
        assert np.array_equal(a, b)
    assert np.array_equal(oa, ob) and np.array_equal(ma, mb) and na == nb and np.array_equal(pa, pb)
    for a, b in zip(sa, sb):
        assert np.array_equal(np.asarray(a), np.asarray(b))


# ------------------------------------------------------------------------------------------------ 2. features against the wide oracle
FEATURE_CASES = [  # sensor, reverse, laser_major, stride, invalid
    ("E65", False, False, 4, False), ("E65", True, True, 8, True), ("L96", False, False, 8, True), ("L96", True, False, 4, False),
    ("OS128", False, False, 4, False), ("OS128", True, True, 8, True), ("OS128", False, True, 4, True), ("V128", False, False, 4, False),
    ("V128", True, False, 8, False),
]   # (invalid V128 scans would put 1 in 40 of 230 k returns into ring 0 with -0.0: ALOAM_ERR_RING_TOO_LARGE, so V128 has no invalid case)


def _invalid(raw, ns, seed):
    """_mix_invalid, then one return in 80 gets 128, 127.5 or -1 (dropped)"""
    out = _mix_invalid(raw, ns, seed)
    rng = np.random.default_rng(seed + 1)
    pick = rng.permutation(len(out))[: len(out) // 80]
    out[pick, 3] = np.array([128.0, 127.5, -1.0], np.float32)[np.arange(len(pick)) % 3]
    return out


@pytest.mark.parametrize("sensor,reverse,laser_major,stride,invalid", FEATURE_CASES)
def test_features_equal_the_wide_oracle(aloam, synth, sensor, reverse, laser_major, stride, invalid):
    ns = WR.n_rings(synth, sensor)
    raw = WR.scan(synth, sensor, 2, reverse=reverse, laser_major=laser_major, cut=0.785 if laser_major else None,
                  coverage=0.6 if laser_major else 1.0)
    if invalid:
        raw = _invalid(raw, ns, ns)
    if stride == 8:
        raw = np.concatenate([raw, np.random.default_rng(1).normal(0, 1e6, (len(raw), 4)).astype(np.float32)], axis=1)
        raw[::7, 4:] = np.nan
    want = WR.Features(raw, ns, synth.RING_RANGES[0])
    c = _wide(aloam, ns, len(raw) + 1024)
    got = c.extract_features(raw)
    curv, label, s, e = c.debug_features(len(got["full"]))
    c.close()
    assert len(s) == ns and len(e) == ns
    assert_matches_oracle(got, curv, label, s, e, want, ns)
    assert len(want.sharp) > 0 and len(want.less_flat) > 0 and int(want.full[:, 3].max()) >= 64
    if sensor == "OS128" and not laser_major:   # whole scans: the highest beams' rings of 17..39 returns are compared too
        n = np.bincount(want.full[:, 3].astype(np.int64), minlength=ns)
        assert ((n >= 17) & (n < 40)).any()


def test_os128_at_2048_azimuth_steps(aloam, synth):
    """262 144 returns, 2048 per ring: max_ring_points = 2048, in a batch of two (the 256-thread ring kernel) as well"""
    raw = WR.scan(synth, "OS128", 1, n_az=2048)
    assert np.bincount(raw[:, 3].astype(int)).max() <= 2048 and len(raw) > 200000
    want = WR.Features(raw, 128, synth.RING_RANGES[0])
    c = _wide(aloam, 128, 262144, max_ring_points=2048, max_batch=2)
    got = c.extract_features(raw)
    curv, label, s, e = c.debug_features(len(got["full"]))
    assert_matches_oracle(got, curv, label, s, e, want, 128)
    c.close()


# ------------------------------------------------------------------------------------------------ 3. odometry
def _close(got, want):
    for k in range(len(want)):
        assert np.abs(got[k, 4:] - want[k, 4:]).max() < 1e-4 and rot_angle(got[k, :4], want[k, :4]) < 1e-4, k
        assert np.abs(got[k, 4:] - want[k, 4:]).max() < 1e-7, (k, got[k, 4:] - want[k, 4:])


@pytest.mark.parametrize("sensor,reverse,distortion,nearby", [("OS128", False, 0, 2.5), ("OS128", True, 1, 2.5), ("V128", False, 0, 7.5),
                                                              ("L96", False, 0, float("inf")), ("E65", True, 1, 2.5)])
def test_odometry_follows_the_oracle_chain(aloam, orc, synth, sensor, reverse, distortion, nearby):
    frames = 5
    ns = WR.n_rings(synth, sensor)
    want, counts = WR.odometry_chain(orc, synth, sensor, frames, reverse, bool(distortion), nearby)
    raws = [WR.scan(synth, sensor, k, reverse=reverse) for k in range(frames)]
    c = _wide(aloam, ns, max(len(r) for r in raws) + 1024, distortion=distortion, nearby_scan=nearby)
    got = []
    for k, r in enumerate(raws):
        q, t, st = c.scan_to_pose(r)
        got.append(np.concatenate([q, t]))
        if k > 0:
            assert (st["n_corner_corr"], st["n_plane_corr"]) == counts[k], k
    got = np.array(got)
    _close(got, want)
    dev = _dev(raws)
    c.reset_odometry()
    p, _ = c.scan_stream([d.data_ptr() for d in dev], [len(r) for r in raws], True)
    assert np.array_equal(p, got)
    c.close()


def test_set_last_takes_rings_up_to_127(aloam, synth):
    f = WR.Features(WR.scan(synth, "OS128", 0), 128, synth.RING_RANGES[0])
    c = _wide(aloam, 128, 200000)
    c.odometry_set_last(f.less_sharp, f.less_flat)   # ring-major, int(intensity) up to 127
    assert int(f.less_flat[:, 3].max()) == 127
    bad = f.less_flat.copy()
    bad[-1, 3] = 128.0
    _expect(aloam, ERR_NOT_RING_MAJOR, lambda: c.odometry_set_last(f.less_sharp, bad))
    c.close()
    n = _wide(aloam, 64, 200000)   # a 64-wide context refuses ring 64
    _expect(aloam, ERR_NOT_RING_MAJOR, lambda: n.odometry_set_last(f.less_sharp, f.less_flat))
    n.close()
    # a ring above max_ring_points
    raw = synth.scan_rings("OS128", 0, n_az=2048)
    c = _wide(aloam, 128, len(raw) + 1024, max_ring_points=1024)
    _expect(aloam, ERR_RING_TOO_LARGE, lambda: c.extract_features(raw))
    c.close()


# ------------------------------------------------------------------------------------------------ 4. mapping, lanes, snapshots
def test_mapped_stream_follows_the_oracle_mapper_with_cube_growth(aloam, orc, synth):
    frames = 5
    raws = [WR.scan(synth, "OS128", k) for k in range(frames)]
    mp = max(len(r) for r in raws) + 1024
    c = _wide(aloam, 128, mp, max_map_points=400000)
    c.set_cube_growth(True)
    dev = _dev(raws)
    odom, mapped = c.scan_stream_mapped([d.data_ptr() for d in dev], [len(r) for r in raws], True)
    c.close()
    want, _ = WR.odometry_chain(orc, synth, "OS128", frames)
    _close(odom, want)
    c = _wide(aloam, 128, mp, max_map_points=400000)
    c.set_cube_growth(True)
    c.mapper_reset()
    cm = orc.CubeMap()
    for k, raw in enumerate(raws):
        gq, gt, _ = c.scan_to_pose(raw)
        assert np.array_equal(np.concatenate([gq, gt]), odom[k]), k
        f = c.extract_features(raw)
        mq, mt, st = c.mapper_step(f["less_sharp"], f["less_flat"], gq, gt)
        assert np.array_equal(np.concatenate([mq, mt]), mapped[k]), k
        assert not st["flags"] & aloam.FLAG_CUBE_OVERFLOW, k
        pose, info = cm.step(f["less_sharp"], f["less_flat"], gq, gt, 0.2, 0.4)
        assert np.abs(mt - pose[4:]).max() < 1e-4 and rot_angle(mq, pose[:4]) < 1e-4, (k, mt - pose[4:])
        so, sg = cm.state(), c.mapper_state()
        assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
    c.close()


def test_sixteen_lanes_snapshots_and_a_64_ring_context(aloam, synth):
    n = 6
    scans = [WR.scan(synth, "OS128", k) for k in range(n + 4)]
    mp = max(len(s) for s in scans) + 1024
    cols, ops = [], []
    for j in range(16):   # lane j starts at step j % 4 on scan j % 3 of the trajectory (reversed ring ids on odd lanes)
        s0 = j % 4
        col = [scans[0]] * s0 + [scans[j % 3 + k] if j % 2 == 0 else np.ascontiguousarray(np.c_[scans[j % 3 + k][:, :3], 127 - scans[j % 3 + k][:, 3]])
                                 for k in range(n - s0)]
        cols.append(col)
        ops.append([IDLE] * s0 + [START] + [SCAN] * (n - s0 - 1))
    ops = np.array(ops).T
    c = _wide(aloam, 128, mp, max_map_points=200000, max_batch=16)
    odom, mapped = _run_lanes(c, cols, ops)
    c.close()
    for j in (0, 5, 10, 15):
        s0 = j % 4
        s = _wide(aloam, 128, mp, max_map_points=200000)
        so, sm = _run_lanes(s, [cols[j][s0:]], [[START]] + [[SCAN]] * (n - s0 - 1))
        assert np.array_equal(odom[s0:, j], so[:, 0]) and np.array_equal(mapped[s0:, j], sm[:, 0]), j
        s.close()
    # suspend lane 0's run after three scans, resume it in another context: the uninterrupted run
    r0 = cols[0]
    c = _wide(aloam, 128, mp, max_map_points=200000)
    _run_lanes(c, [r0[:3]], [[START], [SCAN], [SCAN]])
    blob = c.lane_save(0)
    c.close()
    assert aloam.snapshot_info(blob)["n_scans"] == 128
    r = _wide(aloam, 128, mp, max_map_points=200000)
    r.lane_restore(0, blob)
    ro, rm = _run_lanes(r, [r0[3:]], [[SCAN]] * (n - 3))
    assert np.array_equal(ro[:, 0], odom[3:, 0]) and np.array_equal(rm[:, 0], mapped[3:, 0])
    r.close()
    for ns in (64, 96):   # any other n_scans refuses it
        e = _wide(aloam, ns, mp, max_map_points=200000)
        _expect(aloam, ERR_SNAPSHOT, lambda: e.lane_restore(0, blob))
        e.close()


# ------------------------------------------------------------------------------------------------ 5. prior maps, relocalisation, recovery
def test_prior_map_relocalises_and_recovers_os128_scans(aloam, synth):
    runs = [WR.scan(synth, "OS128", k) for k in range(6)]
    mp = max(len(s) for s in runs) + 1024
    import recovery_cases as RV
    import track_cases as TC
    # cube growth on: at one slab per cube this store overflows from the third frame on (flag 8), and the prior map built from
    # the truncated store is not the oracle's
    m = _wide(aloam, 128, mp, max_map_points=200000)
    m.set_cube_growth(True)
    m.set_map_rows(True, TC.ISQ, TC.PTS)
    _, mapped = _run_lanes(m, [runs], [[START]] + [[SCAN]] * (len(runs) - 1))
    assert not (m.map_rows(len(runs))["flags"] & aloam.FLAG_CUBE_OVERFLOW).any()
    blob = m.lane_save(0)
    m.close()
    split = aloam.snapshot_store_clouds(blob)
    c = _wide(aloam, 128, mp, max_map_points=200000)
    assert c.prior_map_build(split["corner"], split["surf"], split["centre"]) == (0, 0)
    # relocalise scan 3 from a grid of hypotheses around the true map pose
    true = mapped[3, 0]
    hyps = []
    for dx in (-2.0, 0.0, 2.0):
        for dy in (-2.0, 0.0, 2.0):
            for yaw in (-0.2, 0.0, 0.2):
                h = true.copy()
                dq = np.array([0, 0, np.sin(yaw / 2), np.cos(yaw / 2)])
                x1, y1, z1, w1 = dq; x2, y2, z2, w2 = h[:4]
                h[:4] = [w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
                         w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2]
                h[4:] += (dx, dy, 0.0)
                hyps.append(h)
    f = c.extract_features(runs[3])
    res, scores = c.prior_relocalise(np.array(hyps), f["less_sharp"], f["less_flat"], refine=1)
    assert res[0]["hyp"] == 13 and scores.argmax() == 13   # the undisplaced hypothesis
    assert np.abs(res[0]["pose"][4:] - true[4:]).max() < 0.05
    # a recovery-armed localising lane started 1.5 m off re-seats on the prior map, adopting on its START row the candidate and
    # score of the host model of recovery on the oracle's map (tests/recovery_cases.py via wide_ring_oracle.recovery_model)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, RV.deltas(aloam))
    start = mapped[2, 0].copy()
    start[4:] += (1.5, -1.5, 0.0)
    c.lane_localise(0, start[:4], start[4:])
    o, m2 = _run_lanes(c, [runs[2:]], [[START]] + [[SCAN]] * (len(runs) - 3))
    rec = c.recovery_rows(len(runs) - 2)
    rows = c.map_rows(len(runs) - 2)
    c.close()
    _, want = WR.recovery_model(aloam, synth, (1.5, -1.5), frames=len(runs))
    assert rec["adopted"].tolist() == [int(r["adopted"]) for r in want]
    assert rec["best"].tolist() == [r["best"] for r in want] and rec["best_score"].tolist() == [r["best_score"] for r in want]
    assert rows["score"][0] == want[0]["score"] and rows["n_score"][0] == want[0]["n_score"]
    assert np.abs(m2[-1, 0, 4:] - mapped[-1, 0, 4:]).max() < 0.1
