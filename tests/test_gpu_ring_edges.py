"""GPU parity of ring assignment (features.cu ring_of, scanRegistration.cpp:166-205) at every decision of the 16-, 32- and
64-line formulas (tests/ring_edge_cases.py): edge sweeps whose returns take every float32 angle within 40 ulps of each
decision, alone and through the batched stream, and chains over beam layouts whose lasers sit off the bin centres and off the
sensor origin, against the oracle, the oracle chains and the reference's own sources.  Feature bars: those of
tests/test_gpu_features_edges.py (xyz, ring ids, scanStart / scanEnd, curvature, labels and the four clouds bit-exact; the
relTime fraction within 1e-5)."""
import numpy as np
import pytest

import lane_refs as R
import ring_edge_cases as E
from conftest import rot_angle
from test_gpu_sweep_seams import check_features

pytestmark = pytest.mark.gpu

SENSORS = [16, 32, 64]
NS = {"VLP-16-offset": 16, "HDL-32-offset": 32, "HDL-64-offset": 64}


@pytest.fixture(scope="module")
def sweeps():
    return {ns: E.edge_scan(ns)[0] for ns in SENSORS}


@pytest.mark.parametrize("ns", SENSORS)
def test_features_on_edge_sweeps(aloam, orc, sweeps, ns):
    """aloam_extract_features against the oracle on every decision of the formula"""
    raw = sweeps[ns]
    ref = orc.Features(raw, ns, E.MIN_RANGE[ns], orc.SORT_CANONICAL)
    c = aloam.Aloam(n_scans=ns, max_points=60000)
    try:
        check_features(c.extract_features(raw), ref, c, ("edge sweep", ns))
    finally:
        c.close()


@pytest.mark.parametrize("ns", SENSORS)
def test_features_on_edge_sweeps_match_the_reference_source(aloam, orc, sweeps, ns):
    """aloam_extract_features against the clouds the reference's own laserCloudHandler publishes on the edge sweeps"""
    from test_gpu_vs_reference_chains import _load
    import refsource
    raw = sweeps[ns]
    ref = _load(refsource.ref_registration, ns, E.MIN_RANGE[ns]).run(raw, orc.SORT_CANONICAL)
    c = aloam.Aloam(n_scans=ns, max_points=60000)
    try:
        got = c.extract_features(raw)
    finally:
        c.close()
    for name in ("full", "sharp", "less_sharp", "flat", "less_flat"):
        g, r_ = got[name], ref[name]
        assert g.shape == r_.shape, (ns, name, g.shape, r_.shape)
        assert np.array_equal(g[:, :3], r_[:, :3]), (ns, name)
        assert np.array_equal(g[:, 3].astype(np.int32), r_[:, 3].astype(np.int32)), (ns, name)
        assert len(g) == 0 or float(np.abs(g[:, 3] - r_[:, 3]).max()) <= 1e-5, (ns, name)


@pytest.mark.parametrize("max_ring,stride", [(4096, 4), (2304, 4), (4096, 8)])
def test_batched_edge_sweeps_equal_solo(aloam, max_ring, stride):
    """aloam_scan_stream_batch, four VLP-16 lanes each with its own edge sweeps (different sector orders, ranges and room
    shifts scan by scan): every lane bit-identical to its solo aloam_scan_stream, with the 256-thread ring kernel at 2304
    and with 8-float points (host-resident: device-resident scans are 4-float)"""
    import torch
    lanes, n_scan = 4, 4
    trajs = []
    for b in range(lanes):
        tr = []
        for k in range(n_scan):
            raw = E.edge_scan(16, seed=b, shift=(0.05 * k, 0.02 * k * (b + 1)))[0]
            assert np.bincount(E.ring_ids(raw, 16)[E.ring_ids(raw, 16) >= 0]).max() <= max_ring
            if stride == 8:
                wide = np.full((len(raw), 8), np.float32(7.5), np.float32)
                wide[:, :4] = raw
                raw = wide
            tr.append(raw)
        trajs.append(tr)
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    resident = stride == 4
    if resident:
        keep = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
        ptr = lambda b, k: keep[b][k].data_ptr()
    else:
        keep = [[np.ascontiguousarray(s) for s in tr] for tr in trajs]
        ptr = lambda b, k: keep[b][k].ctypes.data
    ptrs = np.array([[ptr(b, k) for b in range(lanes)] for k in range(n_scan)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(lanes)] for k in range(n_scan)])
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_batch=lanes, max_ring_points=max_ring)
    try:
        poses = c.scan_stream_batch(ptrs, counts, resident, stride=stride)
    finally:
        c.close()
    assert np.isfinite(poses).all()
    solo = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_ring_points=max_ring)
    try:
        for b in range(lanes):
            solo.reset_odometry()
            sp, _ = solo.scan_stream([ptr(b, k) for k in range(n_scan)], counts[:, b], resident, stride=stride)
            assert np.array_equal(sp, poses[:, b]), b
    finally:
        solo.close()


def _layout_scans(synth, name, n):
    return [np.ascontiguousarray(E.layout_scan(synth, name, k)) for k in range(n)]


@pytest.mark.parametrize("name,distortion", [("HDL-64-offset", 0), ("VLP-16-offset", 0), ("VLP-16-offset", 1)])
def test_scan_to_pose_and_stream_on_offset_layouts(aloam, orc, synth, name, distortion):
    """scan_to_pose over five scans of a layout: correspondence counts equal the oracle chain's, poses within 1e-4; the
    scan stream gives the per-scan poses bit for bit.  With DISTORTION the ring enters the interpolation ratio s through
    int(intensity)"""
    ns = NS[name]
    mr = E.MIN_RANGE[ns]
    raws = _layout_scans(synth, name, 5)
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
            od.set_last(f.less_sharp, f.less_flat)
            gq, gt, st = ctx.scan_to_pose(raw)
            per_scan.append(np.concatenate([gq, gt]))
            worst = max(worst, float(np.abs(gt - tw).max()), rot_angle(gq, qw))
            if k > 0:
                assert (st["n_corner_corr"], st["n_plane_corr"]) == (info["corner_corr"], info["plane_corr"]), (k, st, info)
                assert info["corner_corr"] > 0 and info["plane_corr"] > 0
        assert worst < 1e-4, worst
        assert float(np.abs(tw).max()) > 0.05
        ctx.reset_odometry()
        poses, _ = ctx.scan_stream([r.ctypes.data for r in raws], [len(r) for r in raws], False)
        assert np.array_equal(poses, np.array(per_scan)), np.abs(poses - np.array(per_scan)).max()
    finally:
        ctx.close()
    print("%s distortion=%d: worst pose deviation from the oracle chain %.2e" % (name, distortion, worst))


def test_hdl64_offset_layout_matches_the_reference_odometry(aloam, orc, synth):
    """scan_to_pose over the HDL-64 layout against the reference's scanRegistration -> laserOdometry sources: world pose of
    every scan within ODOM_BAR, both correspondence counts equal"""
    import test_gpu_vs_reference_chains as VC
    raws = _layout_scans(synth, "HDL-64-offset", 5)
    ref, counts, _ = VC._ref_odometry_chain(orc, synth, "HDL-64", raws, "ring_edges_hdl64")
    c = aloam.Aloam(n_scans=64, max_points=200000)
    try:
        for k, raw in enumerate(raws):
            q, t, st = c.scan_to_pose(raw)
            VC._near(np.concatenate([q, t]), ref[k], VC.ODOM_BAR, "odometry chains", ("HDL-64-offset", k))
            if k > 0:
                assert (st["n_corner_corr"], st["n_plane_corr"]) == counts[k], (k, st, counts[k])
    finally:
        c.close()
    assert float(np.abs(ref[:, 4:]).max()) > 0.05


def test_scan_stream_mapped_on_the_vlp16_offset_layout(aloam, orc, synth):
    """scan_stream_mapped over six scans of the VLP-16 layout: odometry rows equal scan_stream's bit for bit, odometry and
    map poses within 1e-4 of the oracle chain (the bars of test_scan_stream_mapped_on_a_seam_trajectory)"""
    raws = _layout_scans(synth, "VLP-16-offset", 6)
    mapped = R.solo(aloam, raws, "ring-edges-VLP-16-offset", True)
    plain = R.solo(aloam, raws, "ring-edges-VLP-16-offset", False)
    assert np.array_equal(mapped["odom"], plain["odom"])
    o, m = R.oracle(orc, synth, raws, "ring-edges-VLP-16-offset", True)
    R.assert_near(mapped["odom"], o, "odometry")
    dt, dr = R.assert_near(mapped["map"], m, "map")
    print("VLP-16-offset mapped stream: map poses within %.2e m / %.2e rad of the oracle chain" % (dt, dr))
