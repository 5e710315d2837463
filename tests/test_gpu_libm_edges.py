"""GPU parity of the transcendentals of ring assignment and the sweep walk at their rounding edges (tests/libm_edge_cases.py):
returns whose elevation lies within a few double ulps of a float midpoint between two ring decisions, and returns on every
float within +-3 ulps of each azimuth threshold of the walk.  Bars, against the oracle: the ring-major cloud bit-exact
including intensity, scanStart / scanEnd, curvature, labels and the four clouds bit-exact; per threshold return, the
device's int(intensity) and relTime equal the host's."""
import numpy as np
import pytest

import libm_edge_cases as M
import ring_edge_cases as E

pytestmark = pytest.mark.gpu

SENSORS = [16, 32, 64]


def check_exact(got, ref, ctx, tag):
    assert got["full"].shape == ref.full.shape, tag
    assert np.array_equal(got["full"].view(np.uint32), ref.full.view(np.uint32)), (tag, _diff(got["full"], ref.full))
    curv, label, s, e = ctx.debug_features(ref.full.shape[0])
    ns = len(ref.scan_start)
    assert np.array_equal(s[:ns], ref.scan_start) and np.array_equal(e[:ns], ref.scan_end), tag
    for r in range(ns):
        a, b = ref.scan_start[r], ref.scan_end[r]
        if b - a < 6:
            continue
        assert np.array_equal(curv[a:b + 1].view(np.uint32), ref.curvature[a:b + 1].view(np.uint32)), (tag, r)
        assert np.array_equal(label[a:b], ref.label[a:b]), (tag, r)
    for name in ["sharp", "less_sharp", "flat", "less_flat"]:
        g, r_ = got[name], getattr(ref, name)
        assert g.shape == r_.shape and np.array_equal(g.view(np.uint32), r_.view(np.uint32)), (tag, name)


def _diff(g, r):
    if g.shape != r.shape:
        return "shapes"
    bad = np.flatnonzero(np.any(g.view(np.uint32) != r.view(np.uint32), axis=1))
    return [(int(i), g[i].tolist(), r[i].tolist()) for i in bad[:8]]


@pytest.mark.parametrize("ns", SENSORS)
def test_features_on_midpoint_scans(aloam, orc, ns):
    """returns on the float midpoints of every ring decision: the device's ring equals the host's on each"""
    raw, kind = M.midpoint_scan(ns)
    ref = orc.Features(raw, ns, E.MIN_RANGE[ns], orc.SORT_CANONICAL)
    c = aloam.Aloam(n_scans=ns, max_points=60000)
    try:
        check_exact(c.extract_features(raw), ref, c, ("midpoint", ns))
    finally:
        c.close()


@pytest.fixture(scope="module")
def scenes(synth):
    return {ns: M.threshold_scenes(ns, list(synth.nominal_elevations(E.SENSOR_OF[ns]))) for ns in SENSORS}


@pytest.mark.parametrize("ns", SENSORS)
def test_features_on_threshold_scenes(aloam, orc, scenes, ns):
    """every azimuth threshold scene: the device's int(intensity) and relTime of each threshold return equal the host's
    (a failure lists return, comparison, host ori and device intensity), then the full bars"""
    c = aloam.Aloam(n_scans=ns, max_points=60000)
    fails = []
    try:
        for name, s, raw, marks in scenes[ns]:
            ref = orc.Features(raw, ns, E.MIN_RANGE[ns], orc.SORT_CANONICAL)
            got = c.extract_features(raw)
            g, r = got["full"], ref.full
            if g.shape == r.shape:
                key = {bytes(p): i for i, p in enumerate(np.ascontiguousarray(raw[:, :3]))}
                host = M.host_ori(raw[:, 0], raw[:, 1])
                for k in np.flatnonzero(np.any(g.view(np.uint32) != r.view(np.uint32), axis=1)):
                    i = key.get(bytes(np.ascontiguousarray(r[k, :3])), -1)
                    fails.append((name, int(i), int(marks[i]) if i >= 0 else None, float(host[i]) if i >= 0 else None,
                                  float(r[k, 3]), float(g[k, 3])))
            else:
                fails.append((name, "shape", g.shape, r.shape))
            if not fails:
                check_exact(got, ref, c, (name, ns))
    finally:
        c.close()
    assert not fails, fails[:20]


def test_batched_threshold_scenes_equal_solo(aloam, scenes):
    """aloam_scan_stream_batch, 16 VLP-16 lanes, a different threshold scene per lane and scan: every lane's poses
    bit-identical to its solo aloam_scan_stream"""
    sc = scenes[16]
    lanes, n_scan = 16, 3
    trajs = [[np.ascontiguousarray(sc[(b * n_scan + k) % len(sc)][2]) for k in range(n_scan)] for b in range(lanes)]
    maxn = max(s.shape[0] for tr in trajs for s in tr)
    ptrs = np.array([[trajs[b][k].ctypes.data for b in range(lanes)] for k in range(n_scan)], np.uint64)
    counts = np.array([[trajs[b][k].shape[0] for b in range(lanes)] for k in range(n_scan)])
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_batch=lanes)
    try:
        poses = c.scan_stream_batch(ptrs, counts, False)
    finally:
        c.close()
    solo = aloam.Aloam(n_scans=16, max_points=maxn + 1024)
    try:
        for b in range(lanes):
            solo.reset_odometry()
            sp, _ = solo.scan_stream([trajs[b][k].ctypes.data for k in range(n_scan)], counts[:, b], False)
            assert np.array_equal(sp, poses[:, b]), b
    finally:
        solo.close()
