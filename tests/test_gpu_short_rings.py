"""GPU: short dense rings through k_ring_features (paired, single trajectory) and k_ring_features_batch, bit for bit against the
oracle (SORT_CANONICAL).  On a ring of 17..39 returns a segment is shorter than a pick's 5-position reach, and the reference's one
picked array lets the marks run past it into the segments after the next one.  The scenes (tests/short_ring_cases.py) are
shown on the CPU to fail on a kernel that passes on only a segment's own marks (test_oracle_short_rings.py)."""
import numpy as np
import pytest

import edge_scenes as es
import short_ring_cases as SC
from test_gpu_ring_field import assert_matches_oracle
from test_gpu_wide_rings import _close

pytestmark = pytest.mark.gpu


def _ctx(aloam, ns, max_points, **kw):
    mr, lr, pr = 0.3, 0.2, 0.4   # synth.RING_RANGES
    return aloam.Aloam(n_scans=ns, max_points=max_points, ring_source=aloam.RING_FIELD, minimum_range=mr, line_res=lr, plane_res=pr, **kw)


def _features(c, raw):
    got = c.extract_features(raw)
    curv, label, s, e = c.debug_features(len(got["full"]))
    return got, curv, label, s, e


@pytest.mark.parametrize("style", es.DENSE_STYLES)
def test_every_ring_size_16_to_48(aloam, style):
    """one ring of every size 16 (skipped) .. 48 and seven whole turns, 40 driver rings: full cloud, scanStart / End, curvature,
    labels per ring and the four feature clouds equal the oracle"""
    raw = SC.field_scan(style)
    want = SC.oracle(raw, 40, "field")
    assert SC.adjacent_misses(want, 40)
    c = _ctx(aloam, 40, len(raw) + 1024)
    got, curv, label, s, e = _features(c, raw)
    c.close()
    assert_matches_oracle(got, curv, label, s, e, want, 40)
    assert e[0] - s[0] == 5 and all(e[r] - s[r] == n - 11 for r, n in enumerate(SC.FIELD_RINGS))


def test_wide_context_of_mostly_short_rings(aloam):
    """aloam_create_wide, 128 driver rings: 8 whole turns and 120 short dense rings of 17..48 returns in all three styles"""
    raw = SC.wide_scan()
    want = SC.oracle(raw, 128, "wide")
    assert SC.adjacent_misses(want, 128)
    c = _ctx(aloam, 128, len(raw) + 1024, wide=True)
    got, curv, label, s, e = _features(c, raw)
    c.close()
    assert_matches_oracle(got, curv, label, s, e, want, 128)


@pytest.mark.parametrize("ns", [16, 32, 64])
@pytest.mark.parametrize("style", es.DENSE_STYLES)
def test_elevation_mode(aloam, ns, style):
    """elevation-mode rings (the formula of n_scans) among whole turns of the room: the oracle, which the reference's own
    scanRegistration.cpp equals on these scans"""
    raw = SC.elevation_scan(ns, style)
    want = SC.oracle(raw, ns, "elevation")
    assert SC.adjacent_misses(want, ns)
    c = aloam.Aloam(n_scans=ns, max_points=len(raw) + 1024, minimum_range=SC.MIN_RANGE[ns])
    got, curv, label, s, e = _features(c, raw)
    c.close()
    assert_matches_oracle(got, curv, label, s, e, want, ns)


def _oracle_chain(orc, traj):
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    poses, counts = [], []
    for k in range(SC.FRAMES):
        f = SC.oracle(SC.trajectory_scan(traj, k), 40, "field")
        assert SC.adjacent_misses(f, 40), k
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
            counts.append((info["corner_corr"], info["plane_corr"]))
        else:
            counts.append(None)
        od.set_last(f.less_sharp, f.less_flat)
        poses.append(np.concatenate([qw, tw]))
    return np.array(poses), counts


def test_odometry_chain_on_short_rings(aloam, orc):
    """five frames whose short zigzag rings carry sharp picks: poses at the bars of test_gpu_wide_rings and the oracle's
    correspondence counts, then the same through scan_stream"""
    import torch
    want, counts = _oracle_chain(orc, 0)
    assert np.abs(want[-1, 4:]).max() > 0.1
    raws = [SC.trajectory_scan(0, k) for k in range(SC.FRAMES)]
    c = _ctx(aloam, 40, max(len(r) for r in raws) + 1024)
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
    c.close()
    assert np.array_equal(p, got)


def test_batch_on_short_rings_equals_solo_and_the_oracle(aloam, orc):
    """aloam_scan_stream_batch (the 256-thread ring kernel) with the smooth and the dyadic trajectories as its two lanes: poses
    bit-identical to each trajectory's solo scan_stream (the paired kernel), which follows the oracle chain"""
    import torch
    trajs = [[SC.trajectory_scan(b, k) for k in range(SC.FRAMES)] for b in (1, 2)]
    maxn = max(len(s) for tr in trajs for s in tr)
    dev = [[torch.from_numpy(s).cuda() for s in tr] for tr in trajs]
    ptrs = np.array([[dev[b][k].data_ptr() for b in range(2)] for k in range(SC.FRAMES)], np.uint64)
    counts = np.array([[len(trajs[b][k]) for b in range(2)] for k in range(SC.FRAMES)])
    c = _ctx(aloam, 40, maxn + 1024, max_batch=2)
    poses = c.scan_stream_batch(ptrs, counts, True)
    c.close()
    solo = _ctx(aloam, 40, maxn + 1024)
    for b in range(2):
        solo.reset_odometry()
        sp, _ = solo.scan_stream([dev[b][k].data_ptr() for k in range(SC.FRAMES)], counts[:, b], True)
        assert np.array_equal(sp, poses[:, b]), b
        want, _ = _oracle_chain(orc, b + 1)
        _close(poses[:, b], want)
    solo.close()
