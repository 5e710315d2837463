"""CPU: the short dense rings of tests/short_ring_cases.py.  The reference's own scanRegistration.cpp gives the oracle's features on
them, so the oracle's one picked array per ring is the reference's behaviour; every scene the GPU tests run is what it claims
to be (ring sizes, dense arcs), the sequential sweep reproduces the oracle's labels on every ring, and passing on only a
segment's own marks does not -- each scene fails on a kernel that drops the marks running past a short segment."""
import numpy as np
import pytest

import edge_scenes as es
import short_ring_cases as SC
from refsource import ref_registration

NAMES = ("full", "sharp", "less_sharp", "flat", "less_flat")


@pytest.mark.parametrize("ns", [16, 32, 64])
@pytest.mark.parametrize("style", es.DENSE_STYLES)
def test_reference_source_equals_the_oracle_on_short_dense_rings(orc, ns, style):
    """elevation-mode scans whose short rings lie on dense arcs: the reference's laserCloudHandler (its own source, one
    cloudNeighborPicked array for the whole scan) equals oracle/features.cc bit for bit, in CANONICAL mode (what the device
    follows) and LITERAL mode (the reference's std::sort order), including the label and neighbour-picked arrays"""
    raw = SC.elevation_scan(ns, style)
    ref = ref_registration(ns, SC.MIN_RANGE[ns])
    for mode in (orc.SORT_CANONICAL, orc.SORT_LITERAL):
        got = ref.run(raw, mode)
        want = orc.Features(raw, ns, SC.MIN_RANGE[ns], mode)
        for n in NAMES:
            a, b = got[n], getattr(want, n)
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (mode, n)
        core = slice(5, want.full.shape[0] - 5)
        assert np.array_equal(got["curvature"][core].view(np.uint32), want.curvature[core].view(np.uint32)), mode
        assert np.array_equal(got["label"][core], want.label[core]) and np.array_equal(got["picked"][core], want.picked[core]), mode
    assert SC.adjacent_misses(want, ns)


def _check_scene(raw, ns, mode, counts):
    ref = SC.oracle(raw, ns, mode)
    assert list(np.bincount(ref.full[:, 3].astype(np.int64), minlength=ns)) == list(counts)
    short = [r for r, n in enumerate(counts) if 17 <= n < 64]
    assert SC.dense_rings(ref, ns) == short                       # every short ring is dense: its picks reach 5 positions
    for r in short:                                              # consecutive returns under 0.22 m apart
        a, n = SC.ring_inputs(ref, r)[:2]
        d = np.diff(ref.full[a:a + n, :3].astype(np.float64), axis=0)
        assert np.sqrt((d * d).sum(1)).max() < 0.22, r
    miss = SC.adjacent_misses(ref, ns)
    assert miss and all(counts[r] < 40 for r in miss)
    return ref, miss


@pytest.mark.parametrize("style", es.DENSE_STYLES)
def test_field_scenes_every_ring_size(style):
    """40 driver rings: one ring of each size 16..48 and seven whole turns"""
    ref, miss = _check_scene(SC.field_scan(style), 40, "field", SC.FIELD_RINGS)
    assert len(ref.sharp) and len(ref.flat)
    if style == "dyadic":   # ties at both ends of the curvature order
        c = np.concatenate([SC.ring_inputs(ref, r)[2] for r, n in enumerate(SC.FIELD_RINGS) if 17 <= n < 64])
        assert (c == np.float32(0.5625)).sum() > 100 and (c == 0).sum() > 100 + 11 * 32


@pytest.mark.parametrize("ns", [16, 32, 64])
@pytest.mark.parametrize("style", es.DENSE_STYLES)
def test_elevation_scenes(ns, style):
    _check_scene(SC.elevation_scan(ns, style), ns, "elevation", SC.ELEVATION[ns][0])


def test_wide_scene():
    _check_scene(SC.wide_scan(), 128, "wide", SC.wide_counts())


@pytest.mark.parametrize("traj", range(len(SC.TRAJECTORIES)))
def test_trajectory_frames(traj):
    """every frame of the odometry and batch trajectories; the short rings carry sharp picks"""
    for k in range(SC.FRAMES):
        ref, _ = _check_scene(SC.trajectory_scan(traj, k), 40, "field", SC.FIELD_RINGS)
        assert (ref.sharp[:, 3].astype(np.int64) < len(SC.SIZES)).sum() >= 20, k
