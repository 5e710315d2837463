"""GPU: the CUDA path against THE REFERENCE'S OWN SOURCE FILES in execution -- oracle/_ref holds scanRegistration.cpp and
laserOdometry.cpp compiled unmodified (in the build container, where /root/reference exists) against the stand-in headers of
oracle/ref_shim; the libraries travel with the snapshot, nothing here reads /root/reference.  The other GPU tests compare with
the oracle restatement, and tests/test_oracle_vs_reference_source.py (CPU) shows the restatement bit-identical to these libraries;
this file closes the triangle directly.  Skips where the libraries are not present."""
import types

import numpy as np
import pytest

from conftest import rot_angle

pytestmark = pytest.mark.gpu


def _load(fn, *a):
    try:
        return fn(*a)
    except (OSError, AssertionError) as e:      # not built / not loadable on this machine
        pytest.skip("oracle/_ref is not usable here: %r" % (e,))


@pytest.mark.parametrize("sensor", ["VLP-16", "HDL-32", "HDL-64"])
@pytest.mark.parametrize("index", [0, 3])
def test_features_match_the_reference_source(sensor, index, aloam, orc, synth, scans):
    """aloam_extract_features vs the clouds the reference's laserCloudHandler publishes: coordinates bit-exact, ring ids equal,
    relTime fraction within the atan2f rounding of the two libm's (as against the oracle, tests/test_gpu_features.py)"""
    import refsource
    ns, _, mr = synth.SENSORS[sensor][:3]
    raw = scans(sensor, index)
    ref = _load(refsource.ref_registration, ns, mr).run(raw, orc.SORT_CANONICAL)
    c = aloam.Aloam(n_scans=ns, max_points=200000)
    got = c.extract_features(raw)
    c.close()
    for name in ["full", "sharp", "less_sharp", "flat", "less_flat"]:
        g, r_ = got[name], ref[name]
        assert g.shape == r_.shape, name
        assert np.array_equal(g[:, :3], r_[:, :3]), name
        assert np.array_equal(g[:, 3].astype(np.int32), r_[:, 3].astype(np.int32)), name
        assert np.abs(g[:, 3] - r_[:, 3]).max() <= 1e-5, name


def test_odometry_poses_match_the_reference_source_chain(aloam, orc, synth, scans):
    """aloam_scan_to_pose per scan vs the reference's scanRegistration -> laserOdometry chain (its own source for feature
    extraction, TransformToStart, correspondence search, block construction and pose integration): both correspondence counts
    equal, the world pose within the bar of tests/test_gpu_vs_reference_chains.py.  The reference's VoxelGrid runs with the
    device's tie order (index order; std::sort leaves equal voxel indices unordered), so the difference left is the device's"""
    import refsource
    from test_gpu_vs_reference_chains import ODOM_BAR
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    reg = _load(refsource.ref_registration, ns, mr)
    odo = refsource.RefOdometry(_load(refsource.private_copy, "libref_odometry.so", "gpu_chain"))
    c = aloam.Aloam(n_scans=ns, max_points=40000)
    moved = worst = 0.0
    for k in range(5):
        raw = scans("VLP-16", k, n_az=900)
        r = reg.run(raw, orc.SORT_CANONICAL)
        st = odo.process(types.SimpleNamespace(**{n: r[n] for n in ("sharp", "less_sharp", "flat", "less_flat", "full")}), stamp=0.1 * (k + 1))
        gq, gt, gst = c.scan_to_pose(raw)
        worst = max(worst, float(np.abs(gt - st["tw"]).max()), rot_angle(gq, st["qw"]))
        assert np.abs(gt - st["tw"]).max() <= ODOM_BAR and rot_angle(gq, st["qw"]) <= ODOM_BAR, (k, gt - st["tw"])
        if k > 0:
            assert [gst["n_corner_corr"], gst["n_plane_corr"]] == st["counts"].tolist(), (k, gst, st["counts"])
        moved = max(moved, float(np.abs(st["tw"]).max()))
    c.close()
    print("measured VLP-16 chain vs the reference source: %.3g" % worst)
    assert moved > 0.05
