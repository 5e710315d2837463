"""GPU: a context is created, driven through every buffer group it allocates on first use, and destroyed, several times
over; every call succeeds and the results do not depend on the contexts that came before."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _one_context(aloam, raws):
    """extraction, scan stream, map upload + scan-to-map registration, voxel filter, mapper step, mapped scan stream"""
    maxn = max(r.shape[0] for r in raws)
    c = aloam.Aloam(n_scans=16, max_points=maxn + 1024, max_map_points=400000)
    ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
    f0 = c.extract_features(raws[0])
    f1 = c.extract_features(raws[1])
    poses, _ = c.scan_stream(ptrs, counts, False)
    c.map_upload(f0["less_sharp"], f0["less_flat"])
    x, _ = c.mapping_register(c.voxel_filter(f1["less_sharp"], 0.2), c.voxel_filter(f1["less_flat"], 0.4), poses[1])
    q, t, _ = c.mapper_step(f1["less_sharp"], f1["less_flat"], poses[1][:4], poses[1][4:])
    c.reset_odometry()
    odom, mapped = c.scan_stream_mapped(ptrs, counts, False)
    c.close()
    return [f0[k] for k in ("full", "sharp", "less_sharp", "flat", "less_flat")] + [f1["less_flat"], poses, x, q, t, odom, mapped]


def test_three_contexts_in_a_row_give_identical_results(aloam, scans):
    raws = [scans("VLP-16", k, n_az=900) for k in range(4)]
    rounds = [_one_context(aloam, raws) for _ in range(3)]
    for later in rounds[1:]:
        for a, b in zip(rounds[0], later):
            assert a.shape == b.shape and a.tobytes() == b.tobytes()
