"""CPU: the association settings of aloam_config away from their defaults.

* The oracle's association run with DISTANCE_SQ_THRESHOLD / NEARBY_SCAN as parameters equals a plain numpy transcription of
  laserOdometry.cpp:299-483 on hand-built "last" clouds, for every value the GPU tests use (tests/config_cases.py).
* aloam_create refuses the settings the reference cannot mean, before it looks for a device.
* A host model of the ring-window loop of k_odom_assoc: without a bound it runs ~N iterations per query (and overflows for
  N = 1e300 or inf); with the bound of 64 it ends, and the window it gives equals the reference's break tests on every ring."""
import math

import numpy as np
import pytest

import config_cases as K

IDENT_Q, ZERO_T = np.array([0, 0, 0, 1.0]), np.zeros(3)


def _oracle_rows(orc, last, queries, thr, nearby, distortion=False):
    od = orc.Odometry(distortion=distortion, dist_sq_thresh=thr, nearby_scan=nearby)
    od.set_last(last, last)
    cc, pc, _ = od.associate(queries, queries, IDENT_Q, ZERO_T)
    return [(int(a), int(b), int(c), -1) for a, b, c in cc], [tuple(int(v) for v in r) for r in pc]


@pytest.mark.parametrize("nearby", K.NEARBY, ids=K.NEARBY_IDS)
@pytest.mark.parametrize("distortion", [False, True])
def test_oracle_window_equals_the_literal_loops(orc, nearby, distortion):
    last, queries = K.window_scene()
    cc, pc = _oracle_rows(orc, last, queries, 25.0, nearby, distortion)
    assert cc == K.associate(last, queries, 25.0, nearby, True)
    assert pc == K.associate(last, queries, 25.0, nearby, False)
    assert len(cc) == len(queries) and len(pc) == len(queries)
    ring = last[:, 3].astype(np.int32)
    for (i, j, m2, _), (_, _, _, m3) in zip(cc, pc):
        # the scene makes the 2nd / 3rd point the outermost in-window ring on the near side (or the far side at rings 0 / 63)
        rc = int(ring[j])
        dn, up = K.window(rc, nearby)
        edge = (min(rc + up, 63), max(rc - dn, 0))
        assert int(ring[m2]) in edge and int(ring[m3]) in edge, (i, rc, ring[m2], ring[m3])


@pytest.mark.parametrize("thr", K.THRESH[:-1], ids=K.THRESH_IDS[:-1])
def test_oracle_threshold_equals_the_literal_loops(orc, thr):
    last, queries = K.threshold_scene(thr)
    cc, pc = _oracle_rows(orc, last, queries, thr, 2.5)
    want_c, want_p = K.associate(last, queries, thr, 2.5, True), K.associate(last, queries, thr, 2.5, False)
    assert cc == want_c and pc == want_p
    # every planted distance is reached: float(thr) is accepted exactly when it lies below thr in double
    f = np.float32(thr)
    accepted = {float(K.sqd(last[r[2]], queries[r[0]])) for r in want_c}
    assert (float(f) in accepted) == (float(f) < thr)
    assert float(np.nextafter(f, np.float32(0))) in accepted and float(np.nextafter(f, np.float32(np.inf))) not in accepted


def test_threshold_scene_reaches_the_rounding_cases():
    """the three thresholds whose float rounds below them: the kernel's former limit (float)thr rejects a d2 of exactly that
    float, which the reference's double comparison accepts"""
    below = [t for t in K.THRESH[:-1] if float(np.float32(t)) < t]
    assert below == [4.0 + 2.0 ** -23, 0.7, 25.3]
    assert float(np.float32(0.1)) > 0.1 and float(np.float32(25.0)) == 25.0


def test_oracle_defaults_are_the_reference_constants(orc, synth):
    """Odometry() and Odometry(dist_sq_thresh=25, nearby_scan=2.5) give the same association on a real scan pair"""
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    f0, f1 = (orc.Features(synth.scan("VLP-16", k, n_az=900), ns, mr) for k in (0, 1))
    q = np.array([0.001, -0.002, 0.008, 1.0]); q /= np.linalg.norm(q)
    out = []
    for od in (orc.Odometry(), orc.Odometry(dist_sq_thresh=25.0, nearby_scan=2.5)):
        od.set_last(f0.less_sharp, f0.less_flat)
        out.append(od.associate(f1.sharp, f1.flat, q, [0.5, 0.0, 0.0]))
    for a, b in zip(*out):
        assert np.array_equal(a, b)
    assert len(out[0][0]) > 50


@pytest.mark.parametrize("field,values", [("huber", [0.0, -1.0, math.nan]), ("line_res", [0.0, math.nan]), ("plane_res", [0.0, math.nan]),
                                          ("nearby_scan", [0.5, math.nan])])
def test_create_refuses_meaningless_settings_before_the_device(aloam, field, values):
    for v in values:
        with pytest.raises(aloam.AloamError) as e:
            aloam.Aloam(n_scans=16, **{field: v})
        assert e.value.code == -1, (field, v, e.value.code)


def _unbounded_iterations(rc, nearby):
    """iterations of the former loop `while ((double)(rc + up + 1) <= (double)rc + N) ++up;`, counted in closed form; None when
    rc + up + 1 would pass INT_MAX first (signed overflow: the loop never ends in a defined way)"""
    lim = rc + nearby
    if lim >= 2 ** 31:
        return None
    return max(0, math.floor(lim) - rc)


@pytest.mark.parametrize("nearby", K.NEARBY, ids=K.NEARBY_IDS)
def test_ring_window_loop_is_bounded_and_equals_the_break_tests(nearby):
    for rc in range(64):
        dn, up = K.window(rc, nearby)
        assert 1 <= up <= 64 and 1 <= dn <= 64
        for r in range(64):
            kept = not (r > rc + nearby) and not (r < rc - nearby)      # laserOdometry.cpp:319,345,405,433
            assert kept == (rc - dn <= r <= rc + up), (rc, r, dn, up)
    if nearby >= 1e300:
        assert _unbounded_iterations(0, nearby) is None       # the unbounded loop ran into a signed overflow
    assert _unbounded_iterations(5, 1e6) == 1_000_000        # and a million iterations per query at 1e6


def test_ring_window_is_not_symmetric_at_3_minus_2_to_the_48():
    """rc + N and rc - N round differently: the backward side cannot be derived from the forward one"""
    n = 3.0 - 2.0 ** -48
    asym = [rc for rc in range(64) if K.window(rc, n)[0] != K.window(rc, n)[1]]
    assert asym == [30, 31, 32, 33, 34], asym
    assert K.window(32, n) == (2, 3)
