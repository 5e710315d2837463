"""CPU: sweeps cut anywhere (tests/seam_cases.py) through the reference's own scanRegistration.cpp and laserOdometry.cpp
(oracle/_ref, see tests/test_oracle_vs_reference_source.py) against the oracle, bit for bit.  These are the sweeps that run
the four 2 pi fix-ups the default scans never reach and that give returns relTime < 0, i.e. int(intensity) = ring - 1, so
the published less-sharp / less-flat clouds are no longer ascending in int(intensity)."""
import math
import os

import numpy as np
import pytest

import seam_cases as S
from refsource import RefOdometry, private_copy, ref_registration

SENSORS = ["VLP-16", "HDL-32", "HDL-64"]


def test_neutral_seam_scan_is_synth_scan(synth):
    """scan_seam with neutral arguments is scan(), and scan() itself is unchanged (its golden bytes)"""
    for sensor in SENSORS:
        for k in (0, 3):
            a, b = synth.scan(sensor, k), synth.scan_seam(sensor, k)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (sensor, k)
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "features_vlp16_az360.npz"))
    assert np.array_equal(synth.scan("VLP-16", 0, n_az=360).view(np.uint32), g["raw"].view(np.uint32))


def test_seam_scan_refuses_returns_on_a_threshold(synth):
    """a column count divisible by 4 puts columns exactly a quarter turn from the first one: refused"""
    with pytest.raises(synth.SeamTooClose):
        synth.scan_seam("VLP-16", 0, math.pi / 4, 1.0, None, True, False, n_az=600)


def _same(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("sensor", SENSORS)
@pytest.mark.parametrize("cut", S.CUTS, ids=["q1", "q2", "q3", "q4", "zero", "pi_2", "minus_pi_2", "pi"])
def test_scan_registration_source_equals_oracle_on_seams(orc, synth, sensor, cut):
    """LITERAL and CANONICAL: every output of the reference's laserCloudHandler equals oracle/features.cc, intensities included"""
    ns, _, mr = synth.SENSORS[sensor][:3]
    ref = ref_registration(ns, mr)
    for k, (cov, off, lm, ccw) in enumerate(S.layouts(ns)):
        raw = S.seam_scan(synth, sensor, k % 4, cut, cov, off, lm, ccw)
        for mode in (orc.SORT_LITERAL, orc.SORT_CANONICAL):
            got = ref.run(raw, mode)
            want = orc.Features(raw, ns, mr, mode=mode)
            for name in ("full", "sharp", "less_sharp", "flat", "less_flat"):
                assert _same(got[name], getattr(want, name)), (sensor, cut, cov, off is not None, lm, ccw, mode, name)
            if mode == orc.SORT_LITERAL:
                n = want.full.shape[0]
                core = slice(5, n - 5)
                assert np.array_equal(got["curvature"][core].view(np.uint32), want.curvature[core].view(np.uint32))
                assert np.array_equal(got["label"][core], want.label[core])


def test_the_grid_runs_every_fixup_and_breaks_ring_order(orc, synth):
    """a replay of the azimuth walk fires all six 2 pi adjustments somewhere in the grid; the grid produces returns with
    int(intensity) = ring - 1 and less-sharp / less-flat clouds that descend in int(intensity); relTime stays in (-2, 6], so
    int(intensity) is always the ring or the one below it"""
    fired, below, desc_ls, desc_lf = set(), 0, 0, 0
    rel_lo, rel_hi = 0.0, 1.0
    for sensor in SENSORS:
        ns, _, mr = synth.SENSORS[sensor][:3]
        for cut in S.CUTS:
            for k, (cov, off, lm, ccw) in enumerate(S.layouts(ns)):
                if k % 3:
                    continue            # a third of each cut's layouts keeps this test short; every layout value still occurs
                raw = S.seam_scan(synth, sensor, 0, cut, cov, off, lm, ccw)
                f = orc.Features(raw, ns, mr)
                ev, rel = S.replay(raw, f.full, mr)
                fired |= ev
                # one +-2 pi fix-up keeps pre-half returns in [-0.5, 1.5]; post-half ones can stay outside the window, within (-2, 6]
                assert rel.min() > -2 and rel.max() <= 6, (sensor, cut, cov, lm, ccw, rel.min(), rel.max())
                rel_lo, rel_hi = min(rel_lo, rel.min()), max(rel_hi, rel.max())
                # physical ring of every point of the ring-major cloud: ring r spans [scanStart - 5, scanEnd + 6) (:247-252)
                ring = np.repeat(np.arange(ns), np.asarray(f.scan_end) - np.asarray(f.scan_start) + 11)
                fi = f.full[:, 3].astype(np.int32)
                assert ring.shape == fi.shape and np.all((fi == ring) | (fi == ring - 1))
                below += int(np.count_nonzero(fi < ring))
                desc_ls += S.descents(f.less_sharp)
                desc_lf += S.descents(f.less_flat)
                # int(intensity) is the ring or the one below it, and never falls two below an earlier point
                for c in (f.full, f.less_sharp, f.less_flat):
                    r = c[:, 3].astype(np.int32)
                    assert np.all(r >= np.maximum.accumulate(r) - 1)
    assert fired == S.ALL_FIXUPS, sorted(S.ALL_FIXUPS - fired)
    assert below > 0 and desc_ls > 0 and desc_lf > 0, (below, desc_ls, desc_lf)
    assert rel_lo < -0.2 and rel_hi > 1.5, (rel_lo, rel_hi)   # both ends of the range are reached


@pytest.mark.parametrize("name", S.HAND_BUILT)
def test_hand_built_first_returns(orc, synth, name):
    """a first return on the -x axis with y = +0.0 / -0.0 (startOri = -pi / +pi), a first or last return that sets the
    azimuth and is then dropped by its ring angle, a NaN first return: reference == oracle, both modes"""
    _, sensor, raw = next(c for c in S.hand_built(synth) if c[0] == name)
    ns, _, mr = synth.SENSORS[sensor][:3]
    ref = ref_registration(ns, mr)
    for mode in (orc.SORT_LITERAL, orc.SORT_CANONICAL):
        got = ref.run(raw, mode)
        want = orc.Features(raw, ns, mr, mode=mode)
        for part in ("full", "sharp", "less_sharp", "flat", "less_flat"):
            assert _same(got[part], getattr(want, part)), (name, mode, part)
    f = orc.Features(raw, ns, mr)
    if name.startswith("minus_x"):
        assert raw[0, 0] < 0 and raw[0, 1] == 0 and (np.signbit(raw[0, 1]) == name.endswith("minus_zero"))
    if "outside" in name or "below" in name:
        assert not np.any(np.all(f.full[:, :3] == raw[0 if "first" in name else -1, :3], axis=1))   # dropped


@pytest.mark.parametrize("name", list(S.TRAJECTORIES))
def test_laser_odometry_source_equals_oracle_on_seam_trajectories(orc, synth, name):
    """5 scans of a seam trajectory (tests/seam_cases.py TRAJECTORIES): the reference's laserOdometry.cpp gives the oracle's
    q, t, world pose and correspondence counts bit for bit, on last clouds that descend in int(intensity)"""
    sensor = S.TRAJECTORIES[name]["sensor"]
    ns, _, mr = synth.SENSORS[sensor][:3]
    ref = RefOdometry(private_copy("libref_odometry.so", "seam_%s" % name))
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    desc = 0
    for k in range(5):
        f = orc.Features(S.trajectory_scan(synth, name, k), ns, mr, mode=orc.SORT_LITERAL)
        got = ref.process(f, stamp=0.1 * (k + 1))
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
            assert got["counts"].tolist() == [info["corner_corr"], info["plane_corr"]], (k, got["counts"], info)
        od.set_last(f.less_sharp, f.less_flat)
        desc += S.descents(f.less_sharp) + S.descents(f.less_flat)
        assert np.array_equal(got["q"], q) and np.array_equal(got["t"], t), (k, got["q"] - q, got["t"] - t)
        assert np.array_equal(got["qw"], qw) and np.array_equal(got["tw"], tw), k
    assert desc > 0
    assert float(np.abs(tw).max()) > 1.0   # the trajectory moves


@pytest.mark.parametrize("s", [-0.05, -1e-7, 1.5, 9.998])
def test_functors_at_seam_ratios(orc, s):
    """the reference's functors (lidarFactor.hpp) equal the oracle's closed form and autodiff at the ratios a seam sweep gives
    the DISTORTION build: s < 0 on ring 0, s up to ~10 where int(intensity) = ring - 1"""
    import test_oracle_vs_reference_source as T
    from refsource import ref_lib
    import ctypes as C
    lib = ref_lib("libref_factor.so")
    dp = C.POINTER(C.c_double)
    lib.ref_factor_eval.argtypes = [C.c_int, dp, C.c_double, dp, dp, dp, dp, dp]
    lib.ref_factor_eval.restype = C.c_int
    rng = np.random.default_rng(int(abs(s) * 1e4) + 7)
    for trial in range(6):
        q = np.array([0.01, -0.02, 0.015, 1.0]) * rng.uniform(0.5, 1.5, 4) if trial % 2 == 0 else rng.normal(size=4)
        q /= np.linalg.norm(q)
        t = rng.normal(size=3)
        x = np.concatenate([q, t]); P = T.plus_jacobian(q)
        cp, a, b, c = (rng.normal(size=3) * 10 for _ in range(4))
        for kind, pts, block in [(0, [cp, a, b], orc.make_edge(cp, a, b, s)), (1, [cp, a, b, c], orc.make_plane(cp, a, b, c, s))]:
            pts = np.ascontiguousarray(pts, np.float64).reshape(-1)
            r = np.zeros(3); jq = np.zeros(12); jt = np.zeros(9)
            f = lambda v: v.ctypes.data_as(dp)
            rows = lib.ref_factor_eval(kind, f(pts), float(s), f(q), f(t), f(r), f(jq), f(jt))
            j_ref = np.concatenate([jq[:rows * 4].reshape(rows, 4) @ P, jt[:rows * 3].reshape(rows, 3)], axis=1)
            for autodiff in (True, False):
                r_o, j_o, _ = orc.evaluate([block], x, huber=1e12, autodiff=autodiff)
                assert np.allclose(r_o, r[:rows], rtol=1e-12, atol=1e-12), (kind, s, autodiff)
                assert np.allclose(np.asarray(j_o).reshape(j_ref.shape), j_ref, rtol=1e-9, atol=1e-9), (kind, s, autodiff)
