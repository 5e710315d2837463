"""Sweeps cut anywhere, shared by tests/test_oracle_sweep_seams.py (CPU) and tests/test_gpu_sweep_seams.py (GPU).  TEST
INFRASTRUCTURE.

Every scan of synth.scan() starts near azimuth -pi and sweeps one clockwise revolution, column by column, so four of the six
2 pi fix-ups of scanRegistration.cpp:141-153,208-236 never run and relTime never goes below 0.  The grid below cuts the sweep
in every quadrant and on the axes, covers 0.6 to 1.05 revolutions, offsets every beam's firing azimuth by up to +-2 deg,
fires laser-major or column-major and turns either way.  The column counts are odd so that no column sits a quarter or half
turn from the first one (synth.scan_seam refuses returns within 1e-5 rad of an azimuth threshold)."""
import itertools
import math

import numpy as np

CUTS = [math.pi / 4, 3 * math.pi / 4, -3 * math.pi / 4, -math.pi / 4, 0.0, math.pi / 2, -math.pi / 2, math.pi]
COVERAGES = [0.6, 1.0, 1.05]
SEAM_N_AZ = {"VLP-16": 901, "HDL-32": 1101, "HDL-64": 1001}


def ring_offsets(n_scans):
    """a fixed per-beam azimuth offset in [-2, 2] deg, not monotone in the beam"""
    return np.linspace(-2.0, 2.0, n_scans)[np.random.default_rng(n_scans).permutation(n_scans)]


def layouts(n_scans):
    """(coverage, offsets, laser_major, ccw) of one cut"""
    return list(itertools.product(COVERAGES, (None, ring_offsets(n_scans)), (False, True), (False, True)))


def seam_scan(synth, sensor, index, cut, coverage=1.0, offsets=None, laser_major=False, ccw=False, n_az=None):
    return synth.scan_seam(sensor, index, cut, coverage, offsets, laser_major, ccw, n_az=n_az or SEAM_N_AZ[sensor])


# seam trajectories for the chains: cut, offsets and layout fixed along the trajectory, full density.  The HDL-64 one gives
# queries with s = frac(intensity) / 0.1 up to ~9.998 (int(intensity) = ring - 1); the counter-clockwise VLP-16 one gives
# ring-0 returns with relTime < 0, i.e. negative intensities and s < 0.
TRAJECTORIES = {
    "HDL-64": dict(sensor="HDL-64", cut=0.3 - math.pi / 2, coverage=1.0, offsets="ring", laser_major=False, ccw=False),
    "VLP-16": dict(sensor="VLP-16", cut=-2.5, coverage=1.0, offsets="ring", laser_major=False, ccw=False),
    "VLP-16-ccw": dict(sensor="VLP-16", cut=-2.5, coverage=1.0, offsets="ring", laser_major=False, ccw=True),
}


def trajectory_scan(synth, name, index, n_az=None):
    t = TRAJECTORIES[name]
    sensor = t["sensor"]
    off = ring_offsets(synth.SENSORS[sensor][0]) if t["offsets"] == "ring" else None
    n_az = n_az or synth.SENSORS[sensor][1] + 1
    return synth.scan_seam(sensor, index, t["cut"], t["coverage"], off, t["laser_major"], t["ccw"], n_az=n_az)


def ratios(cloud):
    """the DISTORTION build's interpolation ratio of every point: (intensity - int(intensity)) / 0.1, int truncating"""
    return (cloud[:, 3] - cloud[:, 3].astype(np.int32).astype(np.float32)) / 0.1


def with_first(raw, point):
    return np.concatenate([np.asarray(point, np.float32).reshape(1, 4), raw])


def with_last(raw, point):
    return np.concatenate([raw, np.asarray(point, np.float32).reshape(1, 4)])


HAND_BUILT = ["minus_x_axis_y_plus_zero", "minus_x_axis_y_minus_zero", "first_outside_rings", "last_outside_rings",
              "first_nan", "hdl64_first_below_rings"]


def hand_built(synth):
    """(name, sensor, raw): first returns that decide the start azimuth in unusual ways"""
    out = []
    base = seam_scan(synth, "VLP-16", 2, math.pi)
    out.append(("minus_x_axis_y_plus_zero", "VLP-16", with_first(base, [-7.5, 0.0, -1.2, 0.0])))       # startOri = -pi
    out.append(("minus_x_axis_y_minus_zero", "VLP-16", with_first(base, [-7.5, -0.0, -1.2, 0.0])))      # startOri = +pi
    # a return 40 deg above the horizon survives the range filter, sets startOri / endOri, and is dropped by its ring
    out.append(("first_outside_rings", "VLP-16", with_first(base, [2.0, -3.0, 3.0, 0.0])))
    out.append(("last_outside_rings", "VLP-16", with_last(base, [-2.0, -3.0, 3.0, 0.0])))
    out.append(("first_nan", "VLP-16", with_first(base, [np.nan, 1.0, 1.0, 0.0])))
    b64 = seam_scan(synth, "HDL-64", 1, -math.pi / 2)
    out.append(("hdl64_first_below_rings", "HDL-64", with_first(b64, [-4.0, 9.0, -7.0, 0.0])))         # -35 deg: dropped
    return out


def replay(raw, full, minimum_range):
    """numpy replay of scanRegistration.cpp:141-153,208-236 on the returns that reach the azimuth walk (those of `full`):
    the set of fix-ups that fired, and relTime per return (firing order)"""
    p = np.asarray(raw, np.float32)
    finite = np.all(np.isfinite(p[:, :3]), axis=1)
    thres = np.float32(minimum_range)
    keep = finite.copy()
    keep[finite] = (p[finite, 0] * p[finite, 0] + p[finite, 1] * p[finite, 1] + p[finite, 2] * p[finite, 2]) >= thres * thres
    q = p[keep]
    ori_all = -np.arctan2(q[:, 1], q[:, 0]).astype(np.float32)
    start = float(ori_all[0])
    end = float(np.float32(float(ori_all[-1]) + 2 * math.pi))
    fired = set()
    if end - start > 3 * math.pi:
        end = float(np.float32(end - 2 * math.pi)); fired.add("end-=2pi")
    elif end - start < math.pi:
        end = float(np.float32(end + 2 * math.pi)); fired.add("end+=2pi")
    in_full = set(map(bytes, np.ascontiguousarray(full[:, :3], np.float32)))
    walk = np.array([bytes(r) in in_full for r in np.ascontiguousarray(q[:, :3])], bool)
    ori = ori_all[walk].astype(np.float64)
    pre = ori.copy()
    lo, hi = pre < start - math.pi / 2, pre > start + math.pi * 3 / 2
    pre = np.where(lo, ori + 2 * math.pi, np.where(hi, ori - 2 * math.pi, ori)).astype(np.float32).astype(np.float64)
    passed = np.flatnonzero(pre - start > math.pi)
    h = passed[0] if len(passed) else len(pre)            # the return that sets halfPassed is still a pre-half return
    post = (ori + 2 * math.pi).astype(np.float32).astype(np.float64)
    plo, phi = post < end - math.pi * 3 / 2, post > end + math.pi / 2
    post = np.where(plo, post + 2 * math.pi, np.where(phi, post - 2 * math.pi, post)).astype(np.float32).astype(np.float64)
    if np.any(lo[:h + 1]): fired.add("pre+=2pi")
    if np.any(hi[:h + 1]): fired.add("pre-=2pi")
    if np.any(plo[h + 1:]): fired.add("post+=2pi")
    if np.any(phi[h + 1:]): fired.add("post-=2pi")
    o = np.concatenate([pre[:h + 1], post[h + 1:]])
    rel = (o - start) / (end - start)
    return fired, rel


ALL_FIXUPS = {"end-=2pi", "end+=2pi", "pre+=2pi", "pre-=2pi", "post+=2pi", "post-=2pi"}


def descents(cloud):
    """number of places where int(intensity) falls"""
    r = cloud[:, 3].astype(np.int32)
    return int(np.count_nonzero(np.diff(r) < 0))
