"""Seeded synthetic lidar scans (VLP-16 / HDL-32 / HDL-64 shaped, and sensors that report each return's ring) -- ctypes binding
of synth.cc."""
import ctypes as C
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

SENSORS = {  # name -> (n_scans, azimuth steps, minimum_range [launch/*.launch], line_res, plane_res)
    "VLP-16": (16, 1800, 0.3, 0.2, 0.4),
    "HDL-32": (32, 2200, 0.3, 0.2, 0.4),
    "HDL-64": (64, 2000, 5.0, 0.4, 0.8),
}
BASE_SEED = 20240901

# Sensors whose driver reports each return's ring (aloam_config.ring_source = ALOAM_RING_FIELD): name -> (beam elevations [deg]
# in ring order, ring 0 first; azimuth steps).  Apart from the edge tables R1 / R2, none of them is binned right by a Velodyne
# formula of the reference.  Shaped like:
#   OS64  an Ouster OS1-64: uniform +16.6 .. -16.6 deg, ring 0 the highest beam
#   V32C  a Velodyne VLP-32C: the non-uniform table, ring 0 the lowest beam
#   L40   40 uniform beams -25 .. +15 deg (a ring count that is not a power of two), ring 0 the lowest
#   R1, R2  one and two beams, the edges of the ring count
RING_SENSORS = {
    "OS64": (tuple(16.6 - k * 33.2 / 63 for k in range(64)), 1024),
    "V32C": ((-25.0, -15.639, -11.31, -8.843, -7.254, -6.148, -5.333, -4.667, -4.0) + tuple(-4.0 + k / 3.0 for k in range(1, 18)) +
             (2.333, 3.333, 4.667, 7.0, 10.333, 15.0), 1800),
    "L40": (tuple(-25.0 + k * 40.0 / 39 for k in range(40)), 1200),
    "R1": ((-4.0,), 1800),
    "R2": ((-8.0, 2.0), 1800),
}
# Driver-ring sensors of more than 64 beams, for contexts of aloam_create_wide (Aloam(..., wide=True)), in the layout of
# RING_SENSORS.  Shaped like:
#   OS128  an Ouster OS1-128: uniform +22.5 .. -22.5 deg, ring 0 the highest beam
#   V128   a Velodyne VLS-128: non-uniform -25 .. +15 deg, 1.25 deg apart below -5 deg, 10/95 deg apart between -5 and +5,
#          0.625 deg apart above; ring 0 the lowest beam
#   L96    96 uniform beams -25 .. +15 deg (a width that is not a power of two), ring 0 the lowest
#   E65    65 uniform beams +16 .. -16 deg, the narrowest table that needs the wide entry point, ring 0 the highest
WIDE_RING_SENSORS = {
    "OS128": (tuple(22.5 - k * 45.0 / 127 for k in range(128)), 1024),
    "V128": (tuple(-25.0 + k * 1.25 for k in range(16)) + tuple(-5.0 + k * 10.0 / 95 for k in range(96)) +
             tuple(5.625 + k * 0.625 for k in range(16)), 1800),
    "L96": (tuple(-25.0 + k * 40.0 / 95 for k in range(96)), 1024),
    "E65": (tuple(16.0 - k * 0.5 for k in range(65)), 1024),
}
RING_RANGES = (0.3, 0.2, 0.4)   # minimum_range, line_res, plane_res of every RING_SENSORS / WIDE_RING_SENSORS sensor


def build(force=False):
    so = os.path.join(_HERE, "libaloam_synth.so")
    src = os.path.join(_HERE, "synth.cc")
    if force or not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so):
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-shared", "-o", so, src, "-lpthread"])
    return so


def _lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libaloam_synth.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        L.synth_scan.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double,
                                 C.POINTER(C.c_float), C.c_int]
        L.synth_pose.argtypes = [C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.synth_scan_seam.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int,
                                      C.POINTER(C.c_double), C.c_int, C.c_int, C.c_double, C.POINTER(C.c_float), C.c_int]
        L.synth_scan_beams.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int,
                                       C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int,
                                       C.c_int, C.c_double, C.POINTER(C.c_float), C.POINTER(C.c_int), C.c_int]
        L.synth_scan_rings.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_int, C.c_int,
                                       C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int, C.c_int, C.c_double,
                                       C.POINTER(C.c_float), C.c_int]
        _LIB = L
    return _LIB


def scan(sensor, index, seed=BASE_SEED, n_az=None, noise=0.02, max_range=120.0):
    """Raw scan `index` of the trajectory: (n, 4) float32 x,y,z,0 in the sensor frame, firing order."""
    n_scans, az = SENSORS[sensor][0], SENSORS[sensor][1]
    if n_az is not None:
        az = n_az
    out = np.zeros((n_scans * az, 4), np.float32)
    n = _lib().synth_scan(seed, n_scans, az, index, noise, max_range, out.ctypes.data_as(C.POINTER(C.c_float)), out.shape[0])
    if n < 0:
        raise RuntimeError("synth_scan failed: %d" % n)
    return out[:n].copy()


class SeamTooClose(ValueError):
    """a surviving return lies within 1e-5 rad of an azimuth threshold of the reference's sweep walk"""


def scan_seam(sensor, index, cut=None, coverage=1.0, ring_offsets_deg=None, laser_major=False, ccw=False, seed=BASE_SEED,
              n_az=None, noise=0.02, max_range=120.0):
    """Raw scan `index` of the trajectory, cut and fired differently from scan():
    cut               atan2(y, x) [rad] of the first firing column (None: the phase of scan(), pi - 2 pi 0.37 / n_az)
    coverage          revolutions covered, round(coverage * n_az) columns
    ring_offsets_deg  per-beam azimuth offset [deg] (n_scans values): the beam fires at another azimuth, the world stays put
    laser_major       all columns of beam 0, then beam 1, ... instead of column by column
    ccw               atan2(y, x) rises in firing order instead of falling
    With the neutral arguments the result is bit-identical to scan().  Raises SeamTooClose when a surviving return sits
    within 1e-5 rad of an azimuth threshold (host and device atan2f may then take different branches)."""
    n_scans, az, min_range = SENSORS[sensor][:3]
    if n_az is not None:
        az = n_az
    start_col = 0.0 if cut is None else (math.pi - cut) * az / (2 * math.pi) - 0.37
    n_col = int(round(coverage * az))
    off = None
    if ring_offsets_deg is not None:
        off = np.ascontiguousarray(ring_offsets_deg, np.float64)
        assert off.shape == (n_scans,)
    out = np.zeros((n_scans * n_col, 4), np.float32)
    n = _lib().synth_scan_seam(seed, n_scans, az, index, noise, max_range, start_col, n_col,
                               None if off is None else off.ctypes.data_as(C.POINTER(C.c_double)), int(laser_major), int(ccw),
                               min_range, out.ctypes.data_as(C.POINTER(C.c_float)), out.shape[0])
    if n == -3:
        raise SeamTooClose("scan_seam(%s, %d, cut=%r, coverage=%r): a return lies on an azimuth threshold" % (sensor, index, cut, coverage))
    if n < 0:
        raise RuntimeError("synth_scan_seam failed: %d" % n)
    return out[:n].copy()


def nominal_elevations(sensor):
    """the beam elevations [deg] scan() fires: the centres of the reference's ring bins (HDL-64: shifted by -0.04 deg)"""
    n_scans = SENSORS[sensor][0]
    if n_scans == 16:
        return np.array([-15.0 + 2.0 * k for k in range(16)])
    if n_scans == 32:
        return np.array([-92.0 / 3.0 + (k + 0.5) * 4.0 / 3.0 for k in range(32)])
    return np.array([1.96 - k / 3.0 for k in range(32)] + [-8.87 - 0.5 * m for m in range(32)])


def scan_beams(sensor, index, elevations_deg, z_offsets_m=None, cut=None, coverage=1.0, ring_offsets_deg=None,
               laser_major=False, ccw=False, seed=BASE_SEED, n_az=None, noise=0.02, max_range=120.0, return_beams=False):
    """scan_seam() fired by a beam table of its own: laser b at elevation elevations_deg[b] [deg], firing from (0, 0,
    z_offsets_m[b]) [m] in the sensor frame (None: all at the origin).  The number of lasers may differ from the sensor's
    scan-line count; the reference still bins every return by the sensor's ring formula, so lasers off the bin centres or off
    the origin put returns on and across ring edges.  ring_offsets_deg has one value per laser.  With the nominal table
    (nominal_elevations) and zero offsets the result is bit-identical to scan_seam().  return_beams: also the laser of
    every return, (n,) int32.  Raises SeamTooClose like scan_seam()."""
    n_scans, az, min_range = SENSORS[sensor][:3]
    if n_az is not None:
        az = n_az
    el = np.ascontiguousarray(elevations_deg, np.float64)
    nb = el.shape[0]
    dz = None if z_offsets_m is None else np.ascontiguousarray(z_offsets_m, np.float64)
    off = None if ring_offsets_deg is None else np.ascontiguousarray(ring_offsets_deg, np.float64)
    assert el.ndim == 1 and nb > 0 and (dz is None or dz.shape == (nb,)) and (off is None or off.shape == (nb,))
    start_col = 0.0 if cut is None else (math.pi - cut) * az / (2 * math.pi) - 0.37
    n_col = int(round(coverage * az))
    out = np.zeros((nb * n_col, 4), np.float32)
    beams = np.zeros(nb * n_col, np.int32)
    dp = C.POINTER(C.c_double)
    n = _lib().synth_scan_beams(seed, n_scans, az, index, noise, max_range, start_col, n_col, nb, el.ctypes.data_as(dp),
                                None if dz is None else dz.ctypes.data_as(dp), None if off is None else off.ctypes.data_as(dp),
                                int(laser_major), int(ccw), min_range, out.ctypes.data_as(C.POINTER(C.c_float)),
                                beams.ctypes.data_as(C.POINTER(C.c_int)), out.shape[0])
    if n == -3:
        raise SeamTooClose("scan_beams(%s, %d): a return lies on an azimuth threshold" % (sensor, index))
    if n < 0:
        raise RuntimeError("synth_scan_beams failed: %d" % n)
    return (out[:n].copy(), beams[:n].copy()) if return_beams else out[:n].copy()


def scan_rings(sensor, index, reverse=False, cut=None, coverage=1.0, laser_major=False, ccw=False, seed=BASE_SEED, n_az=None,
               noise=0.02, max_range=120.0):
    """Raw scan `index` of the trajectory from RING_SENSORS[sensor] (or WIDE_RING_SENSORS[sensor]), with its driver ring: (n, 4)
    float32 x, y, z, ring.  The
    ring of laser b is b, or n_beams - 1 - b with reverse (the other elevation order).  cut, coverage, laser_major and ccw as
    for scan_seam().  Raises SeamTooClose when a return that survives minimum_range (RING_RANGES) sits within 1e-5 rad of an
    azimuth threshold of the sweep walk: every such return takes part in it."""
    elev, az = RING_SENSORS[sensor] if sensor in RING_SENSORS else WIDE_RING_SENSORS[sensor]
    if n_az is not None:
        az = n_az
    el = np.ascontiguousarray(elev, np.float64)
    nb = el.shape[0]
    rings = np.arange(nb, dtype=np.int32)
    if reverse:
        rings = np.ascontiguousarray(rings[::-1])
    start_col = 0.0 if cut is None else (math.pi - cut) * az / (2 * math.pi) - 0.37
    n_col = int(round(coverage * az))
    out = np.zeros((nb * n_col, 4), np.float32)
    n = _lib().synth_scan_rings(seed, az, index, noise, max_range, start_col, n_col, nb, el.ctypes.data_as(C.POINTER(C.c_double)),
                                rings.ctypes.data_as(C.POINTER(C.c_int)), None, int(laser_major), int(ccw), RING_RANGES[0],
                                out.ctypes.data_as(C.POINTER(C.c_float)), out.shape[0])
    if n == -3:
        raise SeamTooClose("scan_rings(%s, %d): a return lies on an azimuth threshold" % (sensor, index))
    if n < 0:
        raise RuntimeError("synth_scan_rings failed: %d" % n)
    return out[:n].copy()


def pose(index):
    """Ground-truth world pose of scan `index`: (q xyzw, t)."""
    q = np.zeros(4)
    t = np.zeros(3)
    _lib().synth_pose(index, q.ctypes.data_as(C.POINTER(C.c_double)), t.ctypes.data_as(C.POINTER(C.c_double)))
    return q, t


def voxel_downsample(cloud, leaf):
    """Voxel-centroid downsample used to BUILD synthetic maps (numpy; same grid rule as pcl::VoxelGrid, float64 sums --
    it only has to produce a plausible map, the parity-relevant VoxelGrid lives in the oracle / CUDA path)."""
    cloud = np.ascontiguousarray(cloud, np.float32)
    if len(cloud) == 0:
        return cloud.copy()
    ijk = np.floor(cloud[:, :3] / np.float32(leaf)).astype(np.int64)
    ijk -= ijk.min(0)
    dims = ijk.max(0) + 1
    key = ijk[:, 0] + dims[0] * (ijk[:, 1] + dims[1] * ijk[:, 2])
    order = np.argsort(key, kind="stable")
    ks = key[order]
    starts = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]])
    sums = np.add.reduceat(cloud[order].astype(np.float64), starts, axis=0)
    counts = np.diff(np.r_[starts, len(ks)])[:, None]
    return (sums / counts).astype(np.float32)


def rotation_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


MAP_SCANS = list(range(0, 24))        # scans whose features make the base map
MAP_QUERY_SCANS = list(range(24, 40))  # scans registered against it (not part of the map)


def build_map(features, total_points, sensor="HDL-64", seed=BASE_SEED + 3, line_res=0.4, plane_res=0.8):
    """Synthetic voxel map for the scan-to-map configs (SURVEY.md 8d): union of the less-sharp / less-flat features of
    scans MAP_SCANS at their true poses, voxel-filtered at line_res / plane_res, then replicated with 2 cm jitter on a
    lattice of parallel streets (y pitch 30 m, 7 columns) and stacked levels (z pitch 8 m, 18 levels) INSIDE the
    250 x 250 x 150 m volume of the reference's 5 x 5 x 3-cube submap (laserMapping.cpp:512-529) to exactly
    total_points // 5 corner + the rest surf points.  The tile at offset 0 (the one the query scans see) is a clean
    filtered map; if one lattice of tiles is not enough the other tiles are added again with an x shift and fresh jitter.
    `features(raw) -> (less_sharp, less_flat)` is the extraction to use (the product's or the oracle's)."""
    corner, surf = [], []
    for k in MAP_SCANS:
        ls, lf = features(scan(sensor, k))
        qk, tk = pose(k)
        R = rotation_matrix(qk)
        for src, dst in ((ls, corner), (lf, surf)):
            w = src.copy()
            w[:, :3] = (src[:, :3].astype(np.float64) @ R.T + tk).astype(np.float32)
            dst.append(w)
    cbase = voxel_downsample(np.concatenate(corner), line_res)
    sbase = voxel_downsample(np.concatenate(surf), plane_res)
    rng = np.random.default_rng(seed)
    offsets = [(0.0, 0.0, 0.0)]
    for lvl in sorted(range(-9, 9), key=abs):
        for col in sorted(range(-3, 4), key=abs):
            if lvl or col:
                offsets.append((0.0, 30.0 * col, 8.0 * lvl))

    def tile(base, target):
        out, n, rounds = [base], len(base), 0
        while n < target:
            for ox, oy, oz in offsets[1:]:
                c = base.copy()
                c[:, :3] += np.array([ox + 0.37 * rounds, oy, oz], np.float32) + rng.normal(0, 0.02, (len(base), 3)).astype(np.float32)
                out.append(c)
                n += len(c)
                if n >= target:
                    break
            rounds += 1
        return np.ascontiguousarray(np.concatenate(out)[:target])

    return tile(cbase, total_points // 5), tile(sbase, total_points - total_points // 5)
