"""The oracle's feature extraction with driver rings up to 128 (contexts of aloam_create_wide).  TEST INFRASTRUCTURE.

Nothing in the reference past ring binning limits the ring count: laserOdometry.cpp reads int(intensity) only, and
scanRegistration.cpp sizes its per-ring vectors by N_SCANS.  So the wide oracle is the field-mode oracle of
ring_field_oracle.field_source() -- oracle/features.cc with the driver's ring -- with one more edit: its n_scans bound becomes
128.  It is compiled with the other oracle sources into its own private library, once per session, in a temporary directory."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import pyoracle as orc
import ring_field_oracle as RF

_LIB = None
MAX_RINGS = 128

EDIT = ("if (n_scans < 1 || n_scans > 64 || stride < 4) return -1;",
        "if (n_scans < 1 || n_scans > 128 || stride < 4) return -1;")


def wide_source():
    src = RF.field_source()
    if src.count(EDIT[0]) != 1:
        raise RuntimeError("the field-mode oracle no longer holds %r exactly once" % EDIT[0])
    return src.replace(EDIT[0], EDIT[1])


def _lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="wide_ring_")
        src = os.path.join(d, "features_wide.cc")
        with open(src, "w") as f:
            f.write(wide_source())
        others = [os.path.join(RF.ORACLE, s) for s in ("voxelgrid.cc", "kdtree.cc", "lm.cc", "odometry.cc", "mapping.cc", "cubemap.cc", "capi.cc")]
        so = os.path.join(d, "liboracle_wide.so")
        # the flags of oracle/Makefile (liboracle.so)
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-shared", "-I" + RF.ORACLE, "-o", so, src] + others)
        L = C.CDLL(so)
        f32p, f64p, i32p = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int)
        L.orc_features_extract.restype = C.c_void_p
        L.orc_features_extract.argtypes = [f32p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, i32p]
        L.orc_features_size.argtypes = [C.c_void_p, C.c_int]
        L.orc_features_copy.argtypes = [C.c_void_p, C.c_int, f32p]
        L.orc_features_ints.argtypes = [C.c_void_p, C.c_int, i32p]
        L.orc_features_curvature.argtypes = [C.c_void_p, f32p]
        L.orc_features_times.argtypes = [C.c_void_p, f64p]
        L.orc_features_free.argtypes = [C.c_void_p]
        _LIB = L
    return _LIB


def Features(raw, n_scans, min_range, mode=orc.SORT_CANONICAL):
    """ring_field_oracle.Features for n_scans 1..128: raw is (n, 4 | 8) float32 with the ring in column 3"""
    raw = np.ascontiguousarray(raw, np.float32)
    if raw.ndim != 2 or raw.shape[1] < 4:
        raise ValueError("a field-mode raw scan has the ring in float 3")
    lib = _lib()
    saved = orc._LIB
    orc._LIB = lib   # pyoracle.Features reads its results through pyoracle.lib(); the wide library has the same entry points
    try:
        return orc.Features(raw, n_scans, min_range, mode)
    finally:
        orc._LIB = saved


def n_rings(synth, sensor):
    return len(synth.WIDE_RING_SENSORS[sensor][0]) if sensor in synth.WIDE_RING_SENSORS else len(synth.RING_SENSORS[sensor][0])


def scan(synth, sensor, index, **kw):
    """synth.scan_rings(sensor, index, **kw): the whole scan, the highest beams' short rings included"""
    return synth.scan_rings(sensor, index, **kw)


def odometry_chain(orc_mod, synth, sensor, frames, reverse=False, distortion=False, nearby_scan=2.5, n_az=None):
    """world poses (frames x 7) and per-frame (corner, plane) correspondence counts of the oracle's odometry over the wide
    oracle's features of scans 0 .. frames-1"""
    ns = n_rings(synth, sensor)
    od = orc_mod.Odometry(distortion=distortion, nearby_scan=nearby_scan)
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    poses, counts = [], []
    for k in range(frames):
        f = Features(scan(synth, sensor, k, reverse=reverse, n_az=n_az), ns, synth.RING_RANGES[0])
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc_mod.integrate_pose(qw, tw, q, t)
            counts.append((info["corner_corr"], info["plane_corr"]))
        else:
            counts.append(None)
        od.set_last(f.less_sharp, f.less_flat)
        poses.append(np.concatenate([qw, tw]))
    return np.array(poses), counts


def recovery_model(aloam, synth, offset, frames=6, start=2):
    """tests/recovery_cases.recover_track on whole OS128 scans: the oracle maps scans 0 .. frames-1 (its store is the device's with
    cube growth on), freezes the store, and runs a localising lane armed at the map pose of scan `start` moved by `offset` (x, y)
    with recovery over RV.deltas.  Returns (map poses (frames, 7), the lane's rows)."""
    import pyfrozen
    import pyoracle
    import recovery_cases as RV
    import reloc_cases as RC
    feats = [Features(scan(synth, "OS128", k), 128, synth.RING_RANGES[0]) for k in range(frames)]
    od, cm = pyoracle.Odometry(), pyoracle.CubeMap()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    poses = []
    for k, f in enumerate(feats):
        if k > 0:
            q, t, _ = od.register(f.sharp, f.flat, q, t)
            qw, tw = pyoracle.integrate_pose(qw, tw, q, t)
        od.set_last(f.less_sharp, f.less_flat)
        poses.append(cm.step(f.less_sharp, f.less_flat, qw, tw, *synth.RING_RANGES[1:])[0])
    cubes = {}
    for which in (0, 1):
        for i in range(pyfrozen.NCUBE):
            c = cm.cube(which, i)
            if len(c):
                cubes[(which, i)] = c
    frozen = pyfrozen.FrozenMap.from_cubes(cm.state()["centre"], cubes)
    init = np.array(poses[start], np.float64)
    init[4:6] += offset
    rows = RV.recover_track(frozen, RC.FrozenScorer(frozen), feats, init, start, frames, synth.RING_RANGES[1:], RV.deltas(aloam))
    return np.array(poses), rows
