"""The oracle's feature extraction with the driver's ring (aloam_config.ring_source = ALOAM_RING_FIELD).  TEST INFRASTRUCTURE.

Field mode is oracle/features.cc with one decision replaced: a return's ring is float 3 of the raw point when that is an
integer in 0 .. n_scans - 1, and the return is dropped otherwise, where the elevation mode calls ring_of (scanRegistration.cpp
:166-205).  So the module builds it from that file's own text: it carries the fourth float through the NaN / range filter,
accepts n_scans 1..64 and swaps the ring_of call, and compiles the result with the other oracle sources into a private
library, once per session, in a temporary directory.  Every other line, the azimuth walk and the feature stages included, is
the elevation oracle's; a change there that touches one of the four edited lines fails here loudly instead of drifting."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import pyoracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE = os.path.join(ROOT, "oracle")
_LIB = None

# (text of oracle/features.cc, field-mode text); each must occur exactly once
EDITS = [
    ("struct Xyz { float x, y, z; };",
     "struct Xyz { float x, y, z, w; };\n"
     "// the driver's ring: w when it is an integer in 0 .. n_scans - 1, else -1 (NaN fails every comparison, +-inf the range)\n"
     "inline int ring_field(float w, int n_scans) { return w >= 0 && w < n_scans && w == std::trunc(w) ? (int)w : -1; }"),
    ("if (n_scans != 16 && n_scans != 32 && n_scans != 64) return -1;",
     "if (n_scans < 1 || n_scans > 64 || stride < 4) return -1;"),
    ("in.push_back({p[0], p[1], p[2]});", "in.push_back({p[0], p[1], p[2], p[3]});"),
    ("const int id = ring_of(angle, n_scans);", "const int id = ring_field(p.w, n_scans);"),
]


def field_source():
    src = open(os.path.join(ORACLE, "features.cc")).read()
    for old, new in EDITS:
        if src.count(old) != 1:
            raise RuntimeError("oracle/features.cc no longer holds %r exactly once" % old)
        src = src.replace(old, new)
    return src


def _lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix="ring_field_")
        src = os.path.join(d, "features_field.cc")
        with open(src, "w") as f:
            f.write(field_source())
        others = [os.path.join(ORACLE, s) for s in ("voxelgrid.cc", "kdtree.cc", "lm.cc", "odometry.cc", "mapping.cc", "cubemap.cc", "capi.cc")]
        so = os.path.join(d, "liboracle_field.so")
        # the flags of oracle/Makefile (liboracle.so)
        subprocess.check_call(["g++", "-std=c++17", "-O3", "-fPIC", "-ffp-contract=off", "-w", "-shared", "-I" + ORACLE, "-o", so, src] + others)
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
    """pyoracle.Features(raw, n_scans, min_range, mode) in field mode: raw is (n, 4 | 8) float32 with the ring in column 3"""
    raw = np.ascontiguousarray(raw, np.float32)
    if raw.ndim != 2 or raw.shape[1] < 4:
        raise ValueError("a field-mode raw scan has the ring in float 3")
    lib = _lib()
    saved = orc._LIB
    orc._LIB = lib   # pyoracle.Features reads its results through pyoracle.lib(); the field library has the same entry points
    try:
        return orc.Features(raw, n_scans, min_range, mode)
    finally:
        orc._LIB = saved


def formula_rings(raw, n_scans):
    """raw (n, 4) with float 3 set to the elevation formula's ring of each return (-1 where the formula drops it): field mode
    then assigns exactly the rings of the elevation mode"""
    from ring_edge_cases import ring_ids
    out = np.array(raw, np.float32, copy=True)
    out[:, 3] = ring_ids(out, n_scans)
    return out


def elevation_cases(synth):
    """(tag, raw, n_scans, minimum_range) of the elevation sensors: two scans each, a seam scan (cut, 1.05 turns, per-beam
    azimuth offsets, laser-major, counter-clockwise) and a scan whose returns sit on every ring edge of each formula"""
    import ring_edge_cases as E
    import seam_cases as S
    for sensor, n_az in (("VLP-16", 900), ("HDL-32", 1100), ("HDL-64", None)):
        ns, _, mr = synth.SENSORS[sensor][:3]
        for k in (0, 3):
            yield "%s/%d" % (sensor, k), (synth.scan(sensor, k, n_az=n_az) if n_az else synth.scan(sensor, k)), ns, mr
        yield "%s/seam" % sensor, S.seam_scan(synth, sensor, 1, S.CUTS[2], 1.05, S.ring_offsets(ns), True, True), ns, mr
    for ns in (16, 32, 64):
        yield "edges/%d" % ns, E.edge_scan(ns)[0], ns, E.MIN_RANGE[ns]
