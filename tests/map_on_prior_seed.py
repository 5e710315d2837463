"""Seeding the CPU mappers with the starting state of a mapping trajectory on a copy of a prior map (aloam_lane_map_on_prior): the
oracle's CubeMap and the reference's own laserMapping.cpp node of a loaded oracle/_ref/libref_mapping.so.  The C++ side is
tests/cpp/map_on_prior_seed.cc, compiled once per session into a temporary directory.  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NCUBE = 21 * 21 * 11
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(tempfile.mkdtemp(prefix="seed_"), "libmap_on_prior_seed.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-w",
                               "-I" + os.path.join(ROOT, "oracle"), "-I" + os.path.join(ROOT, "oracle", "ref_shim"),
                               "-o", so, os.path.join(ROOT, "tests", "cpp", "map_on_prior_seed.cc")])
        L = C.CDLL(so)
        dp, ip, fp, vp = C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_float), C.c_void_p
        L.seed_cubemap.argtypes = [vp, ip, dp, dp, ip, fp]
        L.seed_ref_node.argtypes = [vp, vp, vp, vp, vp, vp, vp, ip, dp, dp, ip, fp]
        _LIB = L
    return _LIB


def _args(centre, q, t, counts, points):
    cen = np.ascontiguousarray(centre, np.int32)
    q = np.ascontiguousarray(q, np.float64)
    t = np.ascontiguousarray(t, np.float64)
    cnt = np.ascontiguousarray(counts, np.int32).reshape(2, NCUBE)
    pts = np.ascontiguousarray(points, np.float32).reshape(-1, 4)
    if pts.shape[0] != int(np.maximum(cnt, 0).sum()):
        raise ValueError("points must hold the counted points")
    keep = (cen, q, t, cnt, pts)
    return keep, [cen.ctypes.data_as(C.POINTER(C.c_int)), q.ctypes.data_as(C.POINTER(C.c_double)), t.ctypes.data_as(C.POINTER(C.c_double)),
                  cnt.ctypes.data_as(C.POINTER(C.c_int)), pts.ctypes.data_as(C.POINTER(C.c_float))]


def seed_cubemap(cm, centre, q_wmap_wodom, t_wmap_wodom, counts, points):
    """the oracle CubeMap cm (pyoracle.CubeMap) with centre offsets, T_wmap_wodom (q xyzw, t), counts (2, 4851) points per corner /
    surf cube (< 0: none) and the points in ALOAM_EXPORT_MAP order; no valid list, frames = 0"""
    keep, a = _args(centre, q_wmap_wodom, t_wmap_wodom, counts, points)
    _lib().seed_cubemap(cm.h, *a)


def seed_ref(ref, centre, q_wmap_wodom, t_wmap_wodom, counts, points):
    """the same state in the globals of the reference node of ref (refsource.RefMapping, after its ref_map_init): its cube arrays,
    laserCloudCenWidth / Height / Depth, q_wmap_wodom and t_wmap_wodom"""
    keep, a = _args(centre, q_wmap_wodom, t_wmap_wodom, counts, points)
    g = [C.addressof(C.c_char.in_dll(ref.lib, name)) for name in ("laserCloudCornerArray", "laserCloudSurfArray", "laserCloudCenWidth",
                                                                  "laserCloudCenHeight", "laserCloudCenDepth", "q_wmap_wodom", "t_wmap_wodom")]
    _lib().seed_ref_node(*g, *a)
