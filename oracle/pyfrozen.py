"""ctypes binding of oracle/libfrozen.so: the frozen-map frame of localisation against a prior map (oracle/frozen.cc) -- the
mapper's frame without the ring-buffer shift and without insertion / re-filter.  ORACLE = test infrastructure, like pyoracle."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int)
NCUBE = 21 * 21 * 11


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libfrozen.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-f", "frozen.mk", "libfrozen.so"], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.orc_frozen_create.argtypes = [_i32p]
        L.orc_frozen_create.restype = C.c_void_p
        L.orc_frozen_free.argtypes = [C.c_void_p]
        L.orc_frozen_set_cube.argtypes = [C.c_void_p, C.c_int, C.c_int, _f32p, C.c_int]
        L.orc_frozen_get_cube.argtypes = [C.c_void_p, C.c_int, C.c_int, _f32p, C.c_int]
        L.orc_frozen_step.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int, _f64p, _f64p, _f64p, _f64p, C.c_float, C.c_float, C.c_int, C.c_int,
                                      C.c_double, C.c_int, _f64p, _i32p, _i32p]
        L.orc_frozen_high_freq.argtypes = [_f64p] * 5
        L.orc_frozen_high_freq.restype = None
        _LIB = L
    return _LIB


def _cloud(a):
    a = np.ascontiguousarray(a, np.float32)
    assert a.ndim == 2 and a.shape[1] == 4, a.shape
    return a


def _dp(a):
    return a.ctypes.data_as(_f64p)


class FrozenMap:
    """a prior map: the cubes of a store and its centre offsets; frames read it and never write it"""

    def __init__(self, centre=(10, 10, 5)):
        self.centre = tuple(int(v) for v in centre)
        self.h = lib().orc_frozen_create((C.c_int * 3)(*self.centre))

    @classmethod
    def from_cubes(cls, centre, cubes):
        """cubes: {(which, index): (n, 4) cloud}, which = 0 corner, 1 surf"""
        m = cls(centre)
        for (which, index), pts in cubes.items():
            m.set_cube(which, index, pts)
        return m

    @classmethod
    def from_export(cls, centre, counts, points):
        """counts: (2, 4851) points per corner / surf cube (-1 counts as 0); points: the store in ALOAM_EXPORT_MAP order"""
        m = cls(centre)
        off = 0
        for i in range(NCUBE):
            for which in (0, 1):
                n = max(int(counts[which][i]), 0)
                if n:
                    m.set_cube(which, i, points[off:off + n])
                off += n
        return m

    def set_cube(self, which, index, pts):
        p = _cloud(pts)
        assert lib().orc_frozen_set_cube(self.h, which, index, p.ctypes.data_as(_f32p), p.shape[0]) == 0

    def cube(self, which, index):
        n = lib().orc_frozen_get_cube(self.h, which, index, None, 0)
        out = np.zeros((max(n, 1), 4), np.float32)
        lib().orc_frozen_get_cube(self.h, which, index, out.ctypes.data_as(_f32p), n)
        return out[:n].copy()

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_frozen_free(self.h)
            self.h = None


class Localiser:
    """one vehicle localising against a FrozenMap: its T_wmap_wodom starts at (q_init, t_init); scan j registers when
    j % skip == 0 and otherwise gets the high-frequency pose (laserMapping.cpp:197-229).  normalise: q_init / |q_init|, summed in
    index order, as aloam_lane_localise takes it; False keeps its bits (to continue from a mapper's own T_wmap_wodom)"""

    def __init__(self, frozen, q_init, t_init, skip=1, normalise=True):
        self.map = frozen
        q = np.array(q_init, np.float64)
        n2 = 0.0
        for v in q:
            n2 += float(v) * float(v)
        self.q = q / np.sqrt(n2) if normalise else q
        self.t = np.array(t_init, np.float64)
        self.skip, self.scan = int(skip), 0
        self.valid, self.info = [], {}

    def step(self, corner_last, surf_last, q_wodom_curr, t_wodom_curr, line_res=0.4, plane_res=0.8, outer=2, max_iters=4, sort_mode=1,
             huber=0.1):
        qo, to = np.ascontiguousarray(q_wodom_curr, np.float64), np.ascontiguousarray(t_wodom_curr, np.float64)
        pose = np.zeros(7)
        j, self.scan = self.scan, self.scan + 1
        if j % self.skip:
            lib().orc_frozen_high_freq(_dp(self.q), _dp(self.t), _dp(qo), _dp(to), _dp(pose))
            return pose, None
        c, s = _cloud(corner_last), _cloud(surf_last)
        valid = np.zeros(75, np.int32); info = np.zeros(6, np.int32)
        lib().orc_frozen_step(self.map.h, c.ctypes.data_as(_f32p), c.shape[0], s.ctypes.data_as(_f32p), s.shape[0], _dp(qo), _dp(to), _dp(self.q),
                              _dp(self.t), line_res, plane_res, outer, max_iters, huber, sort_mode, _dp(pose), valid.ctypes.data_as(_i32p),
                              info.ctypes.data_as(_i32p))
        keys = ["optimised", "n_valid", "corner_from_map", "surf_from_map", "corner_stack", "surf_stack"]
        self.info = dict(zip(keys, (int(v) for v in info)))
        self.valid = [int(v) for v in valid[:info[1]]]
        return pose, self.info
