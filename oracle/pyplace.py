"""ctypes binding of oracle/libplace.so: the oracle of place recognition (oracle/place.cc) -- the Scan Context descriptor, the
column-shifted distance, query ranking and the keyframe gate of include/aloam_b200.h -- and KeyframeTable, one lane's keyframe
table as the mapped stream calls keep it.  ORACLE = test infrastructure, like pyoracle."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int)
RINGS, SECTORS = 20, 60
# one keyframe record (ALOAM_PLACE_RECORD_BYTES = 4880, little-endian)
RECORD_DTYPE = np.dtype([("pose", "<f8", (7,)), ("scan_index", "<i4"), ("lane", "<i4"), ("max_range", "<f4"), ("z_offset", "<f4"),
                         ("pad", "<i4", (2,)), ("desc", "<f4", (RINGS * SECTORS,))])
assert RECORD_DTYPE.itemsize == 4880


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libplace.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-f", "place.mk", "libplace.so"], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.orc_place_describe.argtypes = [_f32p, C.c_int, _f32p, C.c_int, C.c_float, C.c_float, _f32p]
        L.orc_place_describe.restype = None
        L.orc_place_norms.argtypes = [_f32p, _f64p]
        L.orc_place_norms.restype = None
        L.orc_place_distance.argtypes = [_f32p, _f32p, _f64p, _i32p]
        L.orc_place_distance.restype = None
        L.orc_place_query.argtypes = [_f32p, C.c_int, _f32p, C.c_longlong, C.c_int, C.c_int, _i32p, _i32p, _f64p]
        L.orc_place_query.restype = None
        L.orc_place_gate.argtypes = [_f64p, _f64p, C.c_double]
        L.orc_place_gate.restype = C.c_int
        _LIB = L
    return _LIB


def _cloud(a):
    a = np.ascontiguousarray(np.asarray(a, np.float32).reshape(-1, 4) if np.size(a) else np.zeros((0, 4), np.float32))
    return a


def describe(less_sharp, less_flat, max_range=80.0, z_offset=2.0):
    """the (1200,) float32 descriptor of a scan (ring-major: bin (r, s) at r * 60 + s)"""
    a, b = _cloud(less_sharp), _cloud(less_flat)
    out = np.zeros(RINGS * SECTORS, np.float32)
    lib().orc_place_describe(a.ctypes.data_as(_f32p), a.shape[0], b.ctypes.data_as(_f32p), b.shape[0], max_range, z_offset,
                             out.ctypes.data_as(_f32p))
    return out


def norms(desc):
    d = np.ascontiguousarray(desc, np.float32).ravel()
    out = np.zeros(SECTORS)
    lib().orc_place_norms(d.ctypes.data_as(_f32p), out.ctypes.data_as(_f64p))
    return out


def distance(q, d):
    """(D, shift) of query descriptor q against keyframe descriptor d"""
    q = np.ascontiguousarray(q, np.float32).ravel(); d = np.ascontiguousarray(d, np.float32).ravel()
    D = C.c_double(0); s = C.c_int(0)
    lib().orc_place_distance(q.ctypes.data_as(_f32p), d.ctypes.data_as(_f32p), C.byref(D), C.byref(s))
    return D.value, s.value


def query(descs, db_descs, k):
    """the k best keyframes of db_descs ((M, 1200)) for every query of descs ((n, 1200)), by (D, index) -> (index, shift,
    distance), (n, k) each"""
    q = np.ascontiguousarray(descs, np.float32).reshape(-1, RINGS * SECTORS)
    db = np.ascontiguousarray(db_descs, np.float32).reshape(-1, RINGS * SECTORS)
    n, M = q.shape[0], db.shape[0]
    idx = np.zeros((n, k), np.int32); sh = np.zeros((n, k), np.int32); dist = np.zeros((n, k))
    lib().orc_place_query(q.ctypes.data_as(_f32p), n, db.ctypes.data_as(_f32p), RINGS * SECTORS, M, k, idx.ctypes.data_as(_i32p),
                          sh.ctypes.data_as(_i32p), dist.ctypes.data_as(_f64p))
    return idx, sh, dist


def gate(last_t, t, keyframe_gap):
    lt = None if last_t is None else np.ascontiguousarray(last_t, np.float64)
    tt = np.ascontiguousarray(t, np.float64)
    return bool(lib().orc_place_gate(None if lt is None else lt.ctypes.data_as(_f64p), tt.ctypes.data_as(_f64p),
                                     float(keyframe_gap) * float(keyframe_gap)))


class KeyframeTable:
    """one lane's keyframe table as the mapped stream calls keep it: add() takes a MAPPED row's less-sharp / less-flat clouds and
    its map pose (as the device computed it) and returns the row's place record {keyframe, loop, shift, distance, full}"""

    def __init__(self, lane, max_range=80.0, z_offset=2.0, keyframe_gap=0.0, exclude_recent=0, max_keyframes=65536):
        self.lane, self.max_range, self.z_offset = int(lane), float(max_range), float(z_offset)
        self.gap, self.exclude, self.cap = float(keyframe_gap), int(exclude_recent), int(max_keyframes)
        self.records = np.zeros(0, RECORD_DTYPE)

    def clear(self):
        self.records = np.zeros(0, RECORD_DTYPE)

    def add(self, less_sharp, less_flat, pose, scan_index, start=False):
        if start:
            self.clear()
        n = len(self.records)
        row = {"keyframe": -1, "loop": -1, "shift": -1, "distance": -1.0, "full": 0}
        if not gate(self.records["pose"][-1][4:] if n else None, np.asarray(pose)[4:], self.gap):
            return row
        if n >= self.cap:
            row["full"] = 1
            return row
        r = np.zeros(1, RECORD_DTYPE)
        r["pose"] = np.asarray(pose, np.float64); r["scan_index"] = scan_index; r["lane"] = self.lane
        r["max_range"] = self.max_range; r["z_offset"] = self.z_offset
        r["desc"] = describe(less_sharp, less_flat, self.max_range, self.z_offset)
        self.records = np.concatenate([self.records, r])
        row["keyframe"] = n
        m = n - self.exclude
        if m > 0:
            i, s, d = query(r["desc"], self.records["desc"][:m], 1)
            row.update(loop=int(i[0, 0]), shift=int(s[0, 0]), distance=float(d[0, 0]))
        return row
