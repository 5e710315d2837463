"""ctypes binding of the CPU oracle (oracle/liboracle.so).

ORACLE = test infrastructure.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import this module; the product path (a-loam_b200) never does.
Parity status: see oracle/oracle.h (in-tree code pinned to the reference's source, k-NN to a real FLANN; Ceres / VoxelGrid / Eigen restated).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

SORT_LITERAL, SORT_CANONICAL = 0, 1
EDGE, PLANE, PLANE_NORM = 0, 1, 2
BLOCK_DOUBLES = 11

_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_i32p = C.POINTER(C.c_int)


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    srcs = [os.path.join(_HERE, f) for f in os.listdir(_HERE) if f.endswith((".cc", ".h"))]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        L.orc_features_extract.restype = C.c_void_p
        L.orc_features_extract.argtypes = [_f32p, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, _i32p]
        L.orc_features_size.argtypes = [C.c_void_p, C.c_int]
        L.orc_features_copy.argtypes = [C.c_void_p, C.c_int, _f32p]
        L.orc_features_ints.argtypes = [C.c_void_p, C.c_int, _i32p]
        L.orc_features_curvature.argtypes = [C.c_void_p, _f32p]
        L.orc_features_times.argtypes = [C.c_void_p, _f64p]
        L.orc_features_free.argtypes = [C.c_void_p]
        L.orc_voxel_grid.argtypes = [_f32p, C.c_int, C.c_float, C.c_int, _f32p]
        L.orc_kdtree_build.restype = C.c_void_p
        L.orc_kdtree_build.argtypes = [_f32p, C.c_int]
        L.orc_kdtree_free.argtypes = [C.c_void_p]
        L.orc_kdtree_knn.argtypes = [C.c_void_p, _f32p, C.c_int, C.c_int, C.c_int, _i32p, _f32p]
        L.orc_bruteforce_knn.argtypes = [_f32p, C.c_int, _f32p, C.c_int, C.c_int, C.c_int, _i32p, _f32p]
        L.orc_make_edge.argtypes = [_f64p, _f64p, _f64p, C.c_double, _f64p]
        L.orc_make_plane.argtypes = [_f64p, _f64p, _f64p, _f64p, C.c_double, _f64p]
        L.orc_make_plane_norm.argtypes = [_f64p, _f64p, C.c_double, _f64p]
        L.orc_normal_equations.restype = C.c_double
        L.orc_normal_equations.argtypes = [_f64p, C.c_int, _f64p, C.c_double, C.c_int, _f64p, _f64p]
        L.orc_cost.restype = C.c_double
        L.orc_cost.argtypes = [_f64p, C.c_int, _f64p, C.c_double]
        L.orc_evaluate.argtypes = [_f64p, C.c_int, _f64p, C.c_double, C.c_int, _f64p, _f64p, _f64p]
        L.orc_solve.argtypes = [_f64p, C.c_int, _f64p, C.c_int, C.c_int, C.c_double, _f64p, _f64p, C.c_int]
        L.orc_quat_plus.argtypes = [_f64p, _f64p, _f64p]
        L.orc_odom_create.restype = C.c_void_p
        L.orc_odom_free.argtypes = [C.c_void_p]
        L.orc_odom_set_distortion.argtypes = [C.c_void_p, C.c_int]
        L.orc_transform_to_end.argtypes = [_f32p, C.c_int, _f64p, _f64p, C.c_int, _f32p]
        L.orc_odom_set_last.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int]
        L.orc_odom_associate.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int, _f64p, _f64p, _i32p, _i32p, _i32p, _i32p, _f64p, _i32p]
        L.orc_odom_register.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int, _f64p, _f64p, C.c_int, C.c_int, C.c_int, C.c_double, _f64p, _f64p, _i32p]
        L.orc_integrate_pose.argtypes = [_f64p, _f64p, _f64p, _f64p]
        L.orc_map_create.restype = C.c_void_p
        L.orc_map_free.argtypes = [C.c_void_p]
        L.orc_map_set_map.restype = C.c_double
        L.orc_map_set_map.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int]
        L.orc_map_associate.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int, _f64p, _f64p, _i32p, _f64p, _i32p]
        L.orc_map_register.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int, _f64p, C.c_int, C.c_int, C.c_int, C.c_double, _f64p, _f64p]
        L.orc_transform_associate_to_map.argtypes = [_f64p] * 5
        L.orc_transform_update.argtypes = [_f64p] * 5
        L.orc_eig3_sym.argtypes = [_f64p, _f64p, _f64p]
        L.orc_lsq_5x3.argtypes = [_f64p, _f64p, _f64p]
        L.orc_cubemap_create.restype = C.c_void_p
        L.orc_cubemap_free.argtypes = [C.c_void_p]
        L.orc_cubemap_step.argtypes = [C.c_void_p, _f32p, C.c_int, _f32p, C.c_int, _f64p, _f64p, C.c_float, C.c_float, C.c_int,
                                       C.c_int, C.c_double, C.c_int, _f64p, _i32p]
        L.orc_odom_set_params.argtypes = [C.c_void_p, C.c_double, C.c_double]
        L.orc_cubemap_get.argtypes = [C.c_void_p, C.c_int, _f32p, C.c_int]
        L.orc_cubemap_state.argtypes = [C.c_void_p, _i32p, _i32p, _i32p, C.POINTER(C.c_longlong), _f64p, _f64p]
        L.orc_cubemap_cube.argtypes = [C.c_void_p, C.c_int, C.c_int, _f32p, C.c_int]
        _LIB = L
    return _LIB


def _fp(a):
    return a.ctypes.data_as(_f32p)


def _dp(a):
    return a.ctypes.data_as(_f64p)


def _ip(a):
    return a.ctypes.data_as(_i32p)


def _cloud(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] == 4, a.shape
    return a


class Features:
    """scanRegistration.cpp:129-408 on one raw scan (n x >=3 float32, arrival order)."""

    def __init__(self, raw, n_scans, min_range, mode=SORT_CANONICAL):
        raw = np.ascontiguousarray(raw, dtype=np.float32)
        err = C.c_int(0)
        h = lib().orc_features_extract(_fp(raw), raw.shape[0], raw.shape[1], n_scans, float(min_range), mode, C.byref(err))
        if not h:
            raise RuntimeError("oracle extract_features failed: %d" % err.value)
        L = lib()
        out = []
        for w in range(5):
            n = L.orc_features_size(h, w)
            a = np.zeros((n, 4), np.float32)
            if n:
                L.orc_features_copy(h, w, _fp(a))
            out.append(a)
        self.full, self.sharp, self.less_sharp, self.flat, self.less_flat = out
        self.scan_start = np.zeros(n_scans, np.int32)
        self.scan_end = np.zeros(n_scans, np.int32)
        L.orc_features_ints(h, 0, _ip(self.scan_start))
        L.orc_features_ints(h, 1, _ip(self.scan_end))
        n = self.full.shape[0]
        self.label = np.zeros(n, np.int32)
        self.picked = np.zeros(n, np.int32)
        self.curvature = np.zeros(n, np.float32)
        if n:
            L.orc_features_ints(h, 2, _ip(self.label))
            L.orc_features_ints(h, 3, _ip(self.picked))
            L.orc_features_curvature(h, _fp(self.curvature))
        t = np.zeros(6)
        L.orc_features_times(h, _dp(t))
        self.times = dict(zip(["prepare_ms", "curvature_ms", "sort_ms", "pick_ms", "voxel_ms", "whole_ms"], t))
        L.orc_features_free(h)


def voxel_grid(cloud, leaf, mode=SORT_CANONICAL):
    cloud = _cloud(cloud)
    out = np.zeros_like(cloud)
    n = lib().orc_voxel_grid(_fp(cloud), cloud.shape[0], float(leaf), mode, _fp(out)) if cloud.shape[0] else 0
    return out[:n].copy()


class KdTree:
    def __init__(self, cloud):
        self.cloud = _cloud(cloud)
        self.h = lib().orc_kdtree_build(_fp(self.cloud), self.cloud.shape[0])

    def knn(self, queries, k):
        q = np.ascontiguousarray(queries, dtype=np.float32)
        idx = np.zeros((q.shape[0], k), np.int32)
        sqd = np.zeros((q.shape[0], k), np.float32)
        lib().orc_kdtree_knn(self.h, _fp(q), q.shape[0], q.shape[1], k, _ip(idx), _fp(sqd))
        return idx, sqd

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_kdtree_free(self.h)
            self.h = None


def bruteforce_knn(cloud, queries, k):
    cloud = _cloud(cloud)
    q = np.ascontiguousarray(queries, dtype=np.float32)
    idx = np.zeros((q.shape[0], k), np.int32)
    sqd = np.zeros((q.shape[0], k), np.float32)
    lib().orc_bruteforce_knn(_fp(cloud), cloud.shape[0], _fp(q), q.shape[0], q.shape[1], k, _ip(idx), _fp(sqd))
    return idx, sqd


def make_edge(cp, a, b, s=1.0):
    o = np.zeros(BLOCK_DOUBLES)
    lib().orc_make_edge(_dp(np.asarray(cp, np.float64)), _dp(np.asarray(a, np.float64)), _dp(np.asarray(b, np.float64)), s, _dp(o))
    return o


def make_plane(cp, j, l, m, s=1.0):
    o = np.zeros(BLOCK_DOUBLES)
    lib().orc_make_plane(_dp(np.asarray(cp, np.float64)), _dp(np.asarray(j, np.float64)), _dp(np.asarray(l, np.float64)),
                         _dp(np.asarray(m, np.float64)), s, _dp(o))
    return o


def make_plane_norm(cp, n, d):
    o = np.zeros(BLOCK_DOUBLES)
    lib().orc_make_plane_norm(_dp(np.asarray(cp, np.float64)), _dp(np.asarray(n, np.float64)), d, _dp(o))
    return o


def normal_equations(blocks, x, huber=0.1, autodiff=True):
    blocks = np.ascontiguousarray(blocks, np.float64).reshape(-1, BLOCK_DOUBLES)
    x = np.ascontiguousarray(x, np.float64)
    JtJ = np.zeros((6, 6))
    Jtr = np.zeros(6)
    cost = lib().orc_normal_equations(_dp(blocks), blocks.shape[0], _dp(x), huber, int(autodiff), _dp(JtJ), _dp(Jtr))
    return JtJ, Jtr, cost


def cost(blocks, x, huber=0.1):
    blocks = np.ascontiguousarray(blocks, np.float64).reshape(-1, BLOCK_DOUBLES)
    return lib().orc_cost(_dp(blocks), blocks.shape[0], _dp(np.ascontiguousarray(x, np.float64)), huber)


def evaluate(blocks, x, huber=0.1, autodiff=True):
    blocks = np.ascontiguousarray(blocks, np.float64).reshape(-1, BLOCK_DOUBLES)
    rows = int(np.sum(np.where(blocks[:, 0] == EDGE, 3, 1)))
    r = np.zeros(rows)
    J = np.zeros((rows, 6))
    c = C.c_double(0)
    lib().orc_evaluate(_dp(blocks), blocks.shape[0], _dp(np.ascontiguousarray(x, np.float64)), huber, int(autodiff), _dp(r), _dp(J), C.byref(c))
    return r, J, c.value


_SUMMARY_KEYS = ["termination", "num_iterations", "num_successful", "num_jac_evals", "num_cost_evals", "initial_cost", "final_cost"]


def solve(blocks, x, max_iters=4, autodiff=True, huber=0.1):
    blocks = np.ascontiguousarray(blocks, np.float64).reshape(-1, BLOCK_DOUBLES)
    x = np.array(x, np.float64)
    s = np.zeros(7)
    trace = np.zeros((max_iters + 2, 8))
    rows = lib().orc_solve(_dp(blocks), blocks.shape[0], _dp(x), max_iters, int(autodiff), huber, _dp(s), _dp(trace), trace.shape[0])
    return x, dict(zip(_SUMMARY_KEYS, s)), trace[:rows]


def quat_plus(q, d):
    o = np.zeros(4)
    lib().orc_quat_plus(_dp(np.ascontiguousarray(q, np.float64)), _dp(np.ascontiguousarray(d, np.float64)), _dp(o))
    return o


class Odometry:
    def __init__(self, distortion=False, dist_sq_thresh=25.0, nearby_scan=2.5):
        self.h = lib().orc_odom_create()
        if distortion:
            lib().orc_odom_set_distortion(self.h, 1)     # laserOdometry.cpp:59 #define DISTORTION 1
        lib().orc_odom_set_params(self.h, float(dist_sq_thresh), float(nearby_scan))   # :65-66

    def set_last(self, corner, surf):
        corner, surf = _cloud(corner), _cloud(surf)
        lib().orc_odom_set_last(self.h, _fp(corner), corner.shape[0], _fp(surf), surf.shape[0])

    def associate(self, sharp, flat, q, t):
        sharp, flat = _cloud(sharp), _cloud(flat)
        cc = np.zeros((max(sharp.shape[0], 1), 3), np.int32)
        pc = np.zeros((max(flat.shape[0], 1), 4), np.int32)
        bl = np.zeros((max(sharp.shape[0] + flat.shape[0], 1), BLOCK_DOUBLES))
        ncc, npc, nb = C.c_int(0), C.c_int(0), C.c_int(0)
        lib().orc_odom_associate(self.h, _fp(sharp), sharp.shape[0], _fp(flat), flat.shape[0],
                                 _dp(np.ascontiguousarray(q, np.float64)), _dp(np.ascontiguousarray(t, np.float64)),
                                 _ip(cc), C.byref(ncc), _ip(pc), C.byref(npc), _dp(bl), C.byref(nb))
        return cc[:ncc.value].copy(), pc[:npc.value].copy(), bl[:nb.value].copy()

    def register(self, sharp, flat, q, t, outer=2, max_iters=4, autodiff=True, huber=0.1):
        sharp, flat = _cloud(sharp), _cloud(flat)
        q = np.array(q, np.float64)
        t = np.array(t, np.float64)
        summ = np.zeros((outer, 7))
        times = np.zeros(3)
        counts = np.zeros(2, np.int32)
        lib().orc_odom_register(self.h, _fp(sharp), sharp.shape[0], _fp(flat), flat.shape[0], _dp(q), _dp(t), outer, max_iters,
                                int(autodiff), huber, _dp(summ), _dp(times), _ip(counts))
        info = {"summaries": [dict(zip(_SUMMARY_KEYS, s)) for s in summ], "assoc_ms": times[0], "solve_ms": times[1],
                "tree_ms": times[2], "corner_corr": int(counts[0]), "plane_corr": int(counts[1])}
        return q, t, info

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_odom_free(self.h)
            self.h = None


def transform_to_end(cloud, q, t, distortion=True):
    """laserOdometry.cpp:133-148 (dead code in the reference: only called under `if (0)`)"""
    cloud = _cloud(cloud)
    out = np.zeros_like(cloud)
    lib().orc_transform_to_end(_fp(cloud), cloud.shape[0], _dp(np.ascontiguousarray(q, np.float64)), _dp(np.ascontiguousarray(t, np.float64)),
                               int(distortion), _fp(out))
    return out


def integrate_pose(q_w, t_w, q, t):
    q_w = np.array(q_w, np.float64)
    t_w = np.array(t_w, np.float64)
    lib().orc_integrate_pose(_dp(q_w), _dp(t_w), _dp(np.ascontiguousarray(q, np.float64)), _dp(np.ascontiguousarray(t, np.float64)))
    return q_w, t_w


class Mapping:
    def __init__(self):
        self.h = lib().orc_map_create()
        self.tree_ms = 0.0

    def set_map(self, corner, surf):
        corner, surf = _cloud(corner), _cloud(surf)
        self.tree_ms = lib().orc_map_set_map(self.h, _fp(corner), corner.shape[0], _fp(surf), surf.shape[0])

    def associate(self, corner, surf, x):
        corner, surf = _cloud(corner), _cloud(surf)
        n = max(corner.shape[0] + surf.shape[0], 1)
        fits = np.zeros((n, 14))
        bl = np.zeros((n, BLOCK_DOUBLES))
        nf, nb = C.c_int(0), C.c_int(0)
        lib().orc_map_associate(self.h, _fp(corner), corner.shape[0], _fp(surf), surf.shape[0],
                                _dp(np.ascontiguousarray(x, np.float64)), _dp(fits), C.byref(nf), _dp(bl), C.byref(nb))
        return fits[:nf.value].copy(), bl[:nb.value].copy()

    def register(self, corner, surf, x, outer=2, max_iters=4, autodiff=True, huber=0.1):
        corner, surf = _cloud(corner), _cloud(surf)
        x = np.array(x, np.float64)
        summ = np.zeros((outer, 7))
        times = np.zeros(3)
        rc = lib().orc_map_register(self.h, _fp(corner), corner.shape[0], _fp(surf), surf.shape[0], _dp(x), outer, max_iters,
                                    int(autodiff), huber, _dp(summ), _dp(times))
        info = {"optimised": bool(rc), "summaries": [dict(zip(_SUMMARY_KEYS, s)) for s in summ], "assoc_ms": times[0],
                "solve_ms": times[1], "tree_ms": self.tree_ms}
        return x, info

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_map_free(self.h)
            self.h = None


def transform_associate_to_map(q_wmap_wodom, t_wmap_wodom, q_wodom_curr, t_wodom_curr):
    """laserMapping.cpp:142-146 -> parameters[7]"""
    x = np.zeros(7)
    lib().orc_transform_associate_to_map(_dp(np.ascontiguousarray(q_wmap_wodom, np.float64)), _dp(np.ascontiguousarray(t_wmap_wodom, np.float64)),
                                         _dp(np.ascontiguousarray(q_wodom_curr, np.float64)), _dp(np.ascontiguousarray(t_wodom_curr, np.float64)), _dp(x))
    return x


def transform_update(x, q_wodom_curr, t_wodom_curr):
    """laserMapping.cpp:148-152 -> (q_wmap_wodom, t_wmap_wodom)"""
    q = np.zeros(4); t = np.zeros(3)
    lib().orc_transform_update(_dp(np.ascontiguousarray(x, np.float64)), _dp(np.ascontiguousarray(q_wodom_curr, np.float64)),
                               _dp(np.ascontiguousarray(t_wodom_curr, np.float64)), _dp(q), _dp(t))
    return q, t


class CubeMap:
    """laserMapping.cpp's 21 x 21 x 11 cube store and the per-frame loop around it (oracle/cubemap.cc, SURVEY 8 f-1)"""

    def __init__(self):
        self.h = lib().orc_cubemap_create()

    def step(self, corner_last, surf_last, q_wodom_curr, t_wodom_curr, line_res=0.4, plane_res=0.8, outer=2, max_iters=4,
             sort_mode=SORT_CANONICAL, huber=0.1):
        c, s = _cloud(corner_last), _cloud(surf_last)
        pose = np.zeros(7)
        info = np.zeros(6, np.int32)
        lib().orc_cubemap_step(self.h, _fp(c), c.shape[0], _fp(s), s.shape[0], _dp(np.ascontiguousarray(q_wodom_curr, np.float64)),
                               _dp(np.ascontiguousarray(t_wodom_curr, np.float64)), line_res, plane_res, outer, max_iters, huber, sort_mode,
                               _dp(pose), info.ctypes.data_as(_i32p))
        keys = ["optimised", "n_valid", "corner_from_map", "surf_from_map", "corner_stack", "surf_stack"]
        return pose, dict(zip(keys, (int(v) for v in info)))

    def _get(self, fn, *a):
        n = fn(self.h, *a, None, 0)
        out = np.zeros((max(n, 1), 4), np.float32)
        fn(self.h, *a, _fp(out), n)
        return out[:max(n, 0)].copy()

    def cloud(self, which):
        """0 corner_from_map, 1 surf_from_map, 2 corner_stack, 3 surf_stack of the last step"""
        return self._get(lib().orc_cubemap_get, which)

    def cube(self, which, index):
        return self._get(lib().orc_cubemap_cube, which, index)

    def state(self):
        cen = np.zeros(3, np.int32); nv = np.zeros(1, np.int32); valid = np.zeros(125, np.int32)
        tot = (C.c_longlong * 2)(); q = np.zeros(4); t = np.zeros(3)
        lib().orc_cubemap_state(self.h, cen.ctypes.data_as(_i32p), nv.ctypes.data_as(_i32p), valid.ctypes.data_as(_i32p), tot, _dp(q), _dp(t))
        return {"centre": tuple(int(v) for v in cen), "valid": [int(v) for v in valid[:nv[0]]], "total_corner": int(tot[0]),
                "total_surf": int(tot[1]), "q_wmap_wodom": q, "t_wmap_wodom": t}

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_cubemap_free(self.h)
            self.h = None


def eig3_sym(A):
    A = np.ascontiguousarray(A, np.float64)
    ev = np.zeros(3)
    V = np.zeros((3, 3))
    lib().orc_eig3_sym(_dp(A), _dp(ev), _dp(V))
    return ev, V


def lsq_5x3(A, b):
    n = np.zeros(3)
    lib().orc_lsq_5x3(_dp(np.ascontiguousarray(A, np.float64)), _dp(np.ascontiguousarray(b, np.float64)), _dp(n))
    return n
