"""aloam-b200: H100-native (sm_90a) A-LOAM per-scan registration hot path.

Python here is only a ctypes mirror of the C ABI in include/aloam_b200.h (the reference is C++; its host side is
C++ inside libaloam_b200.so).  There is no CPU fallback: importing works anywhere (so the symbol table can be
checked on a CPU box) but creating a context needs a CUDA device and fails loudly without one.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_HERE, "libaloam_b200.so")
_LIB = None

OK = 0
FLAG_FEW_CORRESPONDENCES, FLAG_MAP_TOO_THIN, FLAG_INITIALISED_ONLY, FLAG_CUBE_OVERFLOW = 1, 2, 4, 8
BLOCK_DOUBLES = 11

EXPORTED_SYMBOLS = [
    "aloam_default_config", "aloam_create", "aloam_destroy", "aloam_strerror", "aloam_extract_features",
    "aloam_odometry_set_last", "aloam_odometry_register", "aloam_map_upload", "aloam_mapping_register",
    "aloam_voxel_filter", "aloam_scan_to_pose", "aloam_scan_to_pose_device", "aloam_reset_odometry", "aloam_knn",
    "aloam_odometry_associate", "aloam_normal_equations", "aloam_solve", "aloam_debug_features", "aloam_mapping_associate",
    "aloam_comm_unique_id", "aloam_comm_init", "aloam_comm_uses_peer_memory", "aloam_map_upload_sharded", "aloam_scan_stream", "aloam_scan_stream_batch", "aloam_scan_stream_mapped", "aloam_transform_to_end", "aloam_mapper_reset", "aloam_mapper_step", "aloam_debug_seg_voxel_filter", "aloam_profile_enable", "aloam_profile_read", "aloam_launch_count",
    "aloam_scan_stream_mapped_batch", "aloam_mapper_debug_state_lane", "aloam_mapper_debug_cube_lane",
    "aloam_scan_stream_lanes", "aloam_debug_shard_emulate", "aloam_debug_map_sizes",
    "aloam_mapper_export", "aloam_set_registered_sink", "aloam_registered_rows",
    "aloam_lane_save", "aloam_lane_restore", "aloam_snapshot_check",
    "aloam_prior_map_load", "aloam_prior_map_clear", "aloam_lane_localise", "aloam_debug_prior_associate",
    "aloam_prior_map_build", "aloam_prior_relocalise",
    "aloam_set_map_rows", "aloam_map_rows",
    "aloam_set_recovery", "aloam_recovery_rows", "aloam_debug_recovery_scores",
    "aloam_lane_map_on_prior", "aloam_set_cube_growth",
    "aloam_io_unpack_points_ring",
    "aloam_create_wide",
    "aloam_prior_map_digest", "aloam_lane_save_localising", "aloam_snapshot_localise_info",
    "aloam_set_place", "aloam_place_rows", "aloam_place_keyframes", "aloam_place_db_load", "aloam_place_db_clear",
    "aloam_place_describe", "aloam_place_query",
    "aloam_set_loops", "aloam_loop_rows", "aloam_loop_verify", "aloam_place_keyframe_cloud",
]
ERR_SNAPSHOT = -11
LANE_IDLE, LANE_SCAN, LANE_START = 0, 1, 2
EXPORT_SURROUND, EXPORT_MAP = 0, 1
PRIOR_MAP = -1   # `lane` of mapper_export: the context's prior map
ROW_IDLE, ROW_MAPPED, ROW_LOCALISED, ROW_SKIPPED = 0, 1, 2, 3   # aloam_map_row.kind
RING_ELEVATION, RING_FIELD = 0, 1   # aloam_config.ring_source: the elevation formula, or the driver's ring in float 3 of a raw point
MAX_RINGS = 128   # ALOAM_MAX_RINGS: the most rings a context takes (Aloam(..., wide=True), driver rings only)
MAX_CUBE_POINTS = 262144   # ALOAM_MAX_CUBE_POINTS: the most points one map cube holds with cube growth on (set_cube_growth)
PLACE_RINGS, PLACE_SECTORS, PLACE_MAX_K = 20, 60, 64   # the Scan Context grid and the most matches a query returns
# one keyframe record (ALOAM_PLACE_RECORD_BYTES, little-endian): the row's map pose (q xyzw, t), its scan index in its trajectory,
# its lane, the descriptor parameters and the ring-major descriptor
PLACE_RECORD_DTYPE = np.dtype([("pose", "<f8", (7,)), ("scan_index", "<i4"), ("lane", "<i4"), ("max_range", "<f4"), ("z_offset", "<f4"),
                               ("pad", "<i4", (2,)), ("desc", "<f4", (PLACE_RINGS * PLACE_SECTORS,))])
assert PLACE_RECORD_DTYPE.itemsize == 4880, "aloam place record layout"


class Config(C.Structure):
    _fields_ = [("n_scans", C.c_int), ("minimum_range", C.c_float), ("line_res", C.c_float), ("plane_res", C.c_float),
                ("outer_iters", C.c_int), ("inner_iters", C.c_int), ("huber", C.c_double), ("dist_sq_thresh", C.c_double),
                ("nearby_scan", C.c_double), ("device", C.c_int), ("max_points", C.c_int), ("max_map_points", C.c_int),
                ("max_batch", C.c_int), ("distortion", C.c_int), ("max_ring_points", C.c_int), ("mapping_skip_frame", C.c_int)]

    # aloam_config.ring_source, appended after mapping_skip_frame, is the int in the 8-byte tail padding of the fields above:
    # the structure keeps the size and layout of aloam_config (80 bytes) with the older field list
    @property
    def ring_source(self):
        return C.c_int.from_buffer(self, _RING_SOURCE_AT).value

    @ring_source.setter
    def ring_source(self, v):
        C.c_int.from_buffer(self, _RING_SOURCE_AT).value = v


_RING_SOURCE_AT = Config.mapping_skip_frame.offset + 4
assert C.sizeof(Config) == _RING_SOURCE_AT + 4, "aloam_config layout"


class CloudView(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_float)), ("n", C.c_int), ("stride_floats", C.c_int)]


class Stats(C.Structure):
    _fields_ = [("n_corner_corr", C.c_int), ("n_plane_corr", C.c_int), ("lm_iters", C.c_int), ("accepted_steps", C.c_int),
                ("flags", C.c_int), ("termination", C.c_int * 4), ("init_cost", C.c_double), ("final_cost", C.c_double),
                ("ms_total", C.c_float)]

    def as_dict(self):
        return {"n_corner_corr": self.n_corner_corr, "n_plane_corr": self.n_plane_corr, "lm_iters": self.lm_iters,
                "accepted_steps": self.accepted_steps, "flags": self.flags, "termination": list(self.termination),
                "init_cost": self.init_cost, "final_cost": self.final_cost, "ms_total": self.ms_total}


class SnapshotInfo(C.Structure):
    _fields_ = [("version", C.c_int), ("mapped", C.c_int), ("n_scans", C.c_int), ("scan_index", C.c_int), ("bytes", C.c_longlong),
                ("map_points", C.c_longlong), ("world", C.c_double * 7)]


class RelocOpts(C.Structure):
    _fields_ = [("inlier_sq", C.c_float), ("max_score_points", C.c_int), ("refine", C.c_int)]


class RelocResult(C.Structure):
    _fields_ = [("hyp", C.c_int), ("score", C.c_int), ("refined_score", C.c_int), ("flags", C.c_int), ("pose", C.c_double * 7)]


class MapRow(C.Structure):
    _fields_ = [("kind", C.c_int), ("err", C.c_int), ("n_valid", C.c_int), ("n_sub", C.c_int * 2), ("n_stack", C.c_int * 2),
                ("score", C.c_int), ("n_score", C.c_int), ("stats", Stats)]


class RecoveryOpts(C.Structure):
    _fields_ = [("trigger_frac", C.c_float), ("accept_frac", C.c_float)]


class RecoveryRow(C.Structure):
    _fields_ = [("triggered", C.c_int), ("best", C.c_int), ("best_score", C.c_int), ("adopted", C.c_int), ("pose", C.c_double * 7)]


class PlaceOpts(C.Structure):
    _fields_ = [("max_range", C.c_float), ("z_offset", C.c_float), ("keyframe_gap", C.c_double), ("exclude_recent", C.c_int),
                ("max_keyframes", C.c_int)]


class PlaceRow(C.Structure):
    _fields_ = [("keyframe", C.c_int), ("loop", C.c_int), ("shift", C.c_int), ("full", C.c_int), ("distance", C.c_double)]


class PlaceMatch(C.Structure):
    _fields_ = [("keyframe", C.c_int), ("shift", C.c_int), ("distance", C.c_double)]


class LoopOpts(C.Structure):
    _fields_ = [("max_distance", C.c_double), ("window", C.c_int), ("cloud_points", C.c_int), ("outer_iters", C.c_int),
                ("inlier_sq", C.c_float)]


class LoopRow(C.Structure):
    _fields_ = [("query", C.c_int), ("cand", C.c_int), ("verified", C.c_int), ("shift", C.c_int), ("n_sub", C.c_int * 2),
                ("score", C.c_int), ("n_score", C.c_int), ("stats", Stats), ("pose", C.c_double * 7), ("rel", C.c_double * 7)]

    def as_dict(self):
        return {"query": self.query, "cand": self.cand, "verified": self.verified, "shift": self.shift, "n_sub": tuple(self.n_sub),
                "score": self.score, "n_score": self.n_score, "stats": self.stats.as_dict(), "pose": np.array(self.pose[:]),
                "rel": np.array(self.rel[:])}


class AloamError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("aloam_b200 error %d: %s" % (code, msg))
        self.code = code


def build(force=False, verbose=False):
    from . import _build
    return _build.build(force=force, verbose=verbose)


def lib():
    """Loads libaloam_b200.so (raises if it has not been built -- there is no fallback)."""
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO_PATH):
            raise ImportError("libaloam_b200.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        L = C.CDLL(SO_PATH)
        dp, fp, ip = C.POINTER(C.c_double), C.POINTER(C.c_float), C.POINTER(C.c_int)
        L.aloam_default_config.argtypes = [C.POINTER(Config), C.c_int]
        L.aloam_default_config.restype = None
        L.aloam_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
        L.aloam_create_wide.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
        L.aloam_destroy.argtypes = [C.c_void_p]
        L.aloam_strerror.argtypes = [C.c_int]
        L.aloam_strerror.restype = C.c_char_p
        cv = CloudView
        L.aloam_extract_features.argtypes = [C.c_void_p, cv] + [C.POINTER(cv)] * 5
        L.aloam_odometry_set_last.argtypes = [C.c_void_p, cv, cv]
        L.aloam_odometry_register.argtypes = [C.c_void_p, cv, cv, dp, dp, C.POINTER(Stats)]
        L.aloam_map_upload.argtypes = [C.c_void_p, cv, cv]
        L.aloam_map_upload_sharded.argtypes = [C.c_void_p, cv, cv]
        L.aloam_mapping_register.argtypes = [C.c_void_p, cv, cv, dp, C.POINTER(Stats)]
        L.aloam_voxel_filter.argtypes = [C.c_void_p, cv, C.c_float, C.POINTER(cv)]
        L.aloam_mapper_reset.argtypes = [C.c_void_p]
        L.aloam_mapper_step.argtypes = [C.c_void_p, cv, cv, dp, dp, dp, dp, C.POINTER(Stats)]
        L.aloam_mapper_debug_state.argtypes = [C.c_void_p, ip, ip, ip, dp, dp, C.POINTER(C.c_longlong)]
        L.aloam_mapper_debug_cube.argtypes = [C.c_void_p, C.c_int, C.c_int, C.POINTER(cv)]
        L.aloam_mapper_debug_state_lane.argtypes = [C.c_void_p, C.c_int, ip, ip, ip, dp, dp, C.POINTER(C.c_longlong)]
        L.aloam_mapper_debug_cube_lane.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.POINTER(cv)]
        L.aloam_debug_seg_voxel_filter.argtypes = [C.c_void_p, C.POINTER(cv), fp, C.c_int, C.c_int, fp, ip, ip]
        L.aloam_scan_to_pose.argtypes = [C.c_void_p, cv, dp, dp, C.POINTER(Stats)]
        L.aloam_scan_to_pose_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int, dp, dp, C.POINTER(Stats)]
        L.aloam_reset_odometry.argtypes = [C.c_void_p]
        L.aloam_scan_stream.argtypes = [C.c_void_p, C.POINTER(cv), C.c_int, C.c_int, dp, C.POINTER(Stats)]
        L.aloam_scan_stream_batch.argtypes = [C.c_void_p, C.POINTER(cv), C.c_int, C.c_int, C.c_int, dp, C.POINTER(Stats)]
        L.aloam_scan_stream_mapped.argtypes = [C.c_void_p, C.POINTER(cv), C.c_int, C.c_int, dp, dp, C.POINTER(Stats)]
        L.aloam_scan_stream_mapped_batch.argtypes = [C.c_void_p, C.POINTER(cv), C.c_int, C.c_int, C.c_int, dp, dp, C.POINTER(Stats)]
        L.aloam_scan_stream_lanes.argtypes = [C.c_void_p, C.POINTER(cv), ip, C.c_int, C.c_int, C.c_int, dp, dp, C.POINTER(Stats)]
        L.aloam_transform_to_end.argtypes = [C.c_void_p, cv, dp, dp, C.c_int, C.POINTER(cv)]
        L.aloam_knn.argtypes = [C.c_void_p, C.c_int, cv, C.c_int, ip, fp]
        L.aloam_odometry_associate.argtypes = [C.c_void_p, cv, cv, dp, dp, ip, ip]
        L.aloam_normal_equations.argtypes = [C.c_void_p, dp, C.c_int, dp, dp, dp, dp]
        L.aloam_solve.argtypes = [C.c_void_p, dp, C.c_int, dp, dp, dp, C.c_int, ip]
        L.aloam_debug_features.argtypes = [C.c_void_p, fp, ip, ip, ip]
        L.aloam_profile_enable.argtypes = [C.c_void_p, C.c_int]
        L.aloam_profile_read.argtypes = [C.c_void_p, dp, C.POINTER(C.c_longlong), C.POINTER(C.c_char_p), C.c_int]
        L.aloam_launch_count.argtypes = [C.c_void_p]
        L.aloam_launch_count.restype = C.c_longlong
        L.aloam_mapping_associate.argtypes = [C.c_void_p, cv, cv, dp, dp]
        L.aloam_comm_unique_id.argtypes = [C.c_char_p]
        L.aloam_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
        L.aloam_debug_shard_emulate.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        L.aloam_debug_map_sizes.argtypes = [C.c_void_p, ip, ip]
        L.aloam_mapper_export.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
        L.aloam_set_registered_sink.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong]
        L.aloam_registered_rows.argtypes = [C.c_void_p, C.POINTER(C.c_longlong), ip, C.c_int]
        L.aloam_lane_save.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
        L.aloam_lane_restore.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong]
        L.aloam_snapshot_check.argtypes = [C.c_void_p, C.c_longlong, C.POINTER(SnapshotInfo)]
        L.aloam_lane_save_localising.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
        L.aloam_snapshot_localise_info.argtypes = [C.c_void_p, C.c_longlong, dp, C.POINTER(C.c_ulonglong), ip, C.POINTER(C.c_longlong)]
        L.aloam_prior_map_digest.argtypes = [C.c_void_p, C.POINTER(C.c_ulonglong)]
        L.aloam_prior_map_load.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong]
        L.aloam_prior_map_clear.argtypes = [C.c_void_p]
        L.aloam_prior_map_build.argtypes = [C.c_void_p, cv, cv, ip, C.POINTER(C.c_longlong)]
        L.aloam_lane_localise.argtypes = [C.c_void_p, C.c_int, dp, dp]
        L.aloam_lane_map_on_prior.argtypes = [C.c_void_p, C.c_int, dp, dp]
        L.aloam_set_cube_growth.argtypes = [C.c_void_p, C.c_int]
        L.aloam_debug_prior_associate.argtypes = [C.c_void_p, C.c_int, cv, cv, dp, dp]
        L.aloam_prior_relocalise.argtypes = [C.c_void_p, cv, cv, dp, C.c_int, C.POINTER(RelocOpts), ip, C.POINTER(RelocResult)]
        L.aloam_set_map_rows.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_int]
        L.aloam_map_rows.argtypes = [C.c_void_p, C.POINTER(MapRow), C.c_int]
        L.aloam_set_recovery.argtypes = [C.c_void_p, C.c_int, C.POINTER(RecoveryOpts), dp, C.c_int]
        L.aloam_recovery_rows.argtypes = [C.c_void_p, C.POINTER(RecoveryRow), C.c_int]
        L.aloam_debug_recovery_scores.argtypes = [C.c_void_p, C.c_int, ip, C.c_int]
        L.aloam_set_place.argtypes = [C.c_void_p, C.c_int, C.POINTER(PlaceOpts)]
        L.aloam_place_rows.argtypes = [C.c_void_p, C.POINTER(PlaceRow), C.c_int]
        L.aloam_place_keyframes.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
        L.aloam_place_db_load.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.aloam_place_db_clear.argtypes = [C.c_void_p]
        L.aloam_place_describe.argtypes = [C.c_void_p, cv, cv, C.c_void_p]
        L.aloam_place_query.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(PlaceMatch)]
        L.aloam_set_loops.argtypes = [C.c_void_p, C.c_int, C.POINTER(LoopOpts)]
        L.aloam_loop_rows.argtypes = [C.c_void_p, C.POINTER(LoopRow), C.c_int]
        L.aloam_loop_verify.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(LoopRow)]
        L.aloam_place_keyframe_cloud.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.POINTER(C.c_longlong)]
        _LIB = L
    return _LIB


def _check(rc):
    if rc != 0:
        raise AloamError(rc, lib().aloam_strerror(rc).decode())


def _view(a):
    """numpy (n, 4|8) float32 -> CloudView (keeps `a` alive through the returned tuple)."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim != 2 or a.shape[1] not in (4, 8):
        raise ValueError("clouds are (n, 4) or (n, 8) float32")
    return CloudView(a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0], a.shape[1]), a


def _out(v):
    if v.n == 0:
        return np.zeros((0, 4), np.float32)
    return np.ctypeslib.as_array(v.data, shape=(v.n, 4)).copy()


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _views(ptrs, counts, stride):
    """CloudView array over raw scans given as addresses and point counts, in the order of the flattened (scan-major) arrays"""
    ptrs = np.asarray(ptrs, np.uint64).ravel()
    counts = np.asarray(counts, np.int64).ravel()
    views = (CloudView * len(ptrs))()
    for i in range(len(ptrs)):
        views[i] = CloudView(C.cast(C.c_void_p(int(ptrs[i])), C.POINTER(C.c_float)), int(counts[i]), stride)
    return views


def _blob(blob):
    """(address, size in bytes, object to keep alive) of a snapshot: a numpy array, bytes, or a contiguous torch tensor (device
    or host memory)"""
    if hasattr(blob, "data_ptr"):
        if not blob.is_contiguous():
            raise ValueError("a snapshot tensor is contiguous")
        return C.c_void_p(blob.data_ptr()), blob.numel() * blob.element_size(), blob
    a = np.ascontiguousarray(np.frombuffer(blob, np.uint8) if isinstance(blob, (bytes, bytearray)) else blob)
    return C.c_void_p(a.ctypes.data), a.nbytes, a


def snapshot_info(blob):
    """checks a lane snapshot in host memory without a context or a GPU (aloam_snapshot_check) -> {version, mapped, n_scans,
    scan_index, bytes, map_points, world, localising}; a localising snapshot (format version 2) adds t_wmap_wodom (q xyzw, t),
    map_digest, map_centre and map_points_prior (corner, surf) of the prior map it names (aloam_snapshot_localise_info).  Raises
    AloamError(ERR_SNAPSHOT) when it is malformed"""
    ptr, n, keep = _blob(blob)
    info = SnapshotInfo()
    _check(lib().aloam_snapshot_check(ptr, n, C.byref(info)))
    out = {"version": info.version, "mapped": bool(info.mapped), "n_scans": info.n_scans, "scan_index": info.scan_index,
           "bytes": info.bytes, "map_points": info.map_points, "world": np.array(info.world[:]), "localising": info.version == 2}
    if out["localising"]:
        t, digest, centre, points = (C.c_double * 7)(), C.c_ulonglong(0), (C.c_int * 3)(), (C.c_longlong * 2)()
        _check(lib().aloam_snapshot_localise_info(ptr, n, t, C.byref(digest), centre, points))
        out.update({"t_wmap_wodom": np.array(t[:]), "map_digest": int(digest.value), "map_centre": tuple(centre[:]),
                    "map_points_prior": (int(points[0]), int(points[1]))})
    return out


def _cloud_view(a):
    """a cloud argument that may live on the device: a float32 torch tensor (n, 4 | 8), contiguous, in device or host memory,
    or anything numpy takes -> (CloudView, object to keep alive)"""
    if hasattr(a, "data_ptr"):
        if a.dim() != 2 or a.shape[1] not in (4, 8) or a.element_size() != 4 or not a.is_floating_point() or not a.is_contiguous():
            raise ValueError("a cloud tensor is a contiguous (n, 4) or (n, 8) float32 tensor")
        return CloudView(C.cast(C.c_void_p(a.data_ptr()), C.POINTER(C.c_float)), a.shape[0], a.shape[1]), a
    return _view(a)


def snapshot_store_clouds(blob):
    """the cube store of a MAPPED lane snapshot in host memory, split into its two clouds (no context, no GPU): {"corner", "surf":
    (n, 4) float32, each type's cubes in cube order; "centre": the store's centre offsets; "counts": (2, 4851) int32, points per
    corner / surf cube, -1 for a cube without a slab}.  prior_map_build(corner, surf, centre) of a single snapshot's clouds
    rebuilds that store's map; the clouds of several snapshots, moved into one frame and concatenated, make a joined map."""
    import struct
    info = snapshot_info(blob)
    if not info["mapped"]:
        raise ValueError("the snapshot holds no cube store")
    b = np.ascontiguousarray(np.frombuffer(bytes(blob), np.uint8) if isinstance(blob, (bytes, bytearray)) else np.asarray(blob, np.uint8)).ravel()
    nls, nlf = struct.unpack_from("<ii", b, 28)
    s = 256 + 16 * (nls + nlf)   # the store section
    centre = struct.unpack_from("<3i", b, s)
    counts = np.frombuffer(b, np.int32, 2 * 4851, s + 592).reshape(2, 4851).copy()
    n = int(struct.unpack_from("<q", b, s + 39408)[0])
    pts = np.frombuffer(b, np.float32, 4 * n, s + 39424).reshape(n, 4)
    # export order: corner cube i, then surf cube i -- the type of every point, then a stable split
    kind = np.repeat(np.tile(np.array([0, 1], np.int8), 4851), np.maximum(counts, 0).T.ravel())
    return {"corner": pts[kind == 0].copy(), "surf": pts[kind == 1].copy(), "centre": tuple(int(v) for v in centre), "counts": counts}


def pose_grid(q_base, t_centre, half_extent_xy, step_xy, yaws):
    """relocalisation hypotheses, (n, 7) float64 rows (q xyzw, t): every heading yaw of `yaws` (radians; a turn about the map z
    axis applied after q_base) at every point t_centre + (i step_xy, j step_xy, 0) of the square lattice with |i step_xy| and
    |j step_xy| <= half_extent_xy.  Rows run over yaw fastest, then y, then x."""
    q0 = np.asarray(q_base, np.float64)
    t0 = np.asarray(t_centre, np.float64)
    if q0.shape != (4,) or t0.shape != (3,) or not step_xy > 0 or half_extent_xy < 0:
        raise ValueError("q_base is 4 doubles (x, y, z, w), t_centre 3, step_xy > 0, half_extent_xy >= 0")
    k = int(np.floor(half_extent_xy / step_xy + 1e-9))
    offs = np.arange(-k, k + 1) * float(step_xy)
    yaws = np.atleast_1d(np.asarray(yaws, np.float64))
    s, c = np.sin(yaws / 2), np.cos(yaws / 2)   # dq = (0, 0, s, c) times q0
    x, y, z, w = q0
    q = np.stack([c * x - s * y, c * y + s * x, c * z + s * w, c * w - s * z], axis=1)
    n = len(offs) * len(offs) * len(yaws)
    out = np.empty((n, 7))
    out[:, :4] = np.tile(q, (len(offs) * len(offs), 1))
    gx, gy = np.meshgrid(offs, offs, indexing="ij")
    out[:, 4] = np.repeat(t0[0] + gx.ravel(), len(yaws))
    out[:, 5] = np.repeat(t0[1] + gy.ravel(), len(yaws))
    out[:, 6] = t0[2]
    return out


def place_hypotheses(matches, records, half_extent_xy, step_xy, yaw_half, yaw_step):
    """relocalisation hypotheses from place matches: for every match (a dict or structured array with keyframe and shift, as
    Aloam.place_query returns) a pose_grid around q_kf * Rz(shift * 2 pi / 60), t_kf of its keyframe record (records: a
    PLACE_RECORD_DTYPE array, the database the query ran against), with headings yaw_half apart at most in steps of yaw_step
    (radians) -> (n, 7) float64, ready for Aloam.prior_relocalise"""
    kf = np.atleast_1d(np.asarray(matches["keyframe"])).ravel()
    sh = np.atleast_1d(np.asarray(matches["shift"])).ravel()
    k = int(np.floor(yaw_half / yaw_step + 1e-9)) if yaw_step > 0 else 0
    yaws = np.arange(-k, k + 1) * float(yaw_step)
    out = []
    for j, s in zip(kf, sh):
        if j < 0:
            continue
        x, y, z, w = records["pose"][int(j)][:4]
        a = float(s) * 2.0 * np.pi / PLACE_SECTORS
        sz, cz = np.sin(a / 2), np.cos(a / 2)   # q_kf * (0, 0, sz, cz)
        q = np.array([x * cz + y * sz, y * cz - x * sz, z * cz + w * sz, w * cz - z * sz])
        out.append(pose_grid(q, records["pose"][int(j)][4:], half_extent_xy, step_xy, yaws))
    return np.concatenate(out) if out else np.zeros((0, 7))


def default_config(n_scans):
    cfg = Config()
    lib().aloam_default_config(C.byref(cfg), n_scans)
    return cfg


class Aloam:
    """One context = one caller thread = one CUDA stream on one GPU (mirrors `aloam_ctx`)."""

    def __init__(self, n_scans=64, device=0, max_points=None, wide=False, **overrides):
        """wide=True creates the context with aloam_create_wide: driver rings (ring_source=RING_FIELD) up to MAX_RINGS"""
        cfg = default_config(n_scans)
        cfg.device = device
        if max_points is not None:
            cfg.max_points = max_points
        for k, v in overrides.items():
            setattr(cfg, k, v)
        self.cfg = cfg
        self._h = C.c_void_p()
        create = lib().aloam_create_wide if wide else lib().aloam_create
        _check(create(C.byref(cfg), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self._h:
            lib().aloam_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # --- scanRegistration.cpp:129-408
    def extract_features(self, raw):
        v, keep = _view(raw)
        outs = [CloudView() for _ in range(5)]
        _check(lib().aloam_extract_features(self._h, v, *[C.byref(o) for o in outs]))
        names = ["full", "sharp", "less_sharp", "flat", "less_flat"]
        return {n: _out(o) for n, o in zip(names, outs)}

    def debug_features(self, n_full):
        curv = np.zeros(n_full, np.float32)
        label = np.zeros(n_full, np.int32)
        s = np.zeros(MAX_RINGS, np.int32)
        e = np.zeros(MAX_RINGS, np.int32)
        ip = C.POINTER(C.c_int)
        _check(lib().aloam_debug_features(self._h, curv.ctypes.data_as(C.POINTER(C.c_float)), label.ctypes.data_as(ip),
                                          s.ctypes.data_as(ip), e.ctypes.data_as(ip)))
        return curv, label, s[:self.cfg.n_scans], e[:self.cfg.n_scans]

    # --- laserOdometry.cpp:554-568 / :274-502
    def odometry_set_last(self, corner_last, surf_last):
        a, ka = _view(corner_last)
        b, kb = _view(surf_last)
        _check(lib().aloam_odometry_set_last(self._h, a, b))

    def odometry_register(self, sharp, flat, q, t):
        a, ka = _view(sharp)
        b, kb = _view(flat)
        q = np.array(q, np.float64)
        t = np.array(t, np.float64)
        st = Stats()
        _check(lib().aloam_odometry_register(self._h, a, b, _dp(q), _dp(t), C.byref(st)))
        return q, t, st.as_dict()

    def odometry_associate(self, sharp, flat, q, t):
        a, ka = _view(sharp)
        b, kb = _view(flat)
        cc = np.zeros((max(a.n, 1), 3), np.int32)
        pc = np.zeros((max(b.n, 1), 4), np.int32)
        ip = C.POINTER(C.c_int)
        _check(lib().aloam_odometry_associate(self._h, a, b, _dp(np.ascontiguousarray(q, np.float64)),
                                              _dp(np.ascontiguousarray(t, np.float64)), cc.ctypes.data_as(ip), pc.ctypes.data_as(ip)))
        return cc[:a.n], pc[:b.n]

    # --- laserMapping.cpp:531-559 / :554-729
    def map_upload(self, corner_map, surf_map):
        a, ka = _view(corner_map)
        b, kb = _view(surf_map)
        _check(lib().aloam_map_upload(self._h, a, b))

    def map_upload_sharded(self, corner_map, surf_map):
        """the whole submap in, this rank's shard (owned x-slabs + halo) cut out on the device and indexed"""
        a, ka = _view(corner_map)
        b, kb = _view(surf_map)
        _check(lib().aloam_map_upload_sharded(self._h, a, b))

    def map_upload_sharded_ptr(self, corner_ptr, n_corner, surf_ptr, n_surf, stride=4):
        a = CloudView(C.cast(C.c_void_p(int(corner_ptr)), C.POINTER(C.c_float)), int(n_corner), stride)
        b = CloudView(C.cast(C.c_void_p(int(surf_ptr)), C.POINTER(C.c_float)), int(n_surf), stride)
        _check(lib().aloam_map_upload_sharded(self._h, a, b))

    def map_upload_ptr(self, corner_ptr, n_corner, surf_ptr, n_surf, stride=4):
        """aloam_map_upload on raw addresses (pinned host memory or device memory; the library infers the copy kind)"""
        a = CloudView(C.cast(C.c_void_p(int(corner_ptr)), C.POINTER(C.c_float)), int(n_corner), stride)
        b = CloudView(C.cast(C.c_void_p(int(surf_ptr)), C.POINTER(C.c_float)), int(n_surf), stride)
        _check(lib().aloam_map_upload(self._h, a, b))

    # --- map cube store (laserMapping.cpp:309-550,736-801)
    def mapper_reset(self):
        _check(lib().aloam_mapper_reset(self._h))

    def mapper_step(self, corner_last, surf_last, q_wodom_curr, t_wodom_curr):
        """one alaserMapping frame -> (q_w_curr, t_w_curr, stats)"""
        a, ka = _view(corner_last)
        b, kb = _view(surf_last)
        qo = np.ascontiguousarray(q_wodom_curr, np.float64); to = np.ascontiguousarray(t_wodom_curr, np.float64)
        q = np.zeros(4); t = np.zeros(3)
        st = Stats()
        _check(lib().aloam_mapper_step(self._h, a, b, _dp(qo), _dp(to), _dp(q), _dp(t), C.byref(st)))
        return q, t, st.as_dict()

    def mapper_state(self, lane=0):
        """cube-store state of one mapper lane (lane 0: aloam_mapper_step and both mapped stream calls)"""
        cen = (C.c_int * 3)(); nv = C.c_int(0); valid = (C.c_int * 125)(); tot = (C.c_longlong * 2)()
        q = np.zeros(4); t = np.zeros(3)
        _check(lib().aloam_mapper_debug_state_lane(self._h, int(lane), cen, C.byref(nv), valid, _dp(q), _dp(t), tot))
        return {"centre": tuple(cen), "valid": list(valid[:nv.value]), "q_wmap_wodom": q, "t_wmap_wodom": t,
                "total_corner": int(tot[0]), "total_surf": int(tot[1])}

    def mapper_cube(self, which, cube_index, lane=0):
        out = CloudView()
        _check(lib().aloam_mapper_debug_cube_lane(self._h, int(lane), which, cube_index, C.byref(out)))
        return _out(out)

    # --- the clouds the reference mapper publishes (laserMapping.cpp:806-848)
    def mapper_export_size(self, what, lane=0):
        n = C.c_longlong(0)
        _check(lib().aloam_mapper_export(self._h, int(lane), int(what), None, 0, C.byref(n)))
        return n.value

    def mapper_export(self, what, lane=0, out=None):
        """the cube store of `lane` in the reference's order (EXPORT_SURROUND: /laser_cloud_surround, EXPORT_MAP: /laser_cloud_map).
        out=None: returns an (n, 4) float32 numpy array.  out = a float32 torch tensor (CUDA or host) of shape (m, 4): filled in
        place (m >= n points), returns out[:n]."""
        n = C.c_longlong(0)
        if out is None:
            size = self.mapper_export_size(what, lane)
            arr = np.zeros((max(size, 1), 4), np.float32)
            _check(lib().aloam_mapper_export(self._h, int(lane), int(what), arr.ctypes.data, arr.shape[0], C.byref(n)))
            return arr[:n.value]
        if out.dtype.itemsize != 4 or not out.is_contiguous() or out.dim() != 2 or out.shape[1] != 4:
            raise ValueError("out is a contiguous (m, 4) float32 tensor")
        _check(lib().aloam_mapper_export(self._h, int(lane), int(what), C.c_void_p(out.data_ptr()), out.shape[0], C.byref(n)))
        return out[:n.value]

    def set_registered_sink(self, sink):
        """sink: a contiguous (m, 4) float32 torch tensor in device or pinned host memory that receives the registered full-
        resolution cloud of every mapped row of the mapped stream calls (see registered_rows); None turns it off"""
        if sink is None:
            _check(lib().aloam_set_registered_sink(self._h, None, 0))
            self._sink = None
            return
        if not sink.is_contiguous() or sink.dim() != 2 or sink.shape[1] != 4:
            raise ValueError("the sink is a contiguous (m, 4) float32 tensor")
        _check(lib().aloam_set_registered_sink(self._h, C.c_void_p(sink.data_ptr()), sink.shape[0]))
        self._sink = sink   # kept alive while it is set

    def registered_rows(self, rows):
        """(begin, count) of the `rows` = n_scans x batch rows (scan-major) of the last mapped stream call: row r's registered
        cloud is sink[begin[r] : begin[r] + count[r]]"""
        begin = np.zeros(max(rows, 1), np.int64); count = np.zeros(max(rows, 1), np.int32)
        _check(lib().aloam_registered_rows(self._h, begin.ctypes.data_as(C.POINTER(C.c_longlong)), count.ctypes.data_as(C.POINTER(C.c_int)), int(rows)))
        return begin[:rows], count[:rows]

    def set_map_rows(self, on=True, inlier_sq=1.0, max_score_points=0):
        """turns per-row records of the mapped stream calls on or off (aloam_set_map_rows): from the next mapped stream call every row
        records its frame's flags, stats and sizes, and with max_score_points > 0 every localising row its prior-map inlier score
        (at most max_score_points stack points per type, inliers at float d2 < inlier_sq) -- see map_rows"""
        _check(lib().aloam_set_map_rows(self._h, int(on), float(inlier_sq), int(max_score_points)))

    def map_rows(self, rows):
        """the `rows` = n_scans x batch rows (scan-major) of the last mapped stream call (aloam_map_rows), as a dict of numpy arrays:
        kind (ROW_*), err, n_valid, score (-1: not scored), n_score, flags, n_corner_corr, n_plane_corr, lm_iters, accepted_steps,
        init_cost, final_cost, each (rows,); n_sub and n_stack (rows, 2); termination (rows, 4)"""
        out = (MapRow * max(int(rows), 1))()
        _check(lib().aloam_map_rows(self._h, out, int(rows)))
        out = out[:int(rows)]
        d = {k: np.array([getattr(r, k) for r in out], np.int32) for k in ("kind", "err", "n_valid", "score", "n_score")}
        for k in ("n_sub", "n_stack"):
            d[k] = np.array([list(getattr(r, k)) for r in out], np.int32).reshape(-1, 2)
        for k in ("flags", "n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps"):
            d[k] = np.array([getattr(r.stats, k) for r in out], np.int32)
        d["termination"] = np.array([list(r.stats.termination) for r in out], np.int32).reshape(-1, 4)
        for k in ("init_cost", "final_cost"):
            d[k] = np.array([getattr(r.stats, k) for r in out], np.float64)
        return d

    def set_recovery(self, on=True, trigger_frac=0.5, accept_frac=0.75, deltas=None):
        """turns recovery of localising lanes on or off (aloam_set_recovery): from the next mapped stream call a localising row whose
        score is below trigger_frac of its scoring points scores the candidates (q_d * q_P normalised, t_P + t_d) around its map pose
        P for every delta d of `deltas` ((n, 7) float64, q xyzw, t: pose_grid(identity, 0, half, step, yaws) lays out a search), and
        the lane's T_wmap_wodom is re-seated at the best one when it beats the row's score and holds accept_frac of its scoring
        points.  Needs set_map_rows with max_score_points > 0.  on=False turns it off and reads nothing else."""
        if not on:
            _check(lib().aloam_set_recovery(self._h, 0, None, None, 0))
            return
        d = np.ascontiguousarray(deltas, np.float64)
        if d.ndim != 2 or d.shape[1] != 7:
            raise ValueError("deltas are (n, 7) float64 rows (q xyzw, t)")
        o = RecoveryOpts(float(trigger_frac), float(accept_frac))
        _check(lib().aloam_set_recovery(self._h, 1, C.byref(o), _dp(d), d.shape[0]))
        self._n_delta = d.shape[0]

    def recovery_rows(self, rows):
        """what recovery did on the `rows` = n_scans x batch rows (scan-major) of the last mapped stream call (aloam_recovery_rows), as
        a dict of numpy arrays: triggered, best (-1: not triggered), best_score (-1), adopted, each (rows,); pose (rows, 7), the best
        candidate's map pose (zeros when not triggered)"""
        out = (RecoveryRow * max(int(rows), 1))()
        _check(lib().aloam_recovery_rows(self._h, out, int(rows)))
        out = out[:int(rows)]
        d = {k: np.array([getattr(r, k) for r in out], np.int32) for k in ("triggered", "best", "best_score", "adopted")}
        d["pose"] = np.array([list(r.pose) for r in out], np.float64).reshape(-1, 7)
        return d

    def debug_recovery_scores(self, lane):
        """the candidate scores, one per delta of the last set_recovery, of lane `lane`'s latest triggered row of the last mapped
        stream call"""
        n_delta = getattr(self, "_n_delta", 0)
        out = np.zeros(max(int(n_delta), 1), np.int32)
        _check(lib().aloam_debug_recovery_scores(self._h, int(lane), out.ctypes.data_as(C.POINTER(C.c_int)), int(n_delta)))
        return out[:int(n_delta)]

    def seg_voxel_filter(self, segs, leaves, idx_bits=31):
        """the mapper's segmented VoxelGrid over `segs` ((n, 4) float32 clouds, one leaf each) in one pass with `idx_bits`
        voxel-index bits in the sort key -> (list of filtered clouds, error word)"""
        keep = [_view(s) for s in segs]
        n = len(keep)
        views = (CloudView * max(n, 1))(*[v for v, _ in keep])
        lv = np.ascontiguousarray(leaves, np.float32)
        total = sum(v.n for v, _ in keep)
        out = np.zeros((max(total, 1), 4), np.float32)
        counts = np.zeros(max(n, 1), np.int32)
        err = C.c_int(0)
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
        _check(lib().aloam_debug_seg_voxel_filter(self._h, views, lv.ctypes.data_as(fp), n, int(idx_bits), out.ctypes.data_as(fp),
                                                  counts.ctypes.data_as(ip), C.byref(err)))
        res, off = [], 0
        for (v, _), k in zip(keep, counts):
            res.append(out[off:off + k].copy())
            off += v.n
        return res, err.value

    def mapping_register(self, corner_stack, surf_stack, x):
        a, ka = _view(corner_stack)
        b, kb = _view(surf_stack)
        x = np.array(x, np.float64)
        st = Stats()
        _check(lib().aloam_mapping_register(self._h, a, b, _dp(x), C.byref(st)))
        return x, st.as_dict()

    def mapping_associate(self, corner_stack, surf_stack, x):
        """per stack point [query, type (-1 rejected, 0 edge, 2 plane-norm), p0(3), p1(3), d, nn(5)] (corner rows first)"""
        a, ka = _view(corner_stack)
        b, kb = _view(surf_stack)
        fits = np.zeros((max(a.n + b.n, 1), 14))
        _check(lib().aloam_mapping_associate(self._h, a, b, _dp(np.ascontiguousarray(x, np.float64)), _dp(fits)))
        return fits[:a.n + b.n]

    def prior_associate(self, lane, corner_stack, surf_stack, x):
        """mapping_associate against the prior map through the window of `lane`'s latest localising frame; nn(5) are indices in
        the submap a mapping frame would gather from the same store"""
        a, ka = _view(corner_stack)
        b, kb = _view(surf_stack)
        fits = np.zeros((max(a.n + b.n, 1), 14))
        _check(lib().aloam_debug_prior_associate(self._h, int(lane), a, b, _dp(np.ascontiguousarray(x, np.float64)), _dp(fits)))
        return fits[:a.n + b.n]

    # --- multi-GPU map sharding: rank 0 makes the id, everybody joins (ship the id with torch.distributed)
    @staticmethod
    def comm_unique_id():
        buf = C.create_string_buffer(128)
        _check(lib().aloam_comm_unique_id(buf))
        return bytes(buf.raw)

    def comm_init(self, rank, world, unique_id):
        _check(lib().aloam_comm_init(self._h, rank, world, C.create_string_buffer(bytes(unique_id), 128)))

    def debug_shard_emulate(self, rank, world, exchange=0, poison_peer_err=False):
        """test hook: act as rank `rank` of `world` without a communicator, the LM all-reduce a loopback through `exchange`
        (0 k_lm_solve, 1 per-evaluation kernels, 2 one-rank peer mailbox); world = 0 ends the emulation"""
        _check(lib().aloam_debug_shard_emulate(self._h, int(rank), int(world), int(exchange), int(bool(poison_peer_err))))

    def debug_map_sizes(self):
        """(points indexed on this rank, submap size of the thin-map test), each (corner, surf)"""
        kept = (C.c_int * 2)(); glob = (C.c_int * 2)()
        _check(lib().aloam_debug_map_sizes(self._h, kept, glob))
        return (kept[0], kept[1]), (glob[0], glob[1])

    def comm_uses_peer_memory(self):
        lib().aloam_comm_uses_peer_memory.argtypes = [C.c_void_p]
        return bool(lib().aloam_comm_uses_peer_memory(self._h))

    def voxel_filter(self, cloud, leaf):
        a, ka = _view(cloud)
        o = CloudView()
        _check(lib().aloam_voxel_filter(self._h, a, float(leaf), C.byref(o)))
        return _out(o)

    # --- fused device-resident pipeline
    def scan_to_pose(self, raw):
        v, keep = _view(raw)
        q = np.zeros(4)
        t = np.zeros(3)
        st = Stats()
        _check(lib().aloam_scan_to_pose(self._h, v, _dp(q), _dp(t), C.byref(st)))
        return q, t, st.as_dict()

    def scan_to_pose_ptr(self, host_ptr, n, stride=4):
        """raw scan given as a host address (e.g. pinned memory owned by the caller)."""
        v = CloudView(C.cast(host_ptr, C.POINTER(C.c_float)), n, stride)
        q = np.zeros(4)
        t = np.zeros(3)
        st = Stats()
        _check(lib().aloam_scan_to_pose(self._h, v, _dp(q), _dp(t), C.byref(st)))
        return q, t, st

    def scan_to_pose_device(self, dev_ptr, n):
        q = np.zeros(4)
        t = np.zeros(3)
        st = Stats()
        _check(lib().aloam_scan_to_pose_device(self._h, C.c_void_p(dev_ptr), n, _dp(q), _dp(t), C.byref(st)))
        return q, t, st

    def scan_stream(self, ptrs, counts, device_resident, stride=4):
        """pipelined scan_to_pose over a sequence: ptrs = host (or device) addresses of the raw scans; returns (n, 7) poses"""
        n = len(ptrs)
        poses = np.zeros((n, 7))
        st = Stats()
        _check(lib().aloam_scan_stream(self._h, _views(ptrs, counts, stride), n, int(device_resident), _dp(poses), C.byref(st)))
        return poses, st

    def scan_stream_mapped(self, ptrs, counts, device_resident, stride=4):
        """aloam_scan_stream_mapped: odometry + scan-to-map of every scan on the device; returns (odom poses, map poses), (n, 7) each"""
        n = len(ptrs)
        odom = np.zeros((n, 7)); mapped = np.zeros((n, 7))
        st = Stats()
        _check(lib().aloam_scan_stream_mapped(self._h, _views(ptrs, counts, stride), n, int(device_resident), _dp(odom), _dp(mapped), C.byref(st)))
        return odom, mapped

    def scan_stream_batch(self, ptrs, counts, device_resident, stride=4):
        """aloam_scan_stream_batch: ptrs / counts are (n_scans, batch) arrays of addresses / point counts (scan-major);
        returns poses (n_scans, batch, 7).  Every kernel launch covers all `batch` trajectories of a step."""
        ptrs = np.asarray(ptrs, np.uint64)
        n, b = ptrs.shape
        poses = np.zeros((n, b, 7))
        st = (Stats * b)()
        _check(lib().aloam_scan_stream_batch(self._h, _views(ptrs, counts, stride), n, b, int(device_resident), _dp(poses), st))
        self.last_batch_stats = [s.as_dict() for s in st]
        return poses

    def scan_stream_mapped_batch(self, ptrs, counts, device_resident, stride=4):
        """aloam_scan_stream_mapped_batch: ptrs / counts are (n_scans, batch) arrays as for scan_stream_batch; returns
        (odom poses, map poses), (n_scans, batch, 7) each.  Every lane is bit-identical to its solo scan_stream_mapped run."""
        ptrs = np.asarray(ptrs, np.uint64)
        n, b = ptrs.shape
        odom = np.zeros((n, b, 7)); mapped = np.zeros((n, b, 7))
        st = (Stats * b)()
        _check(lib().aloam_scan_stream_mapped_batch(self._h, _views(ptrs, counts, stride), n, b, int(device_resident), _dp(odom), _dp(mapped), st))
        self.last_batch_stats = [s.as_dict() for s in st]
        return odom, mapped

    def scan_stream_lanes(self, ptrs, counts, ops, device_resident, mapped=True, stride=4):
        """aloam_scan_stream_lanes: ptrs / counts / ops are (n_scans, batch) arrays, ops[k, b] one of LANE_IDLE, LANE_SCAN,
        LANE_START (an idle entry's address and count are not read).  Returns (odom poses, map poses), (n_scans, batch, 7)
        each, NaN rows where idle; map poses is None when mapped=False (odometry only)."""
        ptrs = np.asarray(ptrs, np.uint64)
        counts = np.asarray(counts, np.int64)
        ops = np.ascontiguousarray(ops, np.int32)
        n, b = ptrs.shape
        if counts.shape != (n, b) or ops.shape != (n, b):
            raise ValueError("ptrs, counts and ops are (n_scans, batch) arrays")
        odom = np.zeros((n, b, 7))
        out = np.zeros((n, b, 7)) if mapped else None
        st = (Stats * b)()
        _check(lib().aloam_scan_stream_lanes(self._h, _views(ptrs, counts, stride), ops.ctypes.data_as(C.POINTER(C.c_int)), n, b, int(device_resident), _dp(odom),
                                             _dp(out) if mapped else None, st))
        self.last_batch_stats = [s.as_dict() for s in st]
        return odom, out

    def lane_save(self, lane, out=None):
        """snapshot of the trajectory `lane` runs (aloam_lane_save).  out=None: returns it as a numpy uint8 array.  out = a
        contiguous uint8 torch tensor (CUDA, or pinned / pageable host memory) with room for it: written in place, returns
        out[:n] (a 1-D view)."""
        n = C.c_longlong(0)
        if out is None:
            _check(lib().aloam_lane_save(self._h, int(lane), None, 0, C.byref(n)))
            arr = np.zeros(max(n.value, 1), np.uint8)
            _check(lib().aloam_lane_save(self._h, int(lane), arr.ctypes.data, arr.size, C.byref(n)))
            return arr[:n.value]
        if out.element_size() != 1 or not out.is_contiguous():
            raise ValueError("out is a contiguous uint8 tensor")
        _check(lib().aloam_lane_save(self._h, int(lane), C.c_void_p(out.data_ptr()), out.numel(), C.byref(n)))
        return out.view(-1)[:n.value]

    def lane_save_localising(self, lane, out=None):
        """snapshot of the localising trajectory `lane` runs (aloam_lane_save_localising, format version 2: its odometry, its
        T_wmap_wodom and the name of its prior map); `out` and the return value as for lane_save"""
        n = C.c_longlong(0)
        if out is None:
            _check(lib().aloam_lane_save_localising(self._h, int(lane), None, 0, C.byref(n)))
            arr = np.zeros(max(n.value, 1), np.uint8)
            _check(lib().aloam_lane_save_localising(self._h, int(lane), arr.ctypes.data, arr.size, C.byref(n)))
            return arr[:n.value]
        if out.element_size() != 1 or not out.is_contiguous():
            raise ValueError("out is a contiguous uint8 tensor")
        _check(lib().aloam_lane_save_localising(self._h, int(lane), C.c_void_p(out.data_ptr()), out.numel(), C.byref(n)))
        return out.view(-1)[:n.value]

    def lane_restore(self, lane, blob):
        """makes `lane` run the trajectory of a snapshot (aloam_lane_restore): a numpy array, bytes, or a torch tensor"""
        ptr, n, keep = _blob(blob)
        _check(lib().aloam_lane_restore(self._h, int(lane), ptr, n))

    # --- localisation against a prior map
    def prior_map_load(self, blob):
        """makes the cube store of a mapped lane snapshot the context's prior map (aloam_prior_map_load): a numpy array, bytes,
        or a torch tensor"""
        ptr, n, keep = _blob(blob)
        _check(lib().aloam_prior_map_load(self._h, ptr, n))

    def prior_map_build(self, corner, surf, centre=None):
        """makes the prior map from two clouds in the map frame (aloam_prior_map_build): each point binned into its 50 m cube of the
        21 x 21 x 11 buffer around `centre` (the ring buffer's centre offsets, default (10, 10, 5)), every cube voxel-filtered as the
        mapper's re-filter.  Clouds: numpy arrays or float32 torch tensors (device or host), (n, 4) or (n, 8).
        Returns (dropped corner, dropped surf): the points outside the buffer or with a non-finite coordinate."""
        a, ka = _cloud_view(corner)
        b, kb = _cloud_view(surf)
        cen = None if centre is None else (C.c_int * 3)(*(int(v) for v in centre))
        dropped = (C.c_longlong * 2)()
        _check(lib().aloam_prior_map_build(self._h, a, b, cen, dropped))
        return int(dropped[0]), int(dropped[1])

    def prior_map_clear(self):
        _check(lib().aloam_prior_map_clear(self._h))

    def prior_map_digest(self):
        """the 64-bit digest of the prior map (aloam_prior_map_digest; include/aloam_b200.h gives the formula), computed on the
        device on first use and kept with the map"""
        d = C.c_ulonglong(0)
        _check(lib().aloam_prior_map_digest(self._h, C.byref(d)))
        return int(d.value)

    def lane_localise(self, lane, q_init, t_init):
        """arms `lane`: its next LANE_START in a mapped scan_stream_lanes call begins a trajectory that registers against the
        prior map, its T_wmap_wodom starting at (q_init xyzw, t_init)"""
        q = np.ascontiguousarray(q_init, np.float64); t = np.ascontiguousarray(t_init, np.float64)
        if q.shape != (4,) or t.shape != (3,):
            raise ValueError("q_init is 4 doubles (x, y, z, w), t_init 3")
        _check(lib().aloam_lane_localise(self._h, int(lane), _dp(q), _dp(t)))

    def lane_map_on_prior(self, lane, q_init, t_init):
        """arms `lane`: its next LANE_START in a mapped scan_stream_lanes call begins a mapping trajectory on a copy of the prior
        map, its T_wmap_wodom starting at (q_init xyzw, t_init); the prior map itself is never written"""
        q = np.ascontiguousarray(q_init, np.float64); t = np.ascontiguousarray(t_init, np.float64)
        if q.shape != (4,) or t.shape != (3,):
            raise ValueError("q_init is 4 doubles (x, y, z, w), t_init 3")
        _check(lib().aloam_lane_map_on_prior(self._h, int(lane), _dp(q), _dp(t)))

    def set_cube_growth(self, on):
        """turns cube growth on (1) or off (0, the default) for the lanes that start a mapped trajectory from now on (aloam_set_cube_growth):
        a cube whose slab fills moves to a larger run of slabs of the same pool, up to MAX_CUBE_POINTS points, instead of dropping
        points; lane 0 of mapper_step takes the setting at mapper_reset, a restored lane its snapshot's.  Drops every
        lane_map_on_prior arming."""
        _check(lib().aloam_set_cube_growth(self._h, int(on)))

    def prior_relocalise(self, hyps, less_sharp=None, less_flat=None, raw=None, inlier_sq=1.0, max_score_points=1024, refine=1,
                         scores=True):
        """scores the hypotheses hyps ((n, 7): candidate T_wmap_wodom, q xyzw, t) of one scan against the prior map and refines
        the `refine` best with a localising frame each (aloam_prior_relocalise).  The scan is its less_sharp / less_flat clouds, or
        a raw scan (`raw`) whose features are extracted first.  Returns (results, scores): results = `refine` dicts {hyp, score,
        refined_score, flags, pose (7,)} best first, scores = the (n,) int32 coarse scores (None when scores=False)."""
        if raw is not None:
            f = self.extract_features(raw)
            less_sharp, less_flat = f["less_sharp"], f["less_flat"]
        a, ka = _view(less_sharp)
        b, kb = _view(less_flat)
        h = np.ascontiguousarray(hyps, np.float64)
        if h.ndim != 2 or h.shape[1] != 7:
            raise ValueError("hyps is an (n, 7) array of poses (q xyzw, t)")
        opts = RelocOpts(float(inlier_sq), int(max_score_points), int(refine))
        out = (RelocResult * max(int(refine), 1))()
        sc = np.zeros(max(h.shape[0], 1), np.int32) if scores else None
        _check(lib().aloam_prior_relocalise(self._h, a, b, _dp(h), h.shape[0], C.byref(opts),
                                            sc.ctypes.data_as(C.POINTER(C.c_int)) if scores else None, out))
        res = [{"hyp": r.hyp, "score": r.score, "refined_score": r.refined_score, "flags": r.flags, "pose": np.array(r.pose[:])}
               for r in out[:int(refine)]]
        return res, (sc[:h.shape[0]] if scores else None)

    # --- place recognition (Scan Context)
    def set_place(self, on=True, max_range=80.0, z_offset=2.0, keyframe_gap=0.0, exclude_recent=0, max_keyframes=4096):
        """sets the descriptor parameters and turns keyframe recording of the mapped stream calls on or off (aloam_set_place); every
        call clears every lane's keyframe table"""
        o = PlaceOpts(float(max_range), float(z_offset), float(keyframe_gap), int(exclude_recent), int(max_keyframes))
        _check(lib().aloam_set_place(self._h, int(on), C.byref(o)))

    def place_describe(self, less_sharp=None, less_flat=None, raw=None):
        """the (1200,) float32 Scan Context descriptor of one scan (ring-major), from its less_sharp / less_flat clouds or from a raw
        scan whose features are extracted first"""
        if raw is not None:
            f = self.extract_features(raw)
            less_sharp, less_flat = f["less_sharp"], f["less_flat"]
        a, ka = _view(less_sharp)
        b, kb = _view(less_flat)
        out = np.zeros(PLACE_RINGS * PLACE_SECTORS, np.float32)
        _check(lib().aloam_place_describe(self._h, a, b, C.c_void_p(out.ctypes.data)))
        return out

    def place_keyframes(self, lane=0):
        """lane `lane`'s keyframe records (aloam_place_keyframes) as a PLACE_RECORD_DTYPE array"""
        n = C.c_longlong(0)
        _check(lib().aloam_place_keyframes(self._h, int(lane), None, 0, C.byref(n)))
        out = np.zeros(max(n.value, 1), PLACE_RECORD_DTYPE)
        _check(lib().aloam_place_keyframes(self._h, int(lane), C.c_void_p(out.ctypes.data), out.shape[0], C.byref(n)))
        return out[:n.value]

    def place_db_load(self, records):
        """makes `records` (a PLACE_RECORD_DTYPE array, or raw bytes of concatenated records) the context's database"""
        r = np.ascontiguousarray(records if isinstance(records, np.ndarray) else np.frombuffer(records, np.uint8))
        if r.nbytes % 4880:
            raise ValueError("records are 4880 bytes each")
        _check(lib().aloam_place_db_load(self._h, C.c_void_p(r.ctypes.data), r.nbytes // 4880))

    def place_db_clear(self):
        _check(lib().aloam_place_db_clear(self._h))

    def place_query(self, descs, k=1):
        """the k best database keyframes of every descriptor of descs ((n, 1200) float32) -> dict of (n, k) arrays keyframe,
        shift, distance"""
        d = np.ascontiguousarray(descs, np.float32).reshape(-1, PLACE_RINGS * PLACE_SECTORS)
        out = (PlaceMatch * (d.shape[0] * int(k)))()
        _check(lib().aloam_place_query(self._h, C.c_void_p(d.ctypes.data), d.shape[0], int(k), out))
        n = d.shape[0]
        return {"keyframe": np.array([m.keyframe for m in out], np.int32).reshape(n, k),
                "shift": np.array([m.shift for m in out], np.int32).reshape(n, k),
                "distance": np.array([m.distance for m in out], np.float64).reshape(n, k)}

    def place_rows(self, rows):
        """the place rows of the `rows` = n_scans x batch rows (scan-major) of the last mapped stream call (aloam_place_rows) -> dict
        of (rows,) arrays keyframe, loop, shift, full (-1 where there is none) and distance (-1.0)"""
        out = (PlaceRow * max(int(rows), 1))()
        _check(lib().aloam_place_rows(self._h, out, int(rows)))
        out = out[:int(rows)]
        d = {k: np.array([getattr(r, k) for r in out], np.int32) for k in ("keyframe", "loop", "shift", "full")}
        d["distance"] = np.array([r.distance for r in out], np.float64)
        return d

    # --- loop verification
    def set_loops(self, on=True, max_distance=0.3, window=10, cloud_points=1000, outer_iters=4, inlier_sq=1.0):
        """turns loop verification of the mapped stream calls on or off (aloam_set_loops; needs set_place on): every mapped keyframe
        row whose place-row distance is <= max_distance (default 0.3) is registered against the submap of its candidate's keyframes
        within `window` (default 10) on each side, each keyframe keeping at most cloud_points (default 1000) points per type of its
        filtered stacks, in outer_iters (default 4) rounds; the score counts inliers at float d^2 < inlier_sq (default 1.0 m^2).
        Every call clears every lane's keyframe table"""
        o = LoopOpts(float(max_distance), int(window), int(cloud_points), int(outer_iters), float(inlier_sq))
        _check(lib().aloam_set_loops(self._h, int(on), C.byref(o)))

    def loop_rows(self, rows):
        """the loop rows of the `rows` = n_scans x batch rows (scan-major) of the last mapped stream call (aloam_loop_rows) -> list
        of dicts query, cand, verified, shift, n_sub, score, n_score, stats, pose, rel (query / cand / shift -1 where not verified)"""
        out = (LoopRow * max(int(rows), 1))()
        _check(lib().aloam_loop_rows(self._h, out, int(rows)))
        return [r.as_dict() for r in out[:int(rows)]]

    def loop_verify(self, lane, query, cand, shift=None, init=None):
        """one verification (aloam_loop_verify) of keyframe `query` of lane `lane` against the submap of keyframe `cand`: from
        q_cand * Rz(shift * 2 pi / 60), t_cand (shift default 0), or from the pose init (q xyzw, t) when given -> the row's dict"""
        out = LoopRow()
        x = None if init is None else np.ascontiguousarray(init, np.float64)
        if x is not None and x.shape != (7,):
            raise ValueError("init is a pose (q xyzw, t) of 7 doubles")
        _check(lib().aloam_loop_verify(self._h, int(lane), int(query), int(cand), -1 if shift is None and x is not None else int(shift or 0),
                                       None if x is None else _dp(x), C.byref(out)))
        return out.as_dict()

    def keyframe_cloud(self, lane, k):
        """keyframe k's stored clouds of lane `lane` (aloam_place_keyframe_cloud; loops on) -> (corner, surf), (n, 4) float32"""
        n = (C.c_longlong * 2)()
        _check(lib().aloam_place_keyframe_cloud(self._h, int(lane), int(k), None, 0, n))
        out = np.zeros((max(n[0] + n[1], 1), 4), np.float32)
        _check(lib().aloam_place_keyframe_cloud(self._h, int(lane), int(k), C.c_void_p(out.ctypes.data), out.shape[0], n))
        return out[:n[0]].copy(), out[n[0]:n[0] + n[1]].copy()

    def transform_to_end(self, cloud, q, t, distortion=True):
        v, keep = _view(cloud)
        o = CloudView()
        _check(lib().aloam_transform_to_end(self._h, v, _dp(np.ascontiguousarray(q, np.float64)), _dp(np.ascontiguousarray(t, np.float64)),
                                            int(distortion), C.byref(o)))
        return _out(o)

    def reset_odometry(self):
        _check(lib().aloam_reset_odometry(self._h))

    # --- measurement hooks
    def profile_enable(self, on=True):
        _check(lib().aloam_profile_enable(self._h, int(on)))

    def profile_read(self):
        """{kernel name: (total ms, launches)} measured with CUDA events on the ctx stream"""
        ms = (C.c_double * 32)()
        cnt = (C.c_longlong * 32)()
        names = (C.c_char_p * 32)()
        n = lib().aloam_profile_read(self._h, ms, cnt, names, 32)
        return {names[k].decode(): (ms[k], cnt[k]) for k in range(n) if names[k] and cnt[k] > 0}

    def launch_count(self):
        return int(lib().aloam_launch_count(self._h))

    # --- fine-grained
    def knn(self, which, queries, k):
        v, keep = _view(queries)
        idx = np.zeros((v.n, k), np.int32)
        sqd = np.zeros((v.n, k), np.float32)
        _check(lib().aloam_knn(self._h, which, v, k, idx.ctypes.data_as(C.POINTER(C.c_int)), sqd.ctypes.data_as(C.POINTER(C.c_float))))
        return idx, sqd

    def normal_equations(self, blocks, x):
        blocks = np.ascontiguousarray(blocks, np.float64).reshape(-1, BLOCK_DOUBLES)
        JtJ = np.zeros((6, 6))
        Jtr = np.zeros(6)
        cost = C.c_double(0)
        _check(lib().aloam_normal_equations(self._h, _dp(blocks), blocks.shape[0], _dp(np.ascontiguousarray(x, np.float64)),
                                            _dp(JtJ), _dp(Jtr), C.byref(cost)))
        return JtJ, Jtr, cost.value

    def solve(self, blocks, x):
        blocks = np.ascontiguousarray(blocks, np.float64).reshape(-1, BLOCK_DOUBLES)
        x = np.array(x, np.float64)
        s = np.zeros(7)
        trace = np.zeros((8, 8))
        rows = C.c_int(0)
        _check(lib().aloam_solve(self._h, _dp(blocks), blocks.shape[0], _dp(x), _dp(s), _dp(trace), 8, C.byref(rows)))
        keys = ["termination", "num_iterations", "num_successful", "num_jac_evals", "num_cost_evals", "initial_cost", "final_cost"]
        return x, dict(zip(keys, s)), trace[:rows.value]
