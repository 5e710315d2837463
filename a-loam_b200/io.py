"""ctypes mirror of include/aloam_io.h: KITTI .bin scans / pose files and PointCloud2 payloads of pcl::PointXYZI
(kittiHelper.cpp:25-35,78-80,97-113,140-151).  Host-side only -- usable without a GPU."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(os.path.join(_HERE, "libaloam_b200.so"))
        L.aloam_io_kitti_bin_points.restype = C.c_long
        L.aloam_io_kitti_bin_points.argtypes = [C.c_char_p]
        L.aloam_io_read_kitti_bin.restype = C.c_long
        L.aloam_io_read_kitti_bin.argtypes = [C.c_char_p, C.POINTER(C.c_float), C.c_long]
        L.aloam_io_parse_kitti_pose.argtypes = [C.c_char_p, C.POINTER(C.c_double)]
        L.aloam_io_kitti_pose_to_lidar.argtypes = [C.POINTER(C.c_double)] * 3
        L.aloam_io_kitti_pose_to_lidar.restype = None
        L.aloam_io_lidar_pose_to_kitti.argtypes = [C.POINTER(C.c_double)] * 3
        L.aloam_io_lidar_pose_to_kitti.restype = None
        L.aloam_io_pack_pointxyzi.argtypes = [C.POINTER(C.c_float), C.c_long, C.POINTER(C.c_ubyte)]
        L.aloam_io_pack_pointxyzi.restype = None
        L.aloam_io_unpack_points.argtypes = [C.POINTER(C.c_ubyte), C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float)]
        L.aloam_io_unpack_points_ring.argtypes = [C.POINTER(C.c_ubyte), C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                                  C.POINTER(C.c_float)]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def read_kitti_bin(path):
    """(n, 4) float32 x, y, z, intensity -- ready for Aloam.scan_to_pose / scan_stream (stride 4)"""
    n = _lib().aloam_io_kitti_bin_points(os.fsencode(path))
    if n < 0:
        raise OSError("cannot open %s" % path)
    out = np.zeros((n, 4), np.float32)
    got = _lib().aloam_io_read_kitti_bin(os.fsencode(path), out.ctypes.data_as(C.POINTER(C.c_float)), n)
    if got != n:
        raise OSError("short read on %s" % path)
    return out


def write_kitti_bin(path, xyzi):
    np.ascontiguousarray(xyzi, np.float32).tofile(path)


def parse_kitti_pose(line):
    """one line of a KITTI poses file -> (3, 4) float64, every number read through float like the reference's stof()"""
    T = np.zeros(12)
    if _lib().aloam_io_parse_kitti_pose(line.encode(), _dp(T)) != 0:
        raise ValueError("not a KITTI pose line: %r" % line[:60])
    return T.reshape(3, 4)


def kitti_pose_to_lidar(T):
    """camera-frame 3x4 -> (q xyzw, t) in the lidar frame as kittiHelper publishes /odometry_gt"""
    T = np.ascontiguousarray(T, np.float64).reshape(12)
    q = np.zeros(4); t = np.zeros(3)
    _lib().aloam_io_kitti_pose_to_lidar(_dp(T), _dp(q), _dp(t))
    return q, t


def lidar_pose_to_kitti(q, t):
    q = np.ascontiguousarray(q, np.float64); t = np.ascontiguousarray(t, np.float64)
    T = np.zeros(12)
    _lib().aloam_io_lidar_pose_to_kitti(_dp(q), _dp(t), _dp(T))
    return T.reshape(3, 4)


def pack_pointxyzi(xyzi):
    """PointCloud2 `data` bytes of a pcl::PointCloud<pcl::PointXYZI> (point_step 32)"""
    a = np.ascontiguousarray(xyzi, np.float32)
    out = np.zeros(32 * len(a), np.uint8)
    _lib().aloam_io_pack_pointxyzi(a.ctypes.data_as(C.POINTER(C.c_float)), len(a), out.ctypes.data_as(C.POINTER(C.c_ubyte)))
    return out


def unpack_points(data, n, point_step=32, off_x=0, off_y=4, off_z=8, off_intensity=16):
    d = np.ascontiguousarray(data, np.uint8)
    if len(d) < n * point_step:
        raise ValueError("payload shorter than n * point_step")
    out = np.zeros((n, 4), np.float32)
    rc = _lib().aloam_io_unpack_points(d.ctypes.data_as(C.POINTER(C.c_ubyte)), n, point_step, off_x, off_y, off_z, off_intensity,
                                       out.ctypes.data_as(C.POINTER(C.c_float)))
    if rc != 0:
        raise ValueError("bad PointCloud2 layout")
    return out


RING_UINT8, RING_UINT16 = 2, 4   # sensor_msgs/PointField datatypes of a driver's ring field


def unpack_points_ring(data, n, point_step, off_x, off_y, off_z, off_ring, ring_type):
    """(n, 4) float32 x, y, z, ring from a PointCloud2 payload with a ring field (ring_type RING_UINT8 or RING_UINT16): the raw
    scan of a context with ring_source = RING_FIELD"""
    d = np.ascontiguousarray(data, np.uint8)
    if len(d) < n * point_step:
        raise ValueError("payload shorter than n * point_step")
    out = np.zeros((n, 4), np.float32)
    rc = _lib().aloam_io_unpack_points_ring(d.ctypes.data_as(C.POINTER(C.c_ubyte)), n, point_step, off_x, off_y, off_z, off_ring,
                                            ring_type, out.ctypes.data_as(C.POINTER(C.c_float)))
    if rc != 0:
        raise ValueError("bad PointCloud2 layout or ring type")
    return out
