"""Helpers of the mapping_skip_frame tests (tests/test_oracle_mapping_skip.py, tests/test_gpu_mapping_skip.py): the oracle chain
with a skip parameter, and drivers of the reference's laserOdometry / laserMapping sources for a sequence of scans.
TEST INFRASTRUCTURE."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from refsource import REF_DIR, ROOT

_F32P, _F64P = C.POINTER(C.c_float), C.POINTER(C.c_double)
_CHAIN = {}


def mapped(j, skip):
    """scan j of a trajectory goes to the mapper (laserOdometry.cpp:570, frameCount % skipFrameNum == 0)"""
    return j % skip == 0


def oracle_chain(orc, synth, scans, skip, key, sensor="VLP-16", sort_mode=None, leaves=None):
    """the oracle's ascanRegistration | alaserOdometry | alaserMapping with mapping_skip_frame = skip: a mapped scan is one
    CubeMap.step (/aft_mapped_to_init), any other scan gets transform_associate_to_map with the T_wmap_wodom of the latest
    mapped scan (/aft_mapped_to_init_high_frec, laserMapping.cpp:214-215).  Returns (odometry poses, map poses), (n, 7) each;
    cached under (key, skip, sort_mode, leaves, n)."""
    sort_mode = orc.SORT_CANONICAL if sort_mode is None else sort_mode
    ck = (key, skip, sort_mode, leaves, len(scans))
    if ck not in _CHAIN:
        ns, _, mr, line_res, plane_res = synth.SENSORS[sensor]
        if leaves is not None:
            line_res, plane_res = leaves
        od, cm = orc.Odometry(), orc.CubeMap()
        q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
        odom, mp = [], []
        for j, raw in enumerate(scans):
            f = orc.Features(raw, ns, mr, mode=sort_mode)
            if j > 0:
                q, t, _ = od.register(f.sharp, f.flat, q, t)
                qw, tw = orc.integrate_pose(qw, tw, q, t)
            od.set_last(f.less_sharp, f.less_flat)
            odom.append(np.concatenate([qw, tw]))
            if mapped(j, skip):
                pose, _ = cm.step(f.less_sharp, f.less_flat, qw, tw, line_res, plane_res, sort_mode=sort_mode)
            else:
                s = cm.state()
                pose = orc.transform_associate_to_map(s["q_wmap_wodom"], s["t_wmap_wodom"], qw, tw)
            mp.append(pose)
        _CHAIN[ck] = (np.array(odom), np.array(mp))
    return _CHAIN[ck]


def skip_driver(name, tag):
    """a private copy of oracle/_ref/<name>, one of the drivers of oracle/ref_skip.mk (libref_odometry_seq.so,
    libref_mapping_skip.so): built where /root/reference exists, the prebuilt file elsewhere, the test skipped if there is none"""
    if os.path.isdir("/root/reference/src"):
        r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "ref_skip.mk", "_ref/" + name], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    src = os.path.join(REF_DIR, name)
    if not os.path.exists(src):
        pytest.skip("oracle/_ref/%s is not built and /root/reference is not present" % name)
    path = os.path.join(tempfile.mkdtemp(prefix="ref_"), name.replace(".so", "_%s.so" % tag))
    shutil.copy(src, path)
    return C.CDLL(path)


class RefOdometrySequence:
    """the reference's laserOdometry.cpp with mapping_skip_frame = skip, a whole sequence in one entry of its main()
    (lib: libref_odometry_seq.so)"""

    def __init__(self, lib, skip):
        self.lib = lib
        lib.ref_odom_init.argtypes = [C.c_int]
        lib.ref_odom_queue.argtypes = [_F32P, C.c_int] * 5 + [C.c_double]
        lib.ref_odom_run_queued.argtypes = [C.c_int]
        lib.ref_odom_turn.argtypes = [C.c_int, _F64P]
        lib.ref_odom_turn_cloud.argtypes = [C.c_int, C.c_int, _F32P, C.c_int]
        lib.ref_odom_init(int(skip))
        self.queued = 0

    def queue(self, f, stamp):
        args = []
        for x in (f["sharp"], f["less_sharp"], f["flat"], f["less_flat"], f["full"]):
            x = np.ascontiguousarray(x, np.float32)
            args += [x.ctypes.data_as(_F32P), x.shape[0]]
        self.lib.ref_odom_queue(*args, float(stamp))
        self.queued += 1

    def run(self):
        """every queued scan, one turn each -> per turn {pose (7), clouds: None or (corner_last, surf_last, full)}"""
        n = self.lib.ref_odom_run_queued(self.queued)
        assert n == self.queued, (n, self.queued)
        out = []
        for i in range(n):
            pose = np.zeros(7)
            pub = self.lib.ref_odom_turn(i, pose.ctypes.data_as(_F64P))
            assert pub in (0, 1)
            clouds = None
            if pub:
                clouds = []
                for w in range(3):
                    m = self.lib.ref_odom_turn_cloud(i, w, None, 0)
                    a = np.zeros((m, 4), np.float32)
                    if m:
                        self.lib.ref_odom_turn_cloud(i, w, a.ctypes.data_as(_F32P), m)
                    clouds.append(a)
            out.append({"pose": pose, "clouds": clouds})
        return out


def ref_map_odometry_only(mapping, q, t, stamp):
    """one odometry message without clouds into the reference's laserMapping (a RefMapping over libref_mapping_skip.so): the
    high-frequency pose it publishes and the number of such messages so far"""
    lib = mapping.lib
    lib.ref_map_odometry_only.argtypes = [_F64P, _F64P, C.c_double]
    lib.ref_map_high_frec_pose.argtypes = [_F64P, _F64P]
    lib.ref_map_high_frec_pose.restype = C.c_long
    q = np.ascontiguousarray(q, np.float64); t = np.ascontiguousarray(t, np.float64)
    lib.ref_map_odometry_only(q.ctypes.data_as(_F64P), t.ctypes.data_as(_F64P), float(stamp))
    pq, pt = np.zeros(4), np.zeros(3)
    n = lib.ref_map_high_frec_pose(pq.ctypes.data_as(_F64P), pt.ctypes.data_as(_F64P))
    return np.concatenate([pq, pt]), n
