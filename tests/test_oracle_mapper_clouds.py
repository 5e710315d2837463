"""CPU: the clouds the reference's own laserMapping.cpp publishes (/laser_cloud_surround every 5th frame, /laser_cloud_map every
20th, /velodyne_cloud_registered every frame; laserMapping.cpp:806-848) equal the oracle's cube store and pointAssociateToMap bit
for bit over 21 VLP-16 frames.  The reference driver (oracle/ref_clouds.mk) is built where /root/reference exists; elsewhere the
prebuilt file is used, or the test skips."""
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import pyclouds

from refsource import NCUBE, REF_DIR, ROOT, RefMapping

SURROUND, MAP, REGISTERED = "/laser_cloud_surround", "/laser_cloud_map", "/velodyne_cloud_registered"


def _clouds_driver(tag):
    name = "libref_mapping_clouds.so"
    if os.path.isdir("/root/reference/src"):
        r = subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "ref_clouds.mk", "_ref/" + name], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
    src = os.path.join(REF_DIR, name)
    if not os.path.exists(src):
        pytest.skip("oracle/_ref/%s is not built and /root/reference is not present" % name)
    path = os.path.join(tempfile.mkdtemp(prefix="ref_"), name.replace(".so", "_%s.so" % tag))
    shutil.copy(src, path)
    lib = C.CDLL(path)
    lib.ref_map_published_cloud.argtypes = [C.c_char_p, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int)]
    lib.ref_map_published_cloud.restype = C.c_long
    return lib


def published(lib, topic):
    """(messages published on `topic` so far, the last one as an (n, 4) float32 array)"""
    n = C.c_int(0)
    lib.ref_map_published_cloud(topic.encode(), None, 0, C.byref(n))
    out = np.zeros((max(n.value, 1), 4), np.float32)
    count = lib.ref_map_published_cloud(topic.encode(), out.ctypes.data_as(C.POINTER(C.c_float)), n.value, C.byref(n))
    return count, out[:n.value]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32).tobytes()


def _oracle_order(cm, idx):
    clouds = [cm.cube(ty, i) for i in idx for ty in (0, 1)]
    clouds = [c for c in clouds if len(c)]
    return np.concatenate(clouds) if clouds else np.zeros((0, 4), np.float32)


def test_associate_to_map_is_the_eigen_transform(orc):
    """orc_associate_to_map: q * p + t in double in Eigen's operation order, stored as float, intensity kept"""
    rng = np.random.default_rng(5)
    cloud = (rng.normal(size=(500, 4)) * [40, 40, 5, 10]).astype(np.float32)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    x = np.concatenate([q, [12.5, -3.25, 0.75]])
    got = pyclouds.associate_to_map(x, cloud)
    v = cloud[:, :3].astype(np.float64)
    u, w = q[:3], q[3]
    uv = np.cross(u, v); uv = uv + uv
    want = ((v + w * uv) + np.cross(u, uv)) + x[4:]
    assert np.array_equal(got[:, :3], want.astype(np.float32)) and np.array_equal(got[:, 3], cloud[:, 3])
    assert pyclouds.associate_to_map(x, np.zeros((0, 4), np.float32)).shape == (0, 4)


def test_reference_published_clouds_equal_the_oracle(orc, synth):
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    lib = _clouds_driver("published")
    ref = RefMapping(lib, 0.2, 0.4, orc.SORT_CANONICAL)
    cm = orc.CubeMap()
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    checked = {SURROUND: 0, MAP: 0}
    for k in range(21):
        f = orc.Features(synth.scan("VLP-16", k, n_az=900), ns, mr, mode=orc.SORT_CANONICAL)
        if k > 0:
            q, t, _ = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
        od.set_last(f.less_sharp, f.less_flat)
        pose, _ = cm.step(f.less_sharp, f.less_flat, qw, tw, 0.2, 0.4, sort_mode=orc.SORT_CANONICAL)
        got = ref.process(f.less_sharp, f.less_flat, f.full, qw, tw, stamp=0.1 * (k + 1))
        assert np.array_equal(got["pose"], pose), k
        n_reg, reg = published(lib, REGISTERED)
        assert n_reg == k + 1 and len(reg) == len(f.full) > 0
        assert _bits(reg) == _bits(pyclouds.associate_to_map(pose, f.full)), k
        n_sur, sur = published(lib, SURROUND)
        assert n_sur == k // 5 + 1
        if k % 5 == 0:
            assert len(sur) > 0 and _bits(sur) == _bits(_oracle_order(cm, cm.state()["valid"])), k
            checked[SURROUND] += 1
        n_map, mp = published(lib, MAP)
        assert n_map == k // 20 + 1
        if k % 20 == 0:
            assert len(mp) >= len(sur) and _bits(mp) == _bits(_oracle_order(cm, range(NCUBE))), k
            checked[MAP] += 1
    assert checked == {SURROUND: 5, MAP: 2}
