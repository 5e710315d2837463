"""ctypes binding of oracle/libclouds.so: the oracle's restatements behind the clouds alaserMapping publishes
(laserMapping.cpp:806-848).  ORACLE = test infrastructure, like pyoracle."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "libclouds.so")
        if not os.path.exists(so):
            subprocess.check_call(["make", "-C", _HERE, "-f", "clouds.mk", "libclouds.so"], stdout=subprocess.DEVNULL)
        L = C.CDLL(so)
        L.orc_associate_to_map.argtypes = [_f64p, _f32p, C.c_int, _f32p]
        L.orc_associate_to_map.restype = None
        _LIB = L
    return _LIB


def associate_to_map(x7, cloud):
    """laserMapping.cpp:154-163 (pointAssociateToMap) over an (n, 4) cloud with parameters[7] = x7 -> (n, 4) float32"""
    c = np.ascontiguousarray(cloud, np.float32)
    assert c.ndim == 2 and c.shape[1] == 4, c.shape
    out = np.zeros((max(c.shape[0], 1), 4), np.float32)
    lib().orc_associate_to_map(np.ascontiguousarray(x7, np.float64).ctypes.data_as(_f64p), c.ctypes.data_as(_f32p), c.shape[0],
                               out.ctypes.data_as(_f32p))
    return out[:c.shape[0]]
