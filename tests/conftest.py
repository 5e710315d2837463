import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def load_pkg():
    return importlib.import_module("a-loam_b200")


def load_synth():
    return importlib.import_module("a-loam_b200.synth")


@pytest.fixture(scope="session")
def synth():
    return load_synth()


@pytest.fixture(scope="session")
def orc():
    import pyoracle
    pyoracle.lib()
    return pyoracle


@pytest.fixture(scope="session")
def aloam():
    return load_pkg()


_SCAN_CACHE = {}


@pytest.fixture(scope="session")
def scans(synth):
    """scans(sensor, index, n_az=None) -> raw (n,4) float32, cached for the session."""
    def get(sensor, index, n_az=None):
        key = (sensor, index, n_az)
        if key not in _SCAN_CACHE:
            _SCAN_CACHE[key] = synth.scan(sensor, index, n_az=n_az)
        return _SCAN_CACHE[key]
    return get


def ulp_diff(a, b):
    """elementwise distance in float32 ulps"""
    a = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.ascontiguousarray(b, np.float32).view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def rot_angle(q1, q2):
    d = abs(float(np.dot(q1, q2)))
    return 2.0 * np.arccos(min(1.0, d))
