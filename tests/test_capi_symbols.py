"""CPU: the C-ABI shared library loads without a GPU and exports every entry point the headers under include/ declare."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    names = set()
    inc = os.path.join(ROOT, "include")
    for h in sorted(os.listdir(inc)):
        if h.endswith(".h"):
            src = re.sub(r"/\*.*?\*/", "", open(os.path.join(inc, h)).read(), flags=re.S)
            names |= set(re.findall(r"\b(aloam_[a-z_0-9]+)\s*\(", src))
    return sorted(names)


def test_header_symbols_exported(aloam):
    assert os.path.exists(aloam.SO_PATH), "run __graft_entry__.build() first"
    lib = ctypes.CDLL(aloam.SO_PATH)
    names = _declared()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), n
    assert set(aloam.EXPORTED_SYMBOLS) <= set(names)


def test_default_config_matches_launch_files(aloam):
    c = aloam.default_config(64)    # launch/aloam_velodyne_HDL_64.launch:3-13
    assert (c.n_scans, c.minimum_range, round(c.line_res, 3), round(c.plane_res, 3)) == (64, 5.0, 0.4, 0.8)
    c = aloam.default_config(16)    # launch/aloam_velodyne_VLP_16.launch:3-13
    assert (c.n_scans, round(c.minimum_range, 3), round(c.line_res, 3), round(c.plane_res, 3)) == (16, 0.3, 0.2, 0.4)
    assert (c.outer_iters, c.inner_iters, c.huber, c.dist_sq_thresh, c.nearby_scan) == (2, 4, 0.1, 25.0, 2.5)


def test_no_cpu_fallback(aloam):
    """without a CUDA device the product refuses to create a context (it never routes through the oracle)"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(aloam.AloamError) as e:
        aloam.Aloam(n_scans=16)
    assert e.value.code in (-5, -6)
    assert aloam.lib().aloam_strerror(-6).decode() == "no CUDA device"


def test_map_capacity_above_2_30_is_rejected_before_the_device(aloam):
    """the map's hash-grid slot count (next power of two above 1.25 x max_map_points) must fit 32 bits: a larger
    max_map_points is an invalid argument, reported before any device is queried"""
    with pytest.raises(aloam.AloamError) as e:
        aloam.Aloam(n_scans=16, max_map_points=2**30 + 1)
    assert e.value.code == -1


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "a-loam_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "pyoracle" not in txt and "liboracle" not in txt and "oracle/" not in txt, f
