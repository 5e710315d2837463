"""CPU: the localising lane snapshot (include/aloam_b200.h, "Snapshot format, version 2").  Blobs are written here from the documented
layout alone and checked by aloam_snapshot_check and aloam_snapshot_localise_info, which need neither a context nor a GPU: well-formed
snapshots are accepted and described; every kind of corruption is refused with ALOAM_ERR_SNAPSHOT; version-1 snapshots are not
localising ones."""
import ctypes as C
import struct

import numpy as np
import pytest

ERR_INVALID_ARG, ERR_SNAPSHOT = -1, -11
SECTION = 128
T_GOOD = (0.0, 0.0, 0.2, 0.98, 12.5, -3.0, 0.75)   # T_wmap_wodom: q (not normalised: the lane's own bits), t
DIGEST = 0xF00DFACE12345678


def _points(n, seed):
    p = np.random.default_rng(seed).uniform(-20, 20, (n, 4)).astype(np.float32)
    p[:, 3] = np.sort(np.random.default_rng(seed).integers(0, 16, n)) + 0.05
    return p.tobytes()


def _blob(nls=40, nlf=90, scan_index=6, T=T_GOOD, world=(0.0, 0.0, 0.1, 0.995, 3.0, -1.0, 0.25), centre=(10, 10, 5),
          points=(1234, 56789), digest=DIGEST, mapped=0, version=2, growth=0, magic=b"ALOAMLS1", total_delta=0):
    h = bytearray(256)
    body = _points(nls, 1) + _points(nlf, 2)
    total = 256 + len(body) + SECTION + total_delta
    h[0:8] = magic
    struct.pack_into("<iiq", h, 8, version, mapped, total)
    struct.pack_into("<iii", h, 24, scan_index, nls, nlf)
    struct.pack_into("<iiiiifff", h, 36, 16, 0, 1, 2, 4, 0.3, 0.2, 0.4)
    struct.pack_into("<iii", h, 68, 16384, 65536, 400000)
    struct.pack_into("<ddd", h, 80, 0.1, 25.0, 2.5)
    struct.pack_into("<7d", h, 104, 0, 0, 0, 1, 0.5, 0, 0)
    struct.pack_into("<7d", h, 160, *world)
    struct.pack_into("<ii", h, 216, 0, growth)
    s = bytearray(SECTION)
    struct.pack_into("<4d", s, 0, *T[:4])
    struct.pack_into("<3d", s, 32, *T[4:])
    struct.pack_into("<Q", s, 56, digest)
    struct.pack_into("<3i", s, 64, *centre)
    struct.pack_into("<2q", s, 80, *points)
    return bytes(h) + body + bytes(s)


def _v1(nls=4, nlf=9):
    """an unmapped version-1 snapshot (the layout of tests/test_lane_snapshot_format.py)"""
    b = bytearray(_blob(nls, nlf)[:256 + 16 * (nls + nlf)])
    struct.pack_into("<iiq", b, 8, 1, 0, len(b))
    return bytes(b)


def _code(aloam, blob, n=None):
    a = np.frombuffer(blob, np.uint8)
    return aloam.lib().aloam_snapshot_check(C.c_void_p(a.ctypes.data), len(blob) if n is None else n, None)


def _loc_info(aloam, blob):
    a = np.frombuffer(blob, np.uint8)
    t, d, cen, pts = (C.c_double * 7)(), C.c_ulonglong(0), (C.c_int * 3)(), (C.c_longlong * 2)()
    rc = aloam.lib().aloam_snapshot_localise_info(C.c_void_p(a.ctypes.data), len(blob), t, C.byref(d), cen, pts)
    return rc, (list(t), d.value, tuple(cen), tuple(pts))


def test_well_formed_localising_snapshots_are_described(aloam):
    b = _blob()
    info = aloam.snapshot_info(b)
    assert info["version"] == 2 and not info["mapped"] and info["localising"] and info["map_points"] == 0
    assert info["n_scans"] == 16 and info["scan_index"] == 6 and info["bytes"] == len(b) == 256 + 16 * 130 + 128
    assert np.array_equal(info["world"], [0.0, 0.0, 0.1, 0.995, 3.0, -1.0, 0.25])
    assert np.array_equal(info["t_wmap_wodom"], T_GOOD) and info["map_digest"] == DIGEST
    assert info["map_centre"] == (10, 10, 5) and info["map_points_prior"] == (1234, 56789)
    rc, (t, d, cen, pts) = _loc_info(aloam, b)
    assert rc == 0 and t == list(T_GOOD) and d == DIGEST and cen == (10, 10, 5) and pts == (1234, 56789)
    # empty "last" clouds, a far but finite map position, extreme centre offsets, a digest with the top bit set
    for blob in (_blob(nls=0, nlf=0), _blob(T=(0, 0, 0, 1.0, 1e9, -1e9, 0)), _blob(centre=(-(1 << 20), 1 << 20, 0)), _blob(digest=2**64 - 1)):
        assert _code(aloam, blob) == 0
    assert aloam.snapshot_info(_blob(digest=2**64 - 1))["map_digest"] == 2**64 - 1
    # every output of aloam_snapshot_localise_info may be NULL
    a = np.frombuffer(b, np.uint8)
    assert aloam.lib().aloam_snapshot_localise_info(C.c_void_p(a.ctypes.data), len(b), None, None, None, None) == 0
    # a version-1 snapshot is described as before, not localising
    v1 = aloam.snapshot_info(_v1())
    assert v1["version"] == 1 and not v1["localising"] and "t_wmap_wodom" not in v1


def test_corruptions_are_refused(aloam):
    good = _blob()
    assert _code(aloam, good) == 0
    S = 256 + 16 * 130
    bad = {
        "size 16 over": _blob(total_delta=16),
        "size 16 under": _blob(total_delta=-16),
        "mapped 1": _blob(mapped=1),
        "cube_growth 1": _blob(growth=1),
        "version 3": _blob(version=3),
        "magic ALOAMLS2": _blob(magic=b"ALOAMLS2"),
        "NaN quaternion": _blob(T=(0, np.nan, 0, 1.0, 0, 0, 0)),
        "infinite quaternion": _blob(T=(0, 0, np.inf, 1.0, 0, 0, 0)),
        "zero quaternion": _blob(T=(0, 0, 0, 0.0, 1, 2, 3)),
        "NaN translation": _blob(T=(0, 0, 0, 1.0, 0, np.nan, 0)),
        "infinite translation": _blob(T=(0, 0, 0, 1.0, 0, 0, -np.inf)),
        "map position beyond int": _blob(T=(0, 0, 0, 1.0, 50.0 * 2**31, 0, 0)),
        "map position beyond int, negative": _blob(T=(0, 0, 0, 1.0, 0, -50.0 * 2**31 - 100, 0)),
        "centre cube beyond int": _blob(T=(0, 0, 0, 1.0, 50.0 * (2**31 - 10), 0, 0), centre=(1000, 10, 5)),
        "centre offset beyond 2^20": _blob(centre=(10, (1 << 20) + 1, 5)),
        "negative point count": _blob(points=(-1, 5)),
        "non-finite world pose": _blob(world=(0, 0, 0, 1.0, np.nan, 0, 0)),
        "scan index 0": _blob(scan_index=0),
    }
    for what, blob in bad.items():
        assert _code(aloam, blob) == ERR_SNAPSHOT, what
        assert _loc_info(aloam, blob)[0] == ERR_SNAPSHOT, what
    # the size handed in must be the snapshot's
    assert _code(aloam, good[:-16]) == ERR_SNAPSHOT
    assert _code(aloam, good, len(good) - 1) == ERR_SNAPSHOT
    assert _code(aloam, good + bytes(16)) == ERR_SNAPSHOT
    assert _code(aloam, good[:S], S) == ERR_SNAPSHOT   # no locator section
    # the map position: T_wmap_wodom applied to the world translation (3, -1, 0.25) with the quaternion as stored
    assert _code(aloam, _blob(T=(0, 0, 0, 1.0, 50.0 * 2**31 - 25.0 - 3.0 - 1e3, 0, 0))) == 0
    assert _code(aloam, _blob(T=(0, 0, 0, 1.0, 50.0 * 2**31 - 25.0 - 3.0 + 1e3, 0, 0))) == ERR_SNAPSHOT
    with pytest.raises(aloam.AloamError) as e:
        aloam.snapshot_info(bad["zero quaternion"])
    assert e.value.code == ERR_SNAPSHOT


def test_localise_info_refuses_version_1(aloam):
    assert _code(aloam, _v1()) == 0
    assert _loc_info(aloam, _v1())[0] == ERR_SNAPSHOT
    assert _loc_info(aloam, _v1(0, 0))[0] == ERR_SNAPSHOT
    assert aloam.lib().aloam_snapshot_localise_info(None, 256, None, None, None, None) == ERR_INVALID_ARG
    assert _loc_info(aloam, _blob()[:255])[0] == ERR_SNAPSHOT
