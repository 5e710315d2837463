"""CPU: the lane snapshot format (include/aloam_b200.h, "Snapshot format, version 1").  Blobs are written here from the documented
layout alone and checked by aloam_snapshot_check, which needs neither a context nor a GPU: well-formed snapshots, mapped and not,
are accepted and described; every kind of corruption is refused with ALOAM_ERR_SNAPSHOT."""
import struct

import numpy as np
import pytest

ERR_INVALID_ARG, ERR_SNAPSHOT = -1, -11
NCUBE, STORE = 4851, 39424


def _header(mapped, scan_index, nls, nlf, total, world, caps=(16384, 65536), max_map=400000):
    h = bytearray(256)
    h[0:8] = b"ALOAMLS1"
    struct.pack_into("<iiq", h, 8, 1, mapped, total)
    struct.pack_into("<iii", h, 24, scan_index, nls, nlf)
    struct.pack_into("<iiiiifff", h, 36, 16, 0, 1, 2, 4, 0.3, 0.2, 0.4)   # n_scans, distortion, skip, outer, inner, ranges
    struct.pack_into("<iii", h, 68, caps[0], caps[1], max_map)
    struct.pack_into("<ddd", h, 80, 0.1, 25.0, 2.5)
    struct.pack_into("<7d", h, 104, 0, 0, 0, 1, 0.5, 0, 0)
    struct.pack_into("<7d", h, 160, *world)
    return h


def _store(counts, valid, n_points=None):
    s = bytearray(STORE)
    struct.pack_into("<4i", s, 0, 10, 10, 5, len(valid))
    struct.pack_into("<%di" % len(valid), s, 16, *valid)
    struct.pack_into("<i", s, 528, 7)
    struct.pack_into("<4d", s, 536, 0, 0, 0, 1)
    struct.pack_into("<3d", s, 568, 1.0, 2.0, 3.0)
    s[592:592 + 2 * NCUBE * 4] = np.ascontiguousarray(counts, np.int32).tobytes()
    struct.pack_into("<q", s, 39408, int(np.maximum(counts, 0).sum()) if n_points is None else n_points)
    return s


def _points(n, seed):
    p = np.random.default_rng(seed).uniform(-20, 20, (n, 4)).astype(np.float32)
    p[:, 3] = np.sort(np.random.default_rng(seed).integers(0, 16, n)) + 0.05   # ring-major intensity
    return p.tobytes()


def _blob(mapped=True, nls=40, nlf=90, counts=None, valid=(100, 200, 4850), scan_index=6, n_points=None, extra_points=0):
    world = (0.0, 0.0, 0.1, 0.995, 3.0, -1.0, 0.25)
    if counts is None:
        counts = np.full((2, NCUBE), -1, np.int32)
        counts[0, [3, 100, 4850]] = [5, 0, 17]
        counts[1, [100, 2000]] = [30, 1]
    body = _points(nls, 1) + _points(nlf, 2)
    if mapped:
        npts = int(np.maximum(counts, 0).sum()) + extra_points
        body += _store(counts, list(valid), n_points) + _points(npts, 3)
    total = 256 + len(body)
    return bytes(_header(int(mapped), scan_index, nls, nlf, total, world)) + body


def _code(aloam, blob, n=None):
    import ctypes as C
    a = np.frombuffer(blob, np.uint8)
    return aloam.lib().aloam_snapshot_check(C.c_void_p(a.ctypes.data), len(blob) if n is None else n, None)


def test_well_formed_snapshots_are_described(aloam):
    b = _blob(mapped=True)
    info = aloam.snapshot_info(b)
    assert info["version"] == 1 and info["mapped"] and info["n_scans"] == 16 and info["scan_index"] == 6
    assert info["bytes"] == len(b) == 256 + 16 * 130 + STORE + 16 * 53 and info["map_points"] == 53
    assert np.array_equal(info["world"], [0.0, 0.0, 0.1, 0.995, 3.0, -1.0, 0.25])
    u = _blob(mapped=False, nls=0, nlf=7, scan_index=1)
    info = aloam.snapshot_info(np.frombuffer(u, np.uint8))
    assert not info["mapped"] and info["bytes"] == len(u) == 256 + 16 * 7 and info["map_points"] == 0 and info["scan_index"] == 1
    # an empty store and a full pool (1024 cubes of each type holding a slab, some of them without points) are well-formed
    assert aloam.snapshot_info(_blob(counts=np.full((2, NCUBE), -1, np.int32), valid=()))["map_points"] == 0
    full = np.full((2, NCUBE), -1, np.int32)
    full[:, :1024] = 0
    full[0, 1023], full[1, 0] = 16384, 65536   # counts at the slab capacities
    assert aloam.snapshot_info(_blob(counts=full))["map_points"] == 16384 + 65536


def _patched(blob, offset, fmt, *values):
    b = bytearray(blob)
    struct.pack_into(fmt, b, offset, *values)
    return bytes(b)


def test_corruptions_are_refused(aloam):
    good = _blob()
    S = 256 + 16 * 130   # the store section of _blob()
    assert _code(aloam, good) == 0
    over = np.full((2, NCUBE), -1, np.int32)
    over[0, :1025] = 0
    bad = {
        "magic": _patched(good, 0, "<8s", b"ALOAMLS2"),
        "version": _patched(good, 8, "<i", 2),
        "mapped flag": _patched(good, 12, "<i", 2),
        "total_bytes": _patched(good, 16, "<q", len(good) + 16),
        "scan index": _patched(good, 24, "<i", 0),
        "negative cloud size": _patched(good, 28, "<i", -1),
        "corner count above its slab capacity": _blob(counts=np.where(np.arange(NCUBE) == 3, 16385, -1).astype(np.int32)[None].repeat(2, 0)),
        "surf count above its slab capacity": _patched(good, S + 592 + 4 * (NCUBE + 2000), "<i", 65537),
        "count below -1": _patched(good, S + 592 + 4 * 7, "<i", -2),
        "more than 1024 slabbed cubes": _blob(counts=over),
        "n_points not the sum of the counts": _blob(n_points=54, extra_points=1),
        "valid index out of range": _patched(good, S + 16 + 4, "<i", NCUBE),
        "negative valid index": _patched(good, S + 16, "<i", -1),
        "n_valid above 125": _patched(good, S + 12, "<i", 126),
        "a surf count changed": _patched(good, S + 592 + 4 * (NCUBE + 100), "<i", 31),
    }
    for what, blob in bad.items():
        assert _code(aloam, blob) == ERR_SNAPSHOT, what
    # the size handed in must be the snapshot's: truncated, or longer than its sections
    assert _code(aloam, good[:-16]) == ERR_SNAPSHOT
    assert _code(aloam, good, len(good) - 1) == ERR_SNAPSHOT
    assert _code(aloam, good + bytes(16)) == ERR_SNAPSHOT
    assert _code(aloam, good[:255]) == ERR_SNAPSHOT
    assert _code(aloam, good[:S + 100], S + 100) == ERR_SNAPSHOT   # cut inside the store table
    u = _blob(mapped=False)
    assert _code(aloam, u) == 0 and _code(aloam, u[:-16]) == ERR_SNAPSHOT
    assert _code(aloam, _patched(u, 12, "<i", 1)) == ERR_SNAPSHOT   # "mapped" without a store section
    with pytest.raises(aloam.AloamError) as e:
        aloam.snapshot_info(bad["magic"])
    assert e.value.code == ERR_SNAPSHOT
    assert aloam.lib().aloam_strerror(ERR_SNAPSHOT).decode().startswith("snapshot malformed")


def test_null_blob_is_an_invalid_argument(aloam):
    assert aloam.lib().aloam_snapshot_check(None, 256, None) == ERR_INVALID_ARG
