"""GPU: a cube store larger than one staging window of host memory (4 M points) moved through every store copy -- restored from,
exported to and saved to pageable host memory, exported to device memory, and loaded as the prior map and exported again.  The
store is a real mapped lane snapshot whose store section is replaced by a synthetic one of about 6.2 M points, laid out exactly as
aloam_lane_save writes one.  Every copy must give back the payload byte for byte, in both export orders."""
import struct

import numpy as np
import pytest

import lane_refs as R

pytestmark = pytest.mark.gpu

NCUBE = 4851
HEADER, TABLE = 256, 39424          # sizeof(SnapHeader), sizeof(SnapStore)
CAP = (16384, 65536)                 # slab capacities of a context with max_points >= 65536
MAXPTS = 65536


def _ctx(aloam):
    return aloam.Aloam(n_scans=16, max_points=MAXPTS, max_batch=1, max_ring_points=4096, max_map_points=400000)


def _big_snapshot(aloam, synth):
    """(blob, payload as (n, 4) float32, counts [2][NCUBE], valid cubes): a mapped lane snapshot of six scans whose store holds the
    valid cubes full (16384 corner, 65536 surf points) and 20 other cubes partly"""
    scans = R.traj(synth, 0, 6)
    dev = R.to_device(scans)
    c = _ctx(aloam)
    ops = np.array([[2]] + [[1]] * (len(dev) - 1), np.int32)
    c.scan_stream_lanes([[d.data_ptr()] for d in dev], [[d.shape[0]] for d in dev], ops, True, mapped=True)
    blob = np.asarray(c.lane_save(0)).copy()
    c.close()
    n_ls, n_lf = struct.unpack_from("<ii", blob, 28)
    store = HEADER + 16 * (n_ls + n_lf)
    table = bytearray(blob[store:store + TABLE].tobytes())
    n_valid = struct.unpack_from("<i", table, 12)[0]
    valid = list(struct.unpack_from("<%di" % n_valid, table, 16))
    assert n_valid > 0
    counts = np.full((2, NCUBE), -1, np.int32)
    for v in valid:
        counts[:, v] = CAP
    others = [i for i in range(NCUBE) if i not in valid][:20]
    for k, i in enumerate(others):
        counts[0, i], counts[1, i] = 1000 + k, 3000 + 7 * k
    n = int(np.maximum(counts, 0).sum())
    assert n > 4 << 20, "the store must not fit one staging window"
    # the table as aloam_lane_save writes it: the fields that outlive a frame kept, the counts, zero1 = 0, n_points, zero2 = 0
    table[592:592 + counts.nbytes] = counts.tobytes()
    struct.pack_into("<iiqq", table, 592 + counts.nbytes, 0, 0, n, 0)
    payload = np.random.default_rng(7).uniform(-500, 500, (n, 4)).astype(np.float32)
    out = np.concatenate([blob[:store], np.frombuffer(bytes(table), np.uint8), payload.view(np.uint8).reshape(-1)])
    struct.pack_into("<q", out, 16, out.size)   # total_bytes
    return out, payload, counts, valid


def _segments(payload, counts, cubes):
    """the payload's corner then surf segment of each of `cubes`"""
    ends = np.cumsum(np.maximum(counts, 0).T.reshape(-1))
    starts = ends - np.maximum(counts, 0).T.reshape(-1)
    return np.concatenate([payload[starts[2 * i + t]:ends[2 * i + t]] for i in cubes for t in (0, 1)])


def test_a_store_beyond_one_staging_window_moves_through_every_copy(aloam, synth):
    import torch
    blob, payload, counts, valid = _big_snapshot(aloam, synth)
    n = payload.shape[0]
    c = _ctx(aloam)
    try:
        c.lane_restore(0, blob)                                                 # host -> store, several windows
        s = c.mapper_state(0)
        assert (s["total_corner"], s["total_surf"]) == tuple(int(x) for x in np.maximum(counts, 0).sum(axis=1))
        host = c.mapper_export(aloam.EXPORT_MAP, 0)                             # store -> pageable host memory
        assert host.shape == payload.shape and host.tobytes() == payload.tobytes(), "EXPORT_MAP to host memory"
        out = torch.empty((n + 5, 4), dtype=torch.float32, device="cuda")       # store -> device memory, in place
        got = c.mapper_export(aloam.EXPORT_MAP, 0, out=out)
        assert got.shape[0] == n and got.cpu().numpy().tobytes() == payload.tobytes(), "EXPORT_MAP to device memory"
        assert np.asarray(c.lane_save(0)).tobytes() == blob.tobytes(), "lane_save of the restored store"
        sur = c.mapper_export(aloam.EXPORT_SURROUND, 0)
        assert sur.tobytes() == _segments(payload, counts, valid).tobytes(), "EXPORT_SURROUND"
        c.prior_map_load(blob)                                                  # host -> prior map
        prior = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP)
        assert prior.tobytes() == payload.tobytes(), "EXPORT_MAP of the prior map"
    finally:
        c.close()
