"""GPU: cube growth at its limits -- an allocation that fails on a fragmented pool, a restore whose runs fill the pool exactly, and
prior maps whose cubes need the upper bits of the 18-bit rank of the prior-map tag (loaded from a growth-on snapshot and built)."""
import struct

import numpy as np
import pytest

import cube_edge_cases as E
import lane_refs as R
import test_gpu_prior_build as PB
import test_gpu_prior_edges as PE

pytestmark = pytest.mark.gpu

ERR_SNAPSHOT = -11
NCUBE, CW, CH = 4851, 21, 21
IDENT_Q = np.array([0.0, 0.0, 0.0, 1.0])
EMPTY = np.zeros((0, 4), np.float32)
IDLE, SCAN, START = 0, 1, 2


def _at(ijk, off=1.0):
    """a point inside cube (i, j, k) of a store with centre offsets (10, 10, 5)"""
    return [(ijk[0] - 10) * 50.0 + off, (ijk[1] - 10) * 50.0 + off, (ijk[2] - 5) * 50.0 + off, 1.0]


def _cube(ijk):
    return ijk[0] + CW * ijk[1] + CW * CH * ijk[2]


def _run_fragmented(aloam, orc):
    """max_points = 1024 (slab capacity 1024), growth on, every filter a pass-through.  Frame 1: one point in each of 1023 cubes,
    cube A first (slab 0) -- 1023 slabs used, slab 1023 free; frame 2: 1023 more points into A (1024, its slab is full); frame 3: two
    more into A, which needs an aligned run of 2 slabs while only slab 1023 is free.  Returns (frame flags, A's cube, the export,
    the oracle's A)"""
    rng = np.random.default_rng(11)
    cubes = [(i, j, k) for k in range(11) for j in range(21) for i in range(21)]
    A = (10, 10, 5)
    cubes.remove(A)
    pick = [A] + [cubes[q] for q in rng.permutation(len(cubes))[:1022]]
    frames = [np.array([_at(c) for c in pick], np.float32)]
    for m in (1023, 2):
        p = np.zeros((m, 4), np.float32)
        p[:, :3] = rng.uniform(-20, 20, (m, 3))
        p[:, 3] = rng.uniform(0, 16, m)
        frames.append(p)
    c = aloam.Aloam(n_scans=16, max_points=1024, max_map_points=400000, line_res=1e-4, plane_res=1e-4)
    c.set_cube_growth(1)
    c.mapper_reset()
    cm = orc.CubeMap() if orc else None
    flags = []
    for f in frames:
        if cm:
            cm.step(EMPTY, f, IDENT_Q, np.zeros(3), 1e-4, 1e-4)
        _, _, st = c.mapper_step(EMPTY, f, IDENT_Q, np.zeros(3))
        flags.append(st["flags"])
    out = (flags, c.mapper_cube(1, _cube(A)).copy(), c.mapper_export(aloam.EXPORT_MAP, 0).copy(), cm.cube(1, _cube(A)) if cm else None)
    c.close()
    return out


def test_growth_on_a_fragmented_pool(aloam, orc):
    """a free slab but no aligned run of two: the frame is flagged, A keeps its one full slab holding the oracle's first 1024
    points (the two new ones dropped), and a second context gives the same store byte for byte"""
    flags, a, export, want = _run_fragmented(aloam, orc)
    assert not flags[0] & aloam.FLAG_CUBE_OVERFLOW and not flags[1] & aloam.FLAG_CUBE_OVERFLOW
    assert flags[2] & aloam.FLAG_CUBE_OVERFLOW
    assert len(want) == 1026 and len(a) == 1024 and a.tobytes() == want[:1024].tobytes()
    flags2, a2, export2, _ = _run_fragmented(aloam, None)
    assert flags2 == flags and a2.tobytes() == a.tobytes() and export2.tobytes() == export.tobytes()


def _split(blob, export):
    """the points of every (type, cube) of a saved store, from its counts and ALOAM_EXPORT_MAP payload"""
    counts = E.store_counts(blob)
    n = np.maximum(counts, 0).T.reshape(-1)
    ends = np.cumsum(n)
    return counts, {(t, i): export[e - k:e] for (i, t), e, k in zip([(i, t) for i in range(NCUBE) for t in (0, 1)], ends, n)}


def _payload(counts, cubes):
    return np.concatenate([cubes[(t, i)] for i in range(NCUBE) for t in (0, 1) if counts[t, i] > 0])


def _slabs(counts, cap):
    used = 0
    for n in counts[counts >= 0]:
        r = 1
        while r * cap < n:
            r *= 2
        used += r
    return used


def test_restore_that_fills_the_pool_exactly(aloam, synth):
    """a growth-on VLP-16 lane at the default leaves, saved after 24 scans with a grown corner cube; count-1 corner cubes are added
    on the three lowest layers of the buffer (never reached) until the runs need exactly 1024 corner slabs.  Restored into another lane and
    into a context whose growth is off, the export is the snapshot's payload byte for byte, and the two continue 8 scans bit for
    bit alike and, while no frame is flagged, like the uninterrupted lane.  One more count-0 cube needs 1025 slabs: refused"""
    n, cut = 32, 24
    scans = R.traj(synth, 0, n)
    dev = R.to_device(scans)
    kw = dict(n_scans=16, max_points=R.maxn([scans]) + 1024, max_map_points=400000, max_batch=2)
    ptrs = np.array([[d.data_ptr()] * 2 for d in dev], np.uint64)
    counts_in = np.array([[s.shape[0]] * 2 for s in scans])

    def ops(rows, lane, first):
        o = np.full((rows, 2), IDLE, np.int32)
        o[:, lane] = SCAN
        o[0, lane] = first
        return o

    c = aloam.Aloam(**kw)
    c.set_cube_growth(1)
    _, whole = c.scan_stream_lanes(ptrs, counts_in, ops(n, 0, START), True)
    _, _ = c.scan_stream_lanes(ptrs[:cut], counts_in[:cut], ops(cut, 0, START), True)
    blob = c.lane_save(0)
    export = c.mapper_export(aloam.EXPORT_MAP, 0).copy()
    cap0 = struct.unpack_from("<i", blob.tobytes(), 68)[0]
    counts, cubes = _split(blob, export)
    assert counts[0].max() > cap0   # a grown corner cube
    free = [i for i in range(3 * CW * CH) if counts[0, i] < 0 and counts[1, i] < 0]   # layers k = 0 .. 2: 100 m and more below
    need = 1024 - _slabs(counts[0], cap0)
    assert 0 < need <= len(free)
    for i in free[:need]:
        counts[0, i] = 1
        cubes[(0, i)] = np.array([_at((i % CW, (i // CW) % CH, i // (CW * CH)), 2.0)], np.float32)
    assert _slabs(counts[0], cap0) == 1024
    full = E.with_store_fields(blob, counts=counts, points=_payload(counts, cubes))
    over = counts.copy()
    over[0, free[need]] = 0
    assert _slabs(over[0], cap0) == 1025
    bad = E.with_store_fields(blob, counts=over, points=_payload(over, cubes))
    with pytest.raises(aloam.AloamError) as e:
        c.lane_restore(1, bad)
    assert e.value.code == ERR_SNAPSHOT
    c.lane_restore(1, full)
    assert c.mapper_export(aloam.EXPORT_MAP, 1).tobytes() == _payload(counts, cubes).tobytes()
    c.set_map_rows(True)
    _, a = c.scan_stream_lanes(ptrs[cut:], counts_in[cut:], ops(n - cut, 1, SCAN), True)
    ra = c.map_rows(2 * (n - cut))["flags"].reshape(n - cut, 2)[:, 1]
    ea = c.mapper_export(aloam.EXPORT_MAP, 1).tobytes()
    c.close()
    d = aloam.Aloam(**kw)   # growth off: the restored lane keeps the snapshot's
    d.lane_restore(0, full)
    _, b = d.scan_stream_lanes(ptrs[cut:], counts_in[cut:], ops(n - cut, 0, SCAN), True)
    assert np.array_equal(a[:, 1], b[:, 0]) and d.mapper_export(aloam.EXPORT_MAP, 0).tobytes() == ea
    d.close()
    ok = np.flatnonzero(ra & aloam.FLAG_CUBE_OVERFLOW)
    upto = ok[0] if len(ok) else n - cut
    assert np.array_equal(a[:upto, 1], whole[cut:cut + upto, 0])


# ---- prior maps with cubes past 65536 points

MAXMAP = 400000


@pytest.fixture(scope="module")
def penv(aloam, synth):
    """as test_gpu_prior_edges.env, with max_map_points large enough for a mapping frame to gather a 2^17-point cube"""
    scans = R.traj(synth, 0, 4, sensor="VLP-16")
    dev = R.to_device(scans)
    cfg = dict(n_scans=16, max_points=PE.MAXPTS, max_ring_points=4096, max_map_points=MAXMAP)
    c = aloam.Aloam(max_batch=1, **cfg)
    ops = np.array([[2]] + [[1]] * 2, np.int32)
    c.scan_stream_lanes([[d.data_ptr()] for d in dev[:3]], [[d.shape[0]] for d in dev[:3]], ops, True, mapped=True)
    tmpl = np.asarray(c.lane_save(0)).copy()
    real = c.mapper_export(aloam.EXPORT_MAP, 0).copy()
    c.close()
    counts, cubes = _split(tmpl, real)
    e = {"tmpl": tmpl, "scans": scans, "dev": dev, "cfg": cfg, "counts": counts, "cubes": cubes,
         "loc": aloam.Aloam(max_batch=1, **cfg), "ref": aloam.Aloam(n_scans=16, max_points=PE.MAXPTS, max_map_points=MAXMAP)}
    yield e
    e["loc"].close()
    e["ref"].close()


def test_growth_on_snapshot_with_a_big_cube_as_a_prior_map(penv, orc, aloam):
    """the real store of a mapped lane with 140000 far filler points put in front of both centre cubes, so the real points there
    sit at ranks 140000 and up (bits 16 and 17 of the tag), saved as a growth-on snapshot (refused with growth off in the header):
    it loads as a prior map; the association of the centre cube's points through a localising lane's window gives the submap
    indices of the float32 brute force, the oracle's fits and aloam_mapping_associate's rows; and the localising frame equals the
    mapping frame of a lane restored from the same snapshot, bit for bit"""
    rng = np.random.default_rng(17)
    S = PE.Store()
    centre = _cube((10, 10, 5))
    for ty in (0, 1):
        fill = np.zeros((140000, 4), np.float32)
        fill[:, :3] = rng.uniform(-24.5, -20.0, (140000, 3))
        S.put(ty, (10, 10, 5), fill)
    for (ty, i), p in penv["cubes"].items():
        if penv["counts"][ty, i] >= 0:
            S.put(ty, (i % CW, (i // CW) % CH, i // (CW * CH)), p)
    blob = S.blob(penv["tmpl"])
    blob = E.with_store_fields(blob, q_wmap=IDENT_Q, t_wmap=np.zeros(3))
    grown = bytearray(blob.tobytes())
    struct.pack_into("<i", grown, 220, 1)
    grown = np.frombuffer(bytes(grown), np.uint8)
    loc = penv["loc"]
    loc.reset_odometry()
    with pytest.raises(aloam.AloamError) as e:
        loc.prior_map_load(blob)          # growth off: 140000 points exceed one slab
    assert e.value.code == ERR_SNAPSHOT
    loc.prior_map_load(grown)
    assert loc.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == S.payload().tobytes()
    # the association: queries 3 cm off the real points of the centre cube
    env = {"loc": loc, "ref": penv["ref"], "dev": penv["dev"]}
    qc, qs = (np.ascontiguousarray(S.cubes[(ty, centre)][140000:140000 + 400].copy()) for ty in (0, 1))
    qc[:, :3] += 0.03
    qs[:, :3] += 0.03
    PE.arm(env, {0: (PE.Q0, np.zeros(3))})
    W = S.window(np.zeros(3))
    got = loc.prior_associate(0, qc, qs, PE.IDENT)
    res = PE.check(env, orc, W, qc, qs, got)
    for ty in (0, 1):
        idx, _, acc = res[ty]
        assert acc.any() and (idx[acc] >= 131072).any(), ty   # neighbours past rank 2^17 were found and decoded
    # one localising frame against the mapping frame of the restored lane
    loc.reset_odometry()
    loc.lane_localise(0, IDENT_Q, np.zeros(3))
    ptrs, counts_in = np.array([[penv["dev"][0].data_ptr()]], np.uint64), np.array([[penv["dev"][0].shape[0]]])
    o, m = loc.scan_stream_lanes(ptrs, counts_in, np.array([[START]], np.int32), True, mapped=True)
    scratch, feats = aloam.Aloam(max_batch=1, **penv["cfg"]), aloam.Aloam(max_batch=1, **penv["cfg"])
    scratch.lane_restore(0, grown)
    f = feats.extract_features(penv["scans"][0])
    q, t, st = scratch.mapper_step(f["less_sharp"], f["less_flat"], o[0, 0][:4], o[0, 0][4:])
    assert not st["flags"] & aloam.FLAG_MAP_TOO_THIN
    assert np.array_equal(m[0, 0], np.concatenate([q, t]))
    scratch.close()
    feats.close()


def test_dense_hdl64_map_builds_with_growth_on(aloam, synth):
    """the 8 M-point synthetic map at the HDL-64 leaves, whose largest corner cube keeps more than 65536 points (refused with growth
    off): with growth on it builds and equals the oracle's build bit for bit"""
    import torch
    corner, surf = PB._synth_map(aloam, synth, 8_000_000)
    ref, ref_dropped = PB._oracle(corner, surf, (0.4, 0.8))
    big = np.diff(ref.packed()["cube_start"], axis=1).max()
    assert 65536 < big <= 262144, big
    c = PB._ctx(aloam, 200000, 1, 64)
    c.set_cube_growth(1)
    got, dropped = PB._build(aloam, c, torch.from_numpy(corner).cuda(), torch.from_numpy(surf).cuda())
    assert dropped == ref_dropped
    assert PB._same(got, ref.export())
    c.close()
