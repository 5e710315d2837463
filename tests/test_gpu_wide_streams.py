"""GPU: the stream paths of 128-wide contexts (aloam_create_wide above 64 rings) at their edges.  The solo entry points
(extract_features, odometry_set_last / _associate, knn) run the cluster ring kernel and size the association from the clouds;
the stream calls run k_ring_features_batch in batches, k_compact into fixed slots (128 x 12 sharp, 24 flat, 120 less-sharp), the
fused k_odom_assoc<128> over 1536 + 3072 query slots split at slot 1536, and the batched index build.  Scenes
(tests/wide_stream_cases.py, checked on the CPU by tests/test_oracle_wide_streams.py) fill every ring's caps, so every fused slot
is occupied up to sharp slot 1535 and flat slot 3071, or hold features only on the high rings; every path is held to the oracle
chain (the bars of test_gpu_wide_rings.py) and every lane to its solo run, bit for bit.  Lanes restored from snapshots whose last
clouds fill max_points at the packed-index bound, and refusals inside a 16-lane batch, complete the set."""
import struct

import numpy as np
import pytest

import wide_stream_cases as S
from conftest import rot_angle
from test_gpu_ring_field import _expect
from test_lane_snapshot_format import _header

pytestmark = pytest.mark.gpu

ERR_RING_TOO_LARGE, ERR_NOT_RING_MAJOR = -7, -8
IDLE, SCAN, START = 0, 1, 2
FRAMES = 5


def _wide(aloam, ns, max_points, **kw):
    mr, lr, pr = 0.3, 0.2, 0.4   # synth.RING_RANGES
    return aloam.Aloam(n_scans=ns, max_points=max_points, ring_source=aloam.RING_FIELD, minimum_range=mr, line_res=lr, plane_res=pr,
                       wide=True, **kw)


def _dev(raws):
    import torch
    return [torch.from_numpy(np.ascontiguousarray(r)).cuda() for r in raws]


def _close(got, want, what=""):
    for k in range(len(want)):
        assert np.abs(got[k, 4:] - want[k, 4:]).max() < 1e-4 and rot_angle(got[k, :4], want[k, :4]) < 1e-4, (what, k)
        assert np.abs(got[k, 4:] - want[k, 4:]).max() < 1e-7, (what, k, got[k, 4:] - want[k, 4:])


def _grid(cols, dev=None):
    """(steps, lanes) addresses and counts of per-lane scan lists (device tensors when dev is given)"""
    n, b = len(cols[0]), len(cols)
    ptrs = np.array([[(dev[j][k].data_ptr() if dev else cols[j][k].ctypes.data) for j in range(b)] for k in range(n)], np.uint64)
    cnt = np.array([[len(cols[j][k]) for j in range(b)] for k in range(n)], np.int64)
    return ptrs, cnt


_CHAINS = {}


def _chain(orc, key, raws, ns, distortion, nearby):
    if key not in _CHAINS:
        _CHAINS[key] = S.oracle_chain(orc, raws, ns, bool(distortion), nearby)[:2]
    return _CHAINS[key]


def _exports(aloam, c, lane=0):
    return [np.asarray(c.mapper_export(w, lane)) for w in (aloam.EXPORT_MAP, aloam.EXPORT_SURROUND)]


# ------------------------------------------------------------------------------------------------ 1. full-cap and high-ring chains
CHAIN_CASES = [("full128", 0, 2.5), ("full128", 1, np.inf), ("full96", 0, np.inf), ("full65", 1, 2.5), ("high64", 0, 2.5),
               ("high64", 1, np.inf), ("ring127", 0, 2.5), ("ends", 1, np.inf), ("seam", 1, 2.5), ("seam", 0, np.inf)]


@pytest.mark.parametrize("scene,distortion,nearby", CHAIN_CASES)
def test_chain_through_every_stream_path(aloam, orc, synth, scene, distortion, nearby):
    """scan_to_pose against the oracle chain (counts equal, poses within 1e-7); scan_stream, scan_stream_batch at 2, 5 and 16
    lanes, scan_stream_lanes with staggered STARTs and idle lanes, scan_stream_mapped_batch: every lane equals the solo run"""
    if scene == "seam":
        ns, raws = 128, [S.seam_scan(synth, k) for k in range(FRAMES)]
    else:
        ns = S.SCENES[scene][0]
        raws = [S.scene_scan(scene, k) for k in range(FRAMES)]
    want, counts = _chain(orc, (scene, distortion, nearby), raws, ns, distortion, nearby)
    mp = max(len(r) for r in raws) + 1024
    c = _wide(aloam, ns, mp, distortion=distortion, nearby_scan=nearby, max_batch=16, max_map_points=400000)
    got = []
    for k, r in enumerate(raws):
        q, t, st = c.scan_to_pose(r)
        got.append(np.concatenate([q, t]))
        if k > 0:
            assert (st["n_corner_corr"], st["n_plane_corr"]) == counts[k], k
    got = np.array(got)
    _close(got, want, scene)
    dev = _dev(raws)
    ptr, cnt = [d.data_ptr() for d in dev], [len(r) for r in raws]
    c.reset_odometry()
    p, _ = c.scan_stream(ptr, cnt, True)
    assert np.array_equal(p, got)
    for nb in (2, 5, 16):   # k_ring_features_batch, the batched k_compact, k_rab_* and k_odom_assoc<128>
        c.reset_odometry()
        pb = c.scan_stream_batch(np.repeat(np.array(ptr, np.uint64)[:, None], nb, 1), np.repeat(np.array(cnt)[:, None], nb, 1), True)
        for j in range(nb):
            assert np.array_equal(pb[:, j], got), (nb, j)
        assert [(s["n_corner_corr"], s["n_plane_corr"]) for s in c.last_batch_stats] == [counts[-1]] * nb
    # lanes: lane 0 from step 0, lane 1 from step 1, lane 2 idle, lane 3 two scans from step 0 then idle, lane 4 from step 2
    plan = {0: (0, 5), 1: (1, 4), 3: (0, 2), 4: (2, 3)}
    steps, lanes = 5, 5
    ops = np.full((steps, lanes), IDLE, np.int32)
    lp = np.zeros((steps, lanes), np.uint64); lc = np.zeros((steps, lanes), np.int64)
    for lane, (s0, ln) in plan.items():
        for i in range(ln):
            ops[s0 + i, lane] = START if i == 0 else SCAN
            lp[s0 + i, lane], lc[s0 + i, lane] = ptr[i], cnt[i]
    c.reset_odometry()
    lo, _ = c.scan_stream_lanes(lp, lc, ops, True, mapped=False)
    assert np.isnan(lo[ops == IDLE]).all()
    for lane, (s0, ln) in plan.items():
        assert np.array_equal(lo[s0:s0 + ln, lane], got[:ln]), lane
    c.close()
    # mapped: the solo stream and three lanes of a mapped batch, with the stores of every lane
    s = _wide(aloam, ns, mp, distortion=distortion, nearby_scan=nearby, max_map_points=400000)
    s.set_cube_growth(True)
    so, sm = s.scan_stream_mapped(ptr, cnt, True)
    sx = _exports(aloam, s)
    s.close()
    assert np.array_equal(so, got)
    m = _wide(aloam, ns, mp, distortion=distortion, nearby_scan=nearby, max_batch=3, max_map_points=400000)
    m.set_cube_growth(True)
    mo, mm = m.scan_stream_mapped_batch(np.repeat(np.array(ptr, np.uint64)[:, None], 3, 1), np.repeat(np.array(cnt)[:, None], 3, 1), True)
    for j in range(3):
        assert np.array_equal(mo[:, j], so) and np.array_equal(mm[:, j], sm), j
        for a, b in zip(_exports(aloam, m, j), sx):
            assert np.array_equal(a, b), j
    m.close()
    if scene in ("ring127",) or (scene == "ends" and nearby != np.inf):
        assert all(x == (0, 0) for x in counts[1:])
    else:
        assert all(x[0] > 0 and x[1] > 0 for x in counts[1:])


# ------------------------------------------------------------------------------------------------ 2. sixteen distinct lanes
def test_sixteen_distinct_lanes_follow_their_oracle_chains(aloam, orc):
    """lane j's features on rings 7 j .. 7 j + 15 with its own motion: every lane of a 16-lane scan_stream_batch against its own
    oracle chain and its solo run; then a mapped 16-lane batch with a registered sink: every lane's odometry and map poses, its
    stores and its /velodyne_cloud_registered rows (the only output that holds a lane's ring-major cloud) equal its solo run's"""
    import torch
    B = 16
    cols = [[S.band_scan(j, k) for k in range(FRAMES)] for j in range(B)]
    mp = max(len(r) for col in cols for r in col) + 1024
    dev = [_dev(col) for col in cols]
    ptrs, cnt = _grid(cols, dev)
    c = _wide(aloam, 128, mp, max_batch=B)
    pb = c.scan_stream_batch(ptrs, cnt, True)
    stats = c.last_batch_stats
    c.close()
    solo = _wide(aloam, 128, mp)
    for j in range(B):
        want, counts = S.oracle_chain(orc, cols[j], 128)[:2]
        _close(pb[:, j], want, "lane %d" % j)
        assert (stats[j]["n_corner_corr"], stats[j]["n_plane_corr"]) == counts[-1], j
        solo.reset_odometry()
        p, _ = solo.scan_stream(list(ptrs[:, j]), list(cnt[:, j]), True)
        assert np.array_equal(pb[:, j], p), j
    solo.close()
    total = int(cnt.sum())
    sink = torch.full((total + 16, 4), np.nan, dtype=torch.float32, device="cuda")
    m = _wide(aloam, 128, mp, max_batch=B, max_map_points=400000)
    m.set_cube_growth(True)
    m.set_registered_sink(sink)
    mo, mm = m.scan_stream_mapped_batch(ptrs, cnt, True)
    begin, count = m.registered_rows(FRAMES * B)
    rows = [[sink[begin[k * B + j]:begin[k * B + j] + count[k * B + j]].cpu().numpy() for k in range(FRAMES)] for j in range(B)]
    stores = [_exports(aloam, m, j) for j in range(B)]
    m.close()
    for j in range(B):
        s = _wide(aloam, 128, mp, max_map_points=400000)
        s.set_cube_growth(True)
        sk = torch.full((int(cnt[:, j].sum()) + 16, 4), np.nan, dtype=torch.float32, device="cuda")
        s.set_registered_sink(sk)
        so, sm = s.scan_stream_mapped(list(ptrs[:, j]), list(cnt[:, j]), True)
        b, n = s.registered_rows(FRAMES)
        assert np.array_equal(mo[:, j], so) and np.array_equal(mm[:, j], sm), j
        for k in range(FRAMES):
            want = sk[b[k]:b[k] + n[k]].cpu().numpy()
            assert len(want) == len(cols[j][k]) and np.array_equal(rows[j][k].view(np.uint32), want.view(np.uint32)), (j, k)
        for a, w in zip(stores[j], _exports(aloam, s)):
            assert np.array_equal(a, w), j
        s.close()


# ------------------------------------------------------------------------------------------------ 3. refusals inside a wide batch
def test_refusals_in_lane_11_of_a_16_lane_batch(aloam):
    """a ring of max_ring_points + 1 returns in lane 11, and a snapshot whose last cloud is not ring-major restored into lane 11:
    each fails with its code, and the next call equals the one of a fresh context"""
    B, max_ring = 16, 1024
    cols = [[S.band_scan(j, k) for k in range(3)] for j in range(B)]
    mp = max(len(r) for col in cols for r in col) + 1024
    ptrs, cnt = _grid(cols)
    over = S.cap_scan(128, (5, 127), 10.0, per_ring=max_ring + 1)
    bad_p, bad_c = ptrs[:1].copy(), cnt[:1].copy()
    bad_p[0, 11], bad_c[0, 11] = over.ctypes.data, len(over)
    kw = dict(max_batch=B, max_ring_points=max_ring)
    ctx, fresh = _wide(aloam, 128, mp, **kw), _wide(aloam, 128, mp, **kw)
    _expect(aloam, ERR_RING_TOO_LARGE, lambda: ctx.scan_stream_batch(bad_p, bad_c, False))
    after = ctx.scan_stream_batch(ptrs, cnt, False)
    assert np.array_equal(after, fresh.scan_stream_batch(ptrs, cnt, False))
    # a lane snapshot of band lane 11 after two scans, its less-flat cloud made non-ring-major (the first point on ring 127)
    ops = np.array([[START], [SCAN]], np.int32)
    solo = _wide(aloam, 128, mp)
    solo.scan_stream_lanes(ptrs[:2, 11:12], cnt[:2, 11:12], ops, False, mapped=False)
    blob = solo.lane_save(0).copy()
    solo.close()
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    assert nls > 0 and nlf > 1
    bad = blob.copy()
    struct.pack_into("<f", bad, 256 + 16 * nls + 12, 127.05)
    for c in (ctx, fresh):
        c.reset_odometry()
    _expect(aloam, ERR_NOT_RING_MAJOR, lambda: ctx.lane_restore(11, bad))
    lops = np.full((3, B), SCAN, np.int32); lops[0] = START
    a, _ = ctx.scan_stream_lanes(ptrs, cnt, lops, False, mapped=False)
    b, _ = fresh.scan_stream_lanes(ptrs, cnt, lops, False, mapped=False)
    assert np.array_equal(a, b) and np.isfinite(a).all()
    # the good blob restores into lane 11 and resumes its solo run
    for c in (ctx, fresh):
        c.reset_odometry()
    ctx.lane_restore(11, blob)
    lops = np.full((1, B), IDLE, np.int32); lops[0, 11] = SCAN
    r, _ = ctx.scan_stream_lanes(ptrs[2:3], cnt[2:3], lops, False, mapped=False)
    solo = _wide(aloam, 128, mp)
    whole, _ = solo.scan_stream_lanes(ptrs[:, 11:12], cnt[:, 11:12], np.array([[START], [SCAN], [SCAN]], np.int32), False, mapped=False)
    solo.close()
    assert np.array_equal(r[0, 11], whole[2, 0])
    ctx.close(); fresh.close()


# ------------------------------------------------------------------------------------------------ 4. restored lanes at the packed-index bound
DELTA = np.float32(2.0 ** -9)


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _bound_blob(aloam, ns, n, raw, warm, world, seed):
    """an unmapped snapshot (the format of include/aloam_b200.h, written with test_lane_snapshot_format's header) whose last
    less-sharp and less-flat clouds are one wide_search_cases.bound_cloud of n points, with the nearest neighbours of the next
    scan's first 48 sharp and 48 flat points -- moved by the warm start -- planted at the last indices, past 2^23 (past 2^24 at 64
    rings) and in exact ties (distance DELTA on either side in z) between a late and an early index"""
    import wide_search_cases as W
    width = 128 if ns > 64 else 64
    cloud = W.bound_cloud(n, width, seed)
    f = S.features(raw, ns)
    R, t = _rot(warm[:4]), np.asarray(warm[4:])
    qs = np.concatenate([f.sharp[:48, :3], f.flat[:48, :3]]).astype(np.float64) @ R.T + t
    top = n - 1
    late = [top - i for i in range(24)] + [(1 << 23) + 1 + 9973 * i for i in range(24)] + [n - 25 - 131 * i for i in range(24)]
    late += [(1 << 24) + 7 + 4099 * i for i in range(24)] if width == 64 else [(1 << 23) + (1 << 22) + 3 + 4099 * i for i in range(24)]
    early = {72 + i: 1000 + 7919 * i for i in range(24)}   # queries 72 .. 95: ties with early indices
    for i, p in enumerate(qs):
        p = np.asarray(p, np.float32)
        cloud[late[i], :3] = p + np.float32([0, 0, DELTA])
        if i in early:
            cloud[early[i], :3] = p - np.float32([0, 0, DELTA])
    cfg = aloam.default_config(ns)
    h = _header(0, 1, n, n, 256 + 32 * n, world)
    struct.pack_into("<iiiii", h, 36, ns, 0, cfg.mapping_skip_frame, cfg.outer_iters, cfg.inner_iters)
    struct.pack_into("<f", h, 56, 0.3)
    struct.pack_into("<ddd", h, 80, cfg.huber, cfg.dist_sq_thresh, cfg.nearby_scan)
    struct.pack_into("<7d", h, 104, *warm)
    struct.pack_into("<i", h, 216, aloam.RING_FIELD)
    body = cloud.tobytes()
    return np.frombuffer(bytes(h) + body + body, np.uint8), cloud


@pytest.mark.parametrize("ns,n,lanes", [(128, (1 << 24) - 1, 3), (64, (1 << 25) - 1, 2)], ids=["128-2^24-1", "64-2^25-1"])
def test_restored_lanes_at_the_packed_index_bound(aloam, orc, ns, n, lanes):
    """snapshots whose last clouds fill max_points (2^24 - 1 at 128 rings, 2^25 - 1 in a 64-ring context of aloam_create_wide)
    restored into lanes 1 and max_batch - 1 of a batched context, then one SCAN step: each lane equals the same blob restored into
    lane 0 of a max_batch = 1 context, and lane 1 equals the oracle's register after set_last with the blob's clouds from the
    blob's warm start.  Device memory, measured with torch.cuda.mem_get_info on an H100 80GB HBM3: a max_batch = 1 context takes
    10.2 GB at 2^24 - 1 points (128 rings) and 20.4 GB at 2^25 - 1 (64 rings), about 610 bytes per point of max_points and lane;
    three lanes take 29.7 GB and 59.2 GB.  So the 128-ring case restores two blobs into lanes 1 and 2 of max_batch = 3 (peak
    about 30 GB) and the 64-ring case one blob into lane 1 of max_batch = 2 (peak 40.3 GB); the test skips when the batched context
    would not fit with 8 GB to spare."""
    import torch
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    one = _wide(aloam, ns, n)
    free1, _ = torch.cuda.mem_get_info()
    per_lane = free0 - free1
    print("\n[wide streams] %d rings, max_points %d: %.2f GB for a max_batch = 1 context" % (ns, n, per_lane / 1e9))
    if free1 < (lanes - 1) * per_lane + (8 << 30):
        one.close()
        pytest.skip("needs %.1f GB of free device memory" % ((lanes * per_lane + (8 << 30)) / 1e9))
    restored = list(range(1, lanes))   # lanes 1 .. max_batch - 1, blob i in lane i + 1
    rings = tuple(range(ns))
    raws = [S.cap_scan(ns, rings, 40.0, frame=k) for k in (1, 2)]
    warms = [np.array([0, 0, np.sin(0.004), np.cos(0.004), 0.05, -0.03, 0.0]), np.array([0, 0, np.sin(-0.003), np.cos(-0.003), 0.02, 0.04, 0.0])]
    worlds = [(0.0, 0.0, np.sin(0.1), np.cos(0.1), 3.0, -1.0, 0.25), (0.0, 0.0, 0.0, 1.0, -2.0, 5.0, 0.0)]
    blobs, clouds = zip(*[_bound_blob(aloam, ns, n, raws[i], warms[i], worlds[i], 11 + i) for i in range(len(restored))])
    # solo: each blob in lane 0 of the max_batch = 1 context
    solo = []
    for i in range(len(restored)):
        one.lane_restore(0, blobs[i])
        o, _ = one.scan_stream_lanes(np.array([[raws[i].ctypes.data]], np.uint64), np.array([[len(raws[i])]]), np.array([[SCAN]], np.int32),
                                     False, mapped=False)
        solo.append((o[0, 0].copy(), dict(one.last_batch_stats[0])))
    one.close()
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info()
    c = _wide(aloam, ns, n, max_batch=lanes)
    free3, _ = torch.cuda.mem_get_info()
    print("[wide streams] max_batch = %d: %.2f GB" % (lanes, (free2 - free3) / 1e9))
    try:
        for i, lane in enumerate(restored):
            c.lane_restore(lane, blobs[i])
        ptrs = np.array([[0] + [raws[i].ctypes.data for i in range(len(restored))]], np.uint64)
        cnts = np.array([[0] + [len(raws[i]) for i in range(len(restored))]])
        o, _ = c.scan_stream_lanes(ptrs, cnts, np.array([[IDLE] + [SCAN] * len(restored)], np.int32), False, mapped=False)
        stats = c.last_batch_stats
        print("[wide streams] peak of the test: %.2f GB in use on the device" % ((torch.cuda.mem_get_info()[1] - torch.cuda.mem_get_info()[0]) / 1e9))
    finally:
        c.close()
    for i in range(len(restored)):
        assert np.array_equal(o[0, i + 1], solo[i][0]), i
        assert (stats[i + 1]["n_corner_corr"], stats[i + 1]["n_plane_corr"]) == (solo[i][1]["n_corner_corr"], solo[i][1]["n_plane_corr"]), i
    # the oracle: set_last with blob 0's clouds, register the next scan's features from the warm start
    f = S.features(raws[0], ns)
    od = orc.Odometry()
    od.set_last(clouds[0], clouds[0])
    del clouds
    q, t, info = od.register(f.sharp, f.flat, warms[0][:4], warms[0][4:])
    assert (stats[1]["n_corner_corr"], stats[1]["n_plane_corr"]) == (info["corner_corr"], info["plane_corr"])
    assert info["corner_corr"] >= 48 and info["plane_corr"] >= 48
    w = np.array(worlds[0])
    qw, tw = orc.integrate_pose(w[:4], w[4:], q, t)
    _close(o[0, 1][None], np.concatenate([qw, tw])[None], "restored lane 1")
