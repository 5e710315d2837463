"""The sharded scan-to-map path on one GPU: a context emulates rank r of W (aloam_debug_shard_emulate), so the device shard cut,
the owned-point counts, the k-NN ownership reject, both sharded LM drivers and the sharded mapper frame run without a second
GPU.  Each rank is compared with the host split of shard.py, with the unsharded run and with the oracle chain restricted to
the rank.  What one GPU cannot check -- the NVLink / IPC transport, the tag order across ranks, ncclAllReduce itself -- stays
with tests/test_gpu_multi.py."""
import importlib
import math

import numpy as np
import pytest

import edge_scenes as es
from test_gpu_lm_edges import DELTA, IDENT, _cost_tol, _problem

shard = importlib.import_module("a-loam_b200.shard")

gpu = pytest.mark.gpu
WORLDS = [2, 3, 4, 5, 8, 16]
ERR_CAPACITY, ERR_STATE, ERR_COMM = -4, -9, -10


# ---------------------------------------------------------------------------------------------------------------- CPU


@pytest.mark.parametrize("world", [2, 3, 5, 8, 16])
def test_owner_of_cell_is_floor_division(world):
    """owner = floor((cx + 2^20) / 8) mod world, non-negative, also left of cx = -2^20 (x below about -1,048,586 m)"""
    cx = (-(1 << 20) + np.arange(-100, 101)).astype(np.int64)
    want = np.array([math.floor((int(c) + (1 << 20)) / 8) % world for c in cx])
    got = shard.owner_of_cell(cx, world)
    assert np.array_equal(got, want) and got.min() >= 0 and got.max() < world
    # a slab of 8 cells has one owner, consecutive slabs go round-robin
    assert np.all(got[1:] == np.where((cx[1:] + (1 << 20)) % 8 == 0, (got[:-1] + 1) % world, got[:-1]))


# ---------------------------------------------------------------------------------------------------------------- helpers


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _world_x(pts, x):
    """float32 world x of stack points at pose x in map_knn5_body's operation order (q * p + t in double, no FMA)"""
    u, w, t = np.asarray(x[:3], np.float64), float(x[3]), float(x[4])
    v = pts[:, :3].astype(np.float64)
    uv = np.stack([u[1] * v[:, 2] - u[2] * v[:, 1], u[2] * v[:, 0] - u[0] * v[:, 2], u[0] * v[:, 1] - u[1] * v[:, 0]], 1)
    uv = uv + uv
    c2x = u[1] * uv[:, 2] - u[2] * uv[:, 1]
    return (((v[:, 0] + w * uv[:, 0]) + c2x) + t).astype(np.float32)


def _knn_ref(orc, cloud, q, k):
    """exact k-NN in (float32 distance, index) order; -1 / inf past the end of a small cloud"""
    if len(cloud) >= k:
        return orc.bruteforce_knn(cloud, q, k)
    idx = np.full((len(q), k), -1, np.int32)
    sqd = np.full((len(q), k), np.inf, np.float32)
    for i in range(len(q)):
        d = es.sqdist_f32(cloud, q[i])
        o = np.lexsort((np.arange(len(cloud)), d))
        idx[i, :len(o)] = o
        sqd[i, :len(o)] = d[o]
    return idx, sqd


def _check_cut(ctx, orc, clouds, queries, rank, world):
    """after an emulated sharded upload: k-NN on this rank == brute force on shard.py's cut (content and stable order), and
    the index's sizes == the host's shard and owned counts.  Returns the owned counts."""
    kept, glob = ctx.debug_map_sizes()
    owned = []
    for t, (cloud, q) in enumerate(zip(clouds, queries)):
        cut = shard.shard_cloud(cloud, rank, world)
        own = int(np.sum(shard.owner_of_cell(shard.cell_x(cloud[:, 0]), world) == rank)) if world > 1 else len(cloud)
        assert kept[t] == len(cut) and glob[t] == own
        owned.append(own)
        idx, sqd = ctx.knn(2 + t, q, 5)
        ridx, rsqd = _knn_ref(orc, cut, q, 5)
        assert np.array_equal(idx, ridx) and _same_bits(sqd, rsqd)
    return owned


def _world_queries(cloud, x, n):
    q = cloud[:n].copy()
    q[:, :3] = (q[:, :3].astype(np.float64) @ _rot(x[:4]).T + x[4:]).astype(np.float32)
    return q


# ---------------------------------------------------------------------------------------------------------------- scenes


@pytest.fixture(scope="module")
def scene(orc, synth, scans):
    """HDL-64: map from scans 0,1,3,4 at their true poses, stacks from scan 2 (as test_gpu_mapping)"""
    ns, az, mr, lres, pres = synth.SENSORS["HDL-64"]
    corner, surf = [], []
    for k in [0, 1, 3, 4]:
        f = orc.Features(scans("HDL-64", k), ns, mr)
        R = _rot(synth.pose(k)[0]); tk = synth.pose(k)[1]
        for src, dst in [(f.less_sharp, corner), (f.less_flat, surf)]:
            w = src.copy(); w[:, :3] = (src[:, :3].astype(np.float64) @ R.T + tk).astype(np.float32); dst.append(w)
    cmap, smap = orc.voxel_grid(np.concatenate(corner), lres), orc.voxel_grid(np.concatenate(surf), pres)
    f2 = orc.Features(scans("HDL-64", 2), ns, mr)
    cs, ss = orc.voxel_grid(f2.less_sharp, lres), orc.voxel_grid(f2.less_flat, pres)
    q2, t2 = synth.pose(2)
    x0 = np.concatenate([q2, t2 + np.array([0.05, -0.04, 0.02])])
    return cmap, smap, cs, ss, x0


@pytest.fixture(scope="module")
def big_map(aloam, synth):
    """1M points (synth.build_map, the product's own feature extraction)"""
    c = aloam.Aloam(n_scans=64, max_points=200000)

    def feats(raw):
        f = c.extract_features(raw)
        return f["less_sharp"], f["less_flat"]
    maps = synth.build_map(feats, 1000000)
    c.close()
    return maps


def _edge_cloud():
    """points exactly on cell and slab boundaries (multiples of CELL and 8 CELL in float32) and one float step either side,
    x = -0.0, negative cells, and a cluster near x = -1.1e6 m (cells left of -2^20)"""
    C = shard.CELL
    xs = [np.float32(k) * C for k in range(-24, 25)] + [np.float32(8 * k) * C for k in range(-3, 4)]
    xs += [np.nextafter(v, np.float32(v + 1)) for v in xs[:] if v != 0] + [np.nextafter(v, np.float32(v - 1)) for v in xs[:] if v != 0]
    xs += [np.float32(-0.0), np.float32(0.0), np.float32(-0.3), np.float32(-8.5), np.float32(-17.2)]
    far = np.float32(-1.1e6) + np.arange(-30, 30, dtype=np.float32) * np.float32(0.375)   # 22.5 m: 3 or 4 slabs
    xs = np.concatenate([np.asarray(xs, np.float32), far])
    rng = np.random.default_rng(5)
    pts = np.zeros((len(xs) * 3, 4), np.float32)
    pts[:, 0] = np.repeat(xs, 3)
    pts[:, 1] = rng.uniform(-2, 2, len(pts)).astype(np.float32)
    pts[:, 2] = rng.uniform(-1, 1, len(pts)).astype(np.float32)
    pts[:, 3] = np.arange(len(pts), dtype=np.float32)
    return pts[rng.permutation(len(pts))]


# ---------------------------------------------------------------------------------------------------------------- the cut


@gpu
@pytest.mark.parametrize("world", WORLDS)
def test_cut_of_host_views_in_chunks(aloam, orc, scene, world):
    """host views of 4 and 8 floats per point, streamed through the stack buffer in chunks of 3500 / 1750 points: every rank's
    index holds shard.py's cut in its order, and its owned counts add up to the whole map"""
    cmap, smap, cs, ss, x0 = scene
    mp = 3500
    queries = [_world_queries(cs, x0, mp // 5), _world_queries(ss, x0, mp // 5)]
    wide = []
    for a in (cmap, smap):
        w = np.full((len(a), 8), -7.0, np.float32); w[:, :4] = a; wide.append(w)
    ctx = aloam.Aloam(n_scans=64, max_points=mp, max_map_points=16384)
    for views in ((cmap, smap), wide):
        total = np.zeros(2, np.int64)
        for r in range(world):
            ctx.debug_shard_emulate(r, world)
            ctx.map_upload_sharded(*views)
            total += _check_cut(ctx, orc, (cmap, smap), queries, r, world)
        assert list(total) == [len(cmap), len(smap)]
    ctx.close()


@gpu
@pytest.mark.parametrize("world", WORLDS)
def test_cut_of_a_device_view_of_1m_points(aloam, orc, big_map, world):
    """a device view is cut in one piece: 1M points are more than 1024 blocks of k_shard_scan"""
    import torch
    cmap, smap = big_map
    assert (len(smap) + 255) // 256 > 1024
    dc, ds = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (cmap, smap))
    queries = [cmap[::997][:200].copy(), smap[::1999][:200].copy()]
    ctx = aloam.Aloam(n_scans=64, max_points=4000, max_map_points=len(smap))
    total = np.zeros(2, np.int64)
    for r in range(world):
        ctx.debug_shard_emulate(r, world)
        ctx.map_upload_sharded_ptr(dc.data_ptr(), len(cmap), ds.data_ptr(), len(smap))
        total += _check_cut(ctx, orc, (cmap, smap), queries, r, world)
    assert list(total) == [len(cmap), len(smap)]
    ctx.close()


@gpu
@pytest.mark.parametrize("world", WORLDS)
def test_cut_of_edge_maps(aloam, orc, world):
    """points on cell / slab boundaries, -0.0, negative cells, x near -1.1e6 m; worlds that do not divide the slab count; at 16
    ranks some shards are empty"""
    cloud = _edge_cloud()
    half = len(cloud) // 2
    clouds = (cloud[:half], cloud[half:])
    queries = [np.concatenate([c[::3], c[1::7] + np.float32([0.45, 0.1, -0.2, 0])]).astype(np.float32)[:600] for c in clouds]
    ctx = aloam.Aloam(n_scans=64, max_points=4000, max_map_points=len(cloud))
    total, empty = np.zeros(2, np.int64), 0
    for r in range(world):
        ctx.debug_shard_emulate(r, world)
        ctx.map_upload_sharded(*clouds)
        total += _check_cut(ctx, orc, clouds, queries, r, world)
        empty += int(shard.shard_mask(clouds[0], r, world).sum() == 0)
    assert list(total) == [len(clouds[0]), len(clouds[1])]
    assert world < 16 or empty > 0
    far = shard.cell_x(clouds[0][:, 0]) < -(1 << 20)
    assert far.any() and np.any((shard.cell_x(clouds[0][far, 0]) + (1 << 20)) % 8 != 0)
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- association


def _fifth(q):
    """a point in the next cell along x whose float32 d^2 to q is 1 - 2^-24 exactly"""
    for dx in np.arange(0.80, 0.95, 0.0007):
        fx = np.float32(q[0] + dx)
        ddx = np.float32(fx - q[0])
        fy0 = np.float32(q[1] + np.sqrt(np.float64(es.ONE_BELOW) - np.float64(ddx * ddx)))
        for k in range(-8, 9):
            p = np.array([fx, np.float32(fy0 + np.float32(k) * np.spacing(fy0)), q[2]], np.float32)
            if es.sqdist_f32(p, q) == es.ONE_BELOW:
                return p
    raise AssertionError("no float32 point at d^2 = 1 - 2^-24")


def _halo_scene():
    """surf neighbourhoods on the plane z = 1.5 whose query sits in the last cell of a slab and whose 5th neighbour lies one slab
    further, in the halo, at float d^2 = 1 - 2^-24 (the largest distance the reference accepts); plus a plain grid"""
    C = shard.CELL
    pts, qs = [], []
    for i, m in enumerate(range(-4, 5)):
        xb = np.float32(8 * m) * C                      # slab boundary
        q = np.array([np.float32(xb - np.float32(0.05)), np.float32(3.0 * i), np.float32(1.5)], np.float32)
        near = q + np.array([[-0.3, 0.1, 0], [-0.2, -0.25, 0], [-0.45, 0.3, 0], [-0.1, -0.4, 0]], np.float32)
        fifth = _fifth(q)
        assert shard.cell_x(q[:1])[0] == 8 * m - 1 and shard.cell_x(fifth[:1])[0] == 8 * m
        pts += [*near, fifth]
        qs.append(q)
    gx, gy = np.meshgrid(np.arange(-30, 30, 0.45), np.arange(-3, 30, 0.45))
    grid = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, 1.5)], 1) + np.array([0, 0.13, 0])
    grid = grid[np.min(np.abs(grid[:, None, :2] - np.asarray(qs)[None, :, :2]).max(2), 1) > 1.5]   # keep the sites clean
    surf = np.zeros((len(pts) + len(grid), 4), np.float32)
    surf[:len(pts), :3] = np.asarray(pts); surf[len(pts):, :3] = grid
    stack = np.zeros((len(qs) + 300, 4), np.float32)
    stack[:len(qs), :3] = np.asarray(qs)
    stack[len(qs):, :3] = grid[::max(1, len(grid) // 300)][:300] + np.array([0.1, 0.05, 0.02])
    corner = np.zeros((40, 4), np.float32); corner[:, 0] = np.arange(40) * 0.3 - 6; corner[:, 1] = 50.0; corner[:, 2] = 1.0
    return corner, surf, corner[::4].copy(), stack, len(qs)


def _partition(ctx, maps, stacks, x, world, ref):
    """fits of every rank mapped back to unsharded indices: each row accepted unsharded is accepted on exactly the rank that
    owns its query's cell, bit for bit; a row rejected unsharded is rejected everywhere.  Returns the per-rank fits."""
    cs, ss = stacks
    qx = np.concatenate([_world_x(cs, x), _world_x(ss, x)])
    owner = shard.owner_of_cell(shard.cell_x(qx), world)
    taken = np.zeros(len(ref), int)
    per_rank = []
    for r in range(world):
        ctx.debug_shard_emulate(r, world)
        ctx.map_upload_sharded(*maps)
        got = ctx.mapping_associate(cs, ss, x)
        acc = got[:, 1] >= 0
        assert np.all(ref[acc, 1] >= 0) and np.all(owner[acc] == r)
        back = got.copy()
        n_c = len(cs)
        for rows, cloud in ((np.flatnonzero(acc[:n_c]), maps[0]), (n_c + np.flatnonzero(acc[n_c:]), maps[1])):
            keep = np.flatnonzero(shard.shard_mask(cloud, r, world))
            back[rows, 9:] = keep[got[rows, 9:].astype(np.int64)]
        assert _same_bits(back[acc], ref[acc])
        taken += acc
        per_rank.append(got)
    want = (ref[:, 1] >= 0).astype(int)
    assert np.array_equal(taken, want)
    return per_rank


def _blocks(fits, cs, ss):
    """the 11-double blocks of the accepted fit rows (corner rows are edges, surf rows plane-norms)"""
    acc = fits[fits[:, 1] >= 0]
    out = np.zeros((len(acc), 11))
    n_c = len(cs)
    for i, row in enumerate(acc):
        edge = row[1] == 0
        cp = (cs if edge else ss)[int(row[0])]
        out[i] = [row[1], *cp[:3].astype(np.float64), *row[2:8], 1.0 if edge else row[8]]
    return out


def _unsharded_fits(aloam, maps, stacks, x):
    c = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
    c.map_upload(*maps)
    ref = c.mapping_associate(*stacks, x)
    return c, ref


@gpu
@pytest.mark.parametrize("world", WORLDS)
def test_ownership_partitions_the_association(aloam, orc, scene, world):
    cmap, smap, cs, ss, x0 = scene
    ref_ctx, ref = _unsharded_fits(aloam, (cmap, smap), (cs, ss), x0)
    assert (ref[:, 1] >= 0).sum() > 1000
    ctx = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
    per_rank = _partition(ctx, (cmap, smap), (cs, ss), x0, world, ref)
    # the normal equations add up over the ranks
    blocks = [_blocks(f, cs, ss) for f in per_rank]
    parts = [ref_ctx.normal_equations(b, x0) if len(b) else (np.zeros((6, 6)), np.zeros(6), 0.0) for b in blocks]
    JtJ = np.array([[math.fsum(p[0][i, j] for p in parts) for j in range(6)] for i in range(6)])
    Jtr = np.array([math.fsum(p[1][i] for p in parts) for i in range(6)])
    cost = math.fsum(p[2] for p in parts)
    all_blocks = _blocks(ref, cs, ss)
    u_JtJ, u_Jtr, u_cost = ref_ctx.normal_equations(all_blocks, x0)
    o_JtJ, o_Jtr, o_cost = orc.normal_equations(all_blocks, x0)
    for a, b in ((JtJ, u_JtJ), (Jtr, u_Jtr)):     # the same blocks summed in another order
        assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max()
    assert abs(cost - u_cost) <= 1e-12 * u_cost
    # against the oracle: test_gpu_lm_edges' bars (the device evaluates each residual in another operation order)
    rows = int(np.sum(np.where(all_blocks[:, 0] == orc.EDGE, 3, 1)))
    assert np.abs(JtJ - o_JtJ).max() <= 1e-10 * np.abs(o_JtJ).max()
    assert np.abs(Jtr - o_Jtr).max() <= 1e-10 * np.abs(o_Jtr).max() + DELTA * np.sqrt(rows * np.diag(o_JtJ).max())
    assert abs(cost - o_cost) <= _cost_tol(o_cost, len(all_blocks), 1e-12)
    ctx.close(); ref_ctx.close()


@gpu
@pytest.mark.parametrize("world", [2, 3, 5])
def test_halo_neighbour_at_the_acceptance_limit(aloam, orc, world):
    """a query in the last cell of a slab whose 5th neighbour is across the slab boundary, in the halo, at d^2 = 1 - 2^-24: its
    owner accepts it with the unsharded fit, the rank that owns the 5th neighbour's cell rejects it"""
    corner, surf, cs, ss, n_sites = _halo_scene()
    x = np.array([0, 0, 0, 1.0, 0, 0, 0])
    ref_ctx, ref = _unsharded_fits(aloam, (corner, surf), (cs, ss), x)
    sites = len(cs) + np.arange(n_sites)
    assert np.all(ref[sites, 1] == 2)
    ctx = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
    per_rank = _partition(ctx, (corner, surf), (cs, ss), x, world, ref)
    fifth_owner = shard.owner_of_cell(shard.cell_x(ss[:n_sites, 0]) + 1, world)
    for i, s in enumerate(sites):
        assert per_rank[fifth_owner[i]][s, 1] == -1
    ctx.close(); ref_ctx.close()


# ---------------------------------------------------------------------------------------------------------------- the LM drivers

STAT_KEYS = ["n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps", "flags", "termination", "init_cost", "final_cost"]


def _oracle_chain(orc, maps, stacks, x, rank, world, outer=2):
    """laserMapping.cpp:562-727 restricted to the rank: associate, keep the rows whose query cell it owns, solve; twice"""
    m = orc.Mapping(); m.set_map(*maps)
    cs, ss = stacks
    x = np.array(x, np.float64)
    for _ in range(outer):
        fits, blocks = m.associate(cs, ss, x)
        if world > 1:
            qx = _world_x(np.stack([(cs if f[1] == 0 else ss)[int(f[0])] for f in fits]), x)
            blocks = blocks[shard.owner_of_cell(shard.cell_x(qx), world) == rank]
        x, _, _ = orc.solve(blocks, x, max_iters=4)
    return x


@gpu
@pytest.mark.parametrize("world", [1, 2, 3])
def test_three_exchanges_one_answer(aloam, orc, scene, world):
    """k_lm_solve, the per-evaluation kernels (k_lm_eval_shard -> copy -> k_lm_tr_shard) and the peer path (k_lm_solve_x with a
    one-rank mailbox) give the same stats and pose (to a few ulps) on every rank, equal to the oracle chain restricted to the rank; the peer
    path twice in a row (mailbox parity and counter carried over).  At one rank: equal to a context that does not emulate."""
    cmap, smap, cs, ss, x0 = scene
    plain = None
    if world == 1:
        c = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
        c.map_upload(cmap, smap)
        plain = c.mapping_register(cs, ss, x0)
        c.close()
    ctx = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
    for r in range(world):
        ctx.debug_shard_emulate(r, world, 0)
        ctx.map_upload_sharded(cmap, smap)
        runs = []
        for ex in (0, 1, 2, 2):
            ctx.debug_shard_emulate(r, world, ex)
            runs.append(ctx.mapping_register(cs, ss, x0))
        x_ref, st_ref = plain if plain else runs[0]
        # the three drivers take the same decisions from the same totals; the trust-region step is compiled into three kernels
        # with fused multiply-adds (lm.cu), so the poses agree to a few ulps of the quaternion (measured: <= 3.5e-18), not bit for bit
        for x, st in runs:
            assert np.abs(x - x_ref).max() <= 1e-15 and all(st[k] == st_ref[k] for k in STAT_KEYS)
        assert _same_bits(runs[2][0], runs[3][0])
        assert st_ref["flags"] == 0
        xo = _oracle_chain(orc, (cmap, smap), (cs, ss), x0, r, world)
        assert np.abs(runs[0][0] - xo).max() < 1e-9
    ctx.close()


@gpu
@pytest.mark.parametrize("name", ["gradient", "parameter", "function", "iterations", "rejected"])
def test_lm_exits_through_every_exchange(aloam, orc, name):
    """each LM exit of test_gpu_lm_edges (and a solve with rejected steps) through aloam_solve on an emulated one-rank world:
    k_lm_tr_shard's bookkeeping in T.acc and the peer path equal the cluster solve's acc_buf, with the same trace"""
    if name == "rejected":
        blocks, x0 = es.near_parallel_planes(orc, 0), IDENT
    else:
        blocks, x0, _ = _problem(orc, name)
    ctx = aloam.Aloam(n_scans=64, max_points=20000)
    ref = ctx.solve(blocks, x0)
    xr, _, _ = orc.solve(blocks, x0, max_iters=4)
    assert np.abs(ref[0] - xr).max() < 1e-9
    if name == "rejected":
        assert ref[1]["num_successful"] < ref[1]["num_iterations"]
    for ex in (1, 2, 2):
        ctx.debug_shard_emulate(0, 1, ex)
        got = ctx.solve(blocks, x0)
        assert _same_bits(got[0], ref[0]) and got[1] == ref[1] and _same_bits(got[2], ref[2])
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- mapper frames


@gpu
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_mapper_frames(aloam, synth, world):
    """5 HDL-64 scans through aloam_scan_stream_mapped on rank r of W: the cut of the device-sized submap
    (map_shard_index_device), the thin-map test on the whole submap and every exchange give the same map poses and mapper
    state; the batched call is refused while emulating"""
    raws = [synth.scan("HDL-64", k) for k in range(5)]
    ptrs, counts = [r.ctypes.data for r in raws], [r.shape[0] for r in raws]
    for r in range(world):
        ref = None
        for ex in (0, 1, 2):
            ctx = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=600000, max_batch=2)
            ctx.debug_shard_emulate(r, world, ex)
            odom, mapped = ctx.scan_stream_mapped(ptrs, counts, False)
            st = ctx.mapper_state()
            if ex == 0:
                with pytest.raises(aloam.AloamError) as e:
                    ctx.scan_stream_mapped_batch(np.array([ptrs, ptrs]).T, np.array([counts, counts]).T, False)
                assert e.value.code == ERR_STATE
            ctx.close()
            got = (odom, mapped, st)
            if ref is None:
                ref = got
                assert np.abs(mapped[:, 4:] - odom[:, 4:]).max() > 0   # the refinement ran
                continue
            # odometry is untouched; the map poses carry the exchanges' last-ulp differences (test_three_exchanges_one_answer)
            # into the next frames, so the stores agree as in tests/multi_gpu_mapping_check.py
            assert _same_bits(got[0], ref[0]) and np.abs(got[1] - ref[1]).max() < 1e-12
            assert got[2]["centre"] == ref[2]["centre"] and got[2]["valid"] == ref[2]["valid"]
            assert abs(got[2]["total_corner"] - ref[2]["total_corner"]) <= 5 and abs(got[2]["total_surf"] - ref[2]["total_surf"]) <= 20


# ---------------------------------------------------------------------------------------------------------------- fixed defects


@gpu
@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("device_view", [False, True])
def test_oversized_shard_is_refused(aloam, scene, world, device_view):
    """a shard larger than max_map_points: ALOAM_ERR_CAPACITY, no map afterwards, and a correct upload then equals a fresh
    context's bit for bit"""
    import torch
    cmap, smap, cs, ss, x0 = scene
    cap = 3000
    assert len(shard.shard_cloud(cmap, 0, world)) > cap
    small = (cmap[:1500], smap[:2500])
    queries = [_world_queries(cs, x0, 400), _world_queries(ss, x0, 400)]

    def make():
        c = aloam.Aloam(n_scans=64, max_points=3500, max_map_points=cap)
        c.debug_shard_emulate(0, world)
        return c

    def run(c):
        c.map_upload_sharded(*small)
        return [*c.knn(2, queries[0], 5), *c.knn(3, queries[1], 5), c.mapping_associate(cs, ss, x0), *c.mapping_register(cs, ss, x0)]

    ctx = make()
    ctx.map_upload_sharded(*small)                     # a map that fits, replaced by the failing upload below
    with pytest.raises(aloam.AloamError) as e:
        if device_view:
            dc, ds = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (cmap, smap))
            ctx.map_upload_sharded_ptr(dc.data_ptr(), len(cmap), ds.data_ptr(), len(smap))
        else:
            ctx.map_upload_sharded(cmap, smap)
    assert e.value.code == ERR_CAPACITY
    with pytest.raises(aloam.AloamError) as e:
        ctx.mapping_register(cs, ss, x0)
    assert e.value.code == ERR_STATE
    got = run(ctx)
    fresh = make()
    want = run(fresh)
    for g, w in zip(got[:4], want[:4]):
        assert _same_bits(g, w)
    acc = want[4][:, 1] >= 0   # the record of a rejected query is written only in part
    assert _same_bits(got[4][:, 1], want[4][:, 1]) and _same_bits(got[4][acc], want[4][acc])
    assert _same_bits(got[5], want[5]) and {k: got[6][k] for k in STAT_KEYS} == {k: want[6][k] for k in STAT_KEYS}
    ctx.close(); fresh.close()


@gpu
def test_peer_error_word_is_reported(aloam, scene):
    """the mailbox's error word set before a call (as a peer timeout leaves it): ALOAM_ERR_COMM; the next call is clean again"""
    cmap, smap, cs, ss, x0 = scene
    ctx = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
    ctx.debug_shard_emulate(0, 2, 2)
    ctx.map_upload_sharded(cmap, smap)
    clean = ctx.mapping_register(cs, ss, x0)
    ctx.debug_shard_emulate(0, 2, 2, poison_peer_err=True)
    with pytest.raises(aloam.AloamError) as e:
        ctx.mapping_register(cs, ss, x0)
    assert e.value.code == ERR_COMM
    again = ctx.mapping_register(cs, ss, x0)
    assert _same_bits(again[0], clean[0]) and all(again[1][k] == clean[1][k] for k in STAT_KEYS)
    ctx.close()


@gpu
def test_emulation_and_a_communicator_exclude_each_other(aloam):
    ctx = aloam.Aloam(n_scans=16, max_points=2000, max_map_points=1000)
    ctx.debug_shard_emulate(1, 3, 1)
    with pytest.raises(aloam.AloamError) as e:
        ctx.comm_init(0, 2, bytes(128))
    assert e.value.code == ERR_STATE
    for bad in ((3, 3, 0), (0, 2, 3), (-1, 2, 0)):
        with pytest.raises(aloam.AloamError) as e:
            ctx.debug_shard_emulate(*bad)
        assert e.value.code == -1
    ctx.debug_shard_emulate(0, 0)
    ctx.close()
