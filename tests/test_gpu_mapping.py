"""GPU parity: scan-to-map association + fits + LM (laserMapping.cpp:554-734) vs the CPU oracle, through the C ABI."""
import numpy as np
import pytest

from conftest import rot_angle

pytestmark = pytest.mark.gpu


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


@pytest.fixture(scope="module")
def scene(orc, synth, scans):
    """map from HDL-64 scans 0,1,3,4 at their true poses, stacks from scan 2"""
    sensor = "HDL-64"
    ns, az, mr, lres, pres = synth.SENSORS[sensor]
    corner, surf = [], []
    for k in [0, 1, 3, 4]:
        f = orc.Features(scans(sensor, k), ns, mr)
        qk, tk = synth.pose(k)
        R = _rot(qk)
        for src, dst in [(f.less_sharp, corner), (f.less_flat, surf)]:
            w = src.copy(); w[:, :3] = (src[:, :3].astype(np.float64) @ R.T + tk).astype(np.float32); dst.append(w)
    cmap = orc.voxel_grid(np.concatenate(corner), lres)
    smap = orc.voxel_grid(np.concatenate(surf), pres)
    f2 = orc.Features(scans(sensor, 2), ns, mr)
    cs, ss = orc.voxel_grid(f2.less_sharp, lres), orc.voxel_grid(f2.less_flat, pres)
    q2, t2 = synth.pose(2)
    x0 = np.concatenate([q2, t2 + np.array([0.05, -0.04, 0.02])])
    return cmap, smap, cs, ss, x0, (q2, t2)


@pytest.fixture(scope="module")
def ctx(aloam, scene):
    c = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=400000)
    c.map_upload(scene[0], scene[1])
    yield c
    c.close()


def test_map_knn_exact(ctx, orc, scene):
    cmap, smap, cs, ss, x0, _ = scene
    R = _rot(x0[:4])
    for which, cloud, q in [(2, cmap, cs), (3, smap, ss[:4000])]:
        qw = q.copy(); qw[:, :3] = (q[:, :3].astype(np.float64) @ R.T + x0[4:]).astype(np.float32)
        idx, sqd = ctx.knn(which, qw, 5)
        ridx, rsqd = orc.bruteforce_knn(cloud, qw, 5)
        assert np.array_equal(idx, ridx) and np.array_equal(sqd, rsqd)
        kidx, ksqd = orc.KdTree(cloud).knn(qw, 5)
        assert np.array_equal(kidx, ridx)


def test_fits_match_oracle(ctx, orc, scene):
    cmap, smap, cs, ss, x0, _ = scene
    m = orc.Mapping(); m.set_map(cmap, smap)
    fits, blocks = m.associate(cs, ss, x0)
    got = ctx.mapping_associate(cs, ss, x0)
    acc = got[got[:, 1] >= 0]
    assert len(acc) == len(fits) and len(fits) > 1000
    assert np.array_equal(acc[:, [0, 1]], fits[:, [0, 1]])          # same queries accepted, same factor kind
    assert np.array_equal(acc[:, 9:], fits[:, 9:])                   # identical 5-NN index lists
    edges = fits[:, 1] == 0
    # lines: a,b = centre +- 0.1 v ; the eigenvector sign is arbitrary (swaps a and b, residual norm unchanged)
    a_ok = np.abs(acc[edges, 2:8] - fits[edges, 2:8]).max(1) < 1e-9
    sw = np.concatenate([fits[edges, 5:8], fits[edges, 2:5]], axis=1)
    b_ok = np.abs(acc[edges, 2:8] - sw).max(1) < 1e-9
    assert np.all(a_ok | b_ok)
    assert np.abs(acc[~edges, 2:9] - fits[~edges, 2:9]).max() < 1e-10  # plane normals and offsets


def test_mapping_register_pose(ctx, orc, scene):
    cmap, smap, cs, ss, x0, (q2, t2) = scene
    m = orc.Mapping(); m.set_map(cmap, smap)
    xr, info = m.register(cs, ss, x0)
    xg, st = ctx.mapping_register(cs, ss, x0)
    assert info["optimised"]
    assert np.abs(xg[4:] - xr[4:]).max() < 1e-4 and rot_angle(xg[:4], xr[:4]) < 1e-4   # north-star tolerance
    assert np.abs(xg[4:] - xr[4:]).max() < 1e-7 and rot_angle(xg[:4], xr[:4]) < 1e-7
    assert np.abs(xg[4:] - t2).max() < np.abs(x0[4:] - t2).max()                          # and it moved towards the truth
    assert st["lm_iters"] == sum(int(s["num_iterations"]) for s in info["summaries"])


def test_thin_map_is_skipped(aloam, scene):
    cmap, smap, cs, ss, x0, _ = scene
    c = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=1000)
    c.map_upload(cmap[:5], smap[:20])
    x, st = c.mapping_register(cs, ss, x0)
    assert np.array_equal(x, x0) and st["flags"] & aloam.FLAG_MAP_TOO_THIN   # laserMapping.cpp:554,730-733
    c.close()


@pytest.mark.parametrize("leaf", [0.2, 0.4, 0.8])
def test_voxel_filter_matches_pcl_restatement(ctx, orc, synth, scans, leaf):
    """aloam_voxel_filter == pcl::VoxelGrid restatement (canonical tie order), bit for bit (laserMapping.cpp:543-549)"""
    ns, az, mr = synth.SENSORS["HDL-64"][:3]
    f = orc.Features(scans("HDL-64", 1), ns, mr)
    for cloud in (f.less_sharp, f.less_flat, f.full[:50000]):
        ref = orc.voxel_grid(cloud, leaf, orc.SORT_CANONICAL)
        got = ctx.voxel_filter(cloud, leaf)
        assert got.shape == ref.shape
        assert np.array_equal(got, ref)
    assert ctx.voxel_filter(np.zeros((0, 4), np.float32), leaf).shape == (0, 4)


def test_voxel_filter_overflow_returns_input(ctx):
    """PCL returns the input unchanged, bit for bit: -0.0 stays -0.0"""
    cloud = np.array([[0, 0, 0, 1], [3000, 3000, 3000, 2], [1, 1, 1, 3], [-0.0, 1, -0.0, 4]], np.float32)
    got = ctx.voxel_filter(cloud, 0.2)
    assert np.array_equal(got, cloud) and np.array_equal(got.view(np.uint32), cloud.view(np.uint32))


def test_map_upload_accepts_device_memory(aloam, scene):
    """aloam_map_upload infers the copy kind: a map resident in device memory gives the same pose as the host upload"""
    import torch
    cmap, smap, cs, ss, x0, _ = scene
    c = aloam.Aloam(n_scans=64, max_points=200000, max_map_points=len(cmap) + len(smap) + 1024)
    c.map_upload(cmap, smap)
    x_host, _ = c.mapping_register(cs, ss, x0)
    dc, ds = torch.from_numpy(np.ascontiguousarray(cmap)).cuda(), torch.from_numpy(np.ascontiguousarray(smap)).cuda()
    c.map_upload_ptr(dc.data_ptr(), dc.shape[0], ds.data_ptr(), ds.shape[0])
    x_dev, _ = c.mapping_register(cs, ss, x0)
    assert np.array_equal(x_host, x_dev)
    c.close()


def _same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_sharded_upload_on_one_rank_equals_map_upload(aloam, scene):
    """without a communicator this rank owns every cell, so aloam_map_upload_sharded cuts nothing away: host views of 4 and
    8 floats per point, streamed through the stack buffer a chunk at a time, and a device view index what aloam_map_upload
    indexes -- the same neighbours, fits and registered pose, bit for bit"""
    import torch
    cmap, smap, cs, ss, x0, _ = scene
    mp = 3500   # upload chunks of 3500 (4 floats per point) or 1750 (8 floats) points: both maps span several, the stacks fit
    assert max(len(cs), len(ss)) <= mp < min(len(cmap), len(smap))
    R = _rot(x0[:4])
    queries = []
    for q in (cs[:mp // 5], ss[:mp // 5]):   # k = 5 neighbours of at most max_points / 5 queries
        qw = q.copy(); qw[:, :3] = (q[:, :3].astype(np.float64) @ R.T + x0[4:]).astype(np.float32)
        queries.append(qw)

    def run(upload):
        c = aloam.Aloam(n_scans=64, max_points=mp, max_map_points=16384)
        upload(c)
        out = [*c.knn(2, queries[0], 5), *c.knn(3, queries[1], 5), c.mapping_associate(cs, ss, x0), c.mapping_register(cs, ss, x0)[0]]
        c.close()
        return out

    def wide(a):
        w = np.full((len(a), 8), -7.0, np.float32)
        w[:, :4] = a
        return w

    dc, ds = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (cmap, smap))
    ref = run(lambda c: c.map_upload(cmap, smap))
    for upload in (lambda c: c.map_upload_sharded(cmap, smap),
                   lambda c: c.map_upload_sharded(wide(cmap), wide(smap)),
                   lambda c: c.map_upload_sharded_ptr(dc.data_ptr(), len(cmap), ds.data_ptr(), len(smap))):
        got = run(upload)
        for g, r in zip(got[:4], ref[:4]):
            assert _same_bits(g, r)
        fits, ref_fits = got[4], ref[4]
        assert _same_bits(fits[:, 1], ref_fits[:, 1])
        acc = ref_fits[:, 1] >= 0   # the record of a rejected query is written only in part
        assert acc.sum() > 1000 and _same_bits(fits[acc], ref_fits[acc])
        assert _same_bits(got[5], ref[5])


# ---- the single-cloud filter at its size limits: > 1024 blocks of 1024 keys (k_vox_blockscan strides), voxel indices of 1 to
# 4 bytes (the sort always runs 4 passes over the 32-bit key; all-zero high digits leave a stable sort unchanged), runs across
# blocks, clouds near +-5 km

def _index_bytes(cloud, leaf):
    f = np.float32
    inv = f(1) / f(leaf)
    mn, mx = cloud[:, :3].min(0), cloud[:, :3].max(0)
    cells = 1
    for a in range(3):
        cells *= int(np.floor(f(mx[a]) * inv)) - int(np.floor(f(mn[a]) * inv)) + 1
    bits = 1
    while bits < 32 and (1 << bits) < cells:
        bits += 1
    return (bits + 7) // 8


@pytest.fixture(scope="module")
def big_ctx(aloam):
    c = aloam.Aloam(n_scans=16, max_points=1300000)
    yield c
    c.close()


def _cube_cloud(rng, n, centre, side):
    out = np.zeros((n, 4), np.float32)
    out[:, :3] = np.asarray(centre) + rng.uniform(-side / 2, side / 2, size=(n, 3))
    out[:, 3] = rng.uniform(0, 64, n)
    return out


@pytest.mark.parametrize("index_bytes,side", [(1, 1.0), (2, 6.0), (3, 40.0), (4, 70.0)])
def test_voxel_filter_radix_pass_counts(big_ctx, orc, index_bytes, side):
    rng = np.random.default_rng(index_bytes)
    cloud = _cube_cloud(rng, 200000, (-3.1, 7.7, 0.4), side)
    assert _index_bytes(cloud, 0.2) == index_bytes
    ref = orc.voxel_grid(cloud, 0.2, orc.SORT_CANONICAL)
    got = big_ctx.voxel_filter(cloud, 0.2)
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("sign", [1, -1])
def test_voxel_filter_1_3_million_points_near_5_km(big_ctx, orc, sign):
    """1.3 M points (1270 blocks of 1024 keys) around (+-4990, -+4990, 20) m; one voxel holds 5000 points, so its run
    crosses several blocks"""
    rng = np.random.default_rng(60 + sign)
    centre = (sign * 4990.0, -sign * 4990.0, 20.0)
    cloud = _cube_cloud(rng, 1300000, centre, 30.0)
    run = _cube_cloud(rng, 5000, (0, 0, 0), 0.15)
    run[:, :3] = np.floor(np.asarray(centre) / 0.4) * 0.4 + 0.2 + run[:, :3]
    cloud[rng.choice(len(cloud), 5000, replace=False)] = run
    ref = orc.voxel_grid(cloud, 0.4, orc.SORT_CANONICAL)
    got = big_ctx.voxel_filter(cloud, 0.4)
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
