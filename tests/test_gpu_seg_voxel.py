"""GPU parity: the segmented VoxelGrid of the mapper (voxel.cu, the per-cube re-filter of laserMapping.cpp:787-801 and the
stack filters of :543-549) through aloam_debug_seg_voxel_filter, bit for bit against the pcl::VoxelGrid restatement
(canonical tie order), segment by segment.  Covers the paths a frame of normal size never reaches: runs of one voxel that
continue across blocks of 1024 sorted keys, several sort tiles per CTA of the cooperative radix sort, segment windows when
the index bits leave no room for all segment numbers, and the two pass-through cases (PCL's index overflow, key overflow)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

INT_MAX = 2**31 - 1
LEAVES = (0.1, 0.2, 0.4, 0.8)


def index_range(cloud, leaf):
    """PCL's index range in float32 arithmetic: (dxyz product, cells of the key)"""
    f = np.float32
    inv = f(1) / f(leaf)
    mn, mx = cloud[:, :3].min(0), cloud[:, :3].max(0)
    d = [int((f(mx[a]) - f(mn[a])) * inv) + 1 for a in range(3)]
    div = [int(np.floor(f(mx[a]) * inv)) - int(np.floor(f(mn[a]) * inv)) + 1 for a in range(3)]
    return d[0] * d[1] * d[2], div[0] * div[1] * div[2]


def expected(orc, cloud, leaf, idx_bits):
    """(filtered cloud, key overflow?) as the device must give it"""
    if len(cloud) == 0:
        return cloud, False
    dprod, cells = index_range(cloud, leaf)
    if dprod > INT_MAX:
        return cloud, False                       # PCL: "leaf size is too small", input unchanged
    if cells > 2**idx_bits:
        return cloud, True                        # cannot be encoded: unchanged and flagged
    return orc.voxel_grid(cloud, leaf, orc.SORT_CANONICAL), False


def check(ctx, orc, segs, leaves, idx_bits):
    got, err = ctx.seg_voxel_filter(segs, leaves, idx_bits)
    assert len(got) == len(segs)
    any_key = False
    for s, (cloud, leaf, g) in enumerate(zip(segs, leaves, got)):
        ref, key = expected(orc, cloud, leaf, idx_bits)
        any_key |= key
        assert g.shape == ref.shape, (s, leaf, g.shape, ref.shape)
        assert np.array_equal(g.view(np.uint32), ref.view(np.uint32)), (s, leaf)
    assert err == (1 if any_key else 0)
    return got


def cluster_cloud(rng, n, centre=(0, 0, 0), side=8.0, leaf=0.2):
    """n points in a box of `side` metres: a third on a half-leaf lattice (exact repeats, multi-point voxels), the rest
    spread, so voxels hold 1 to many points in input order that is not sorted"""
    c = np.asarray(centre, np.float64)
    k = n // 3
    lat = rng.integers(-int(side / leaf), int(side / leaf), size=(k, 3)) * (leaf / 2)
    spread = rng.uniform(-side / 2, side / 2, size=(n - k, 3))
    xyz = np.concatenate([lat, spread]) + c
    rng.shuffle(xyz)
    out = np.zeros((n, 4), np.float32)
    out[:, :3] = xyz
    out[:, 3] = rng.uniform(0, 16, n)
    return out


@pytest.fixture(scope="module")
def ctx(aloam):
    # slab capacities 16384 / 20000 -> sort buffers of 75 * 36384 = 2.7 M keys
    c = aloam.Aloam(n_scans=16, max_points=20000, max_map_points=20000)
    yield c
    c.close()


def _segments(rng, n_segs):
    """empty segments first, in the middle and last, single-point segments, the four leaves mixed"""
    segs, leaves = [], []
    for s in range(n_segs):
        leaf = LEAVES[s % 4]
        if s == 0 or s == n_segs // 2 or (s == n_segs - 1 and n_segs > 1):
            cloud = np.zeros((0, 4), np.float32)
        elif s % 7 == 3:
            cloud = cluster_cloud(rng, 1, leaf=leaf)
        else:
            cloud = cluster_cloud(rng, int(rng.integers(2, 700)), centre=rng.uniform(-300, 300, 3), side=float(rng.uniform(1, 10)), leaf=leaf)
        segs.append(cloud)
        leaves.append(leaf)
    return segs, leaves


@pytest.mark.parametrize("idx_bits", [31, 28, 24])
@pytest.mark.parametrize("n_segs", [1, 2, 75, 150, 160])
def test_segment_counts_and_windows(ctx, orc, n_segs, idx_bits):
    """idx_bits 31 / 28 / 24: windows of 2, of 16, none; 75 and 150 are not multiples of either window"""
    rng = np.random.default_rng(1000 * n_segs + idx_bits)
    segs, leaves = _segments(rng, n_segs)
    check(ctx, orc, segs, leaves, idx_bits)


@pytest.mark.parametrize("idx_bits", [31, 24])
def test_block_boundary_sizes(ctx, orc, idx_bits):
    """segments of 1023, 1024, 1025 and 4097 points: segment and block boundaries fall on, before and after each other"""
    rng = np.random.default_rng(7 + idx_bits)
    segs = [cluster_cloud(rng, n, centre=rng.uniform(-50, 50, 3), side=6.0) for n in (1023, 1024, 1025, 4097, 1, 1024)]
    check(ctx, orc, segs, [0.2, 0.1, 0.4, 0.2, 0.8, 0.1], idx_bits)


def test_several_sort_tiles_per_cta(ctx, orc):
    """320 k keys in one pass: more than one tile of 1024 keys per CTA of the cooperative radix sort"""
    rng = np.random.default_rng(5)
    segs = [cluster_cloud(rng, n, centre=rng.uniform(-20, 20, 3), side=12.0) for n in (90000, 1, 150000, 80001)]
    segs.insert(2, np.zeros((0, 4), np.float32))
    got = check(ctx, orc, segs, [0.1, 0.2, 0.4, 0.2, 0.8], 24)
    assert sum(len(s) for s in segs) > 300000 and len(got[0]) < len(segs[0])


def test_long_runs_cross_blocks(ctx, orc):
    """one voxel of 5000 points (its run crosses at least four block boundaries), runs of 1, 3 and 1025 points, and two
    adjacent segments with the same geometry (equal voxel indices, different segment numbers)"""
    rng = np.random.default_rng(17)
    leaf = 0.2
    big = np.zeros((5000, 4), np.float32)
    big[:, :3] = 1.05 + rng.uniform(0, 0.09, size=(5000, 3))      # voxel (5, 5, 5) of a 0.2 leaf
    big[:, 3] = rng.uniform(0, 100, 5000)
    r1025 = big[:1025].copy(); r1025[:, 0] += 1.0
    r3 = big[:3].copy(); r3[:, 1] -= 6.0
    r1 = big[:1].copy(); r1[:, 2] += 3.0
    seg_a = np.concatenate([big, r3, r1025, r1, cluster_cloud(rng, 700, side=4.0)])
    seg_a = seg_a[rng.permutation(len(seg_a))]
    seg_b = seg_a.copy()                                          # same voxels, next segment
    seg_c = big[:1500].copy()                                     # one voxel: a single run
    for idx_bits in (31, 28, 24):
        got = check(ctx, orc, [seg_a, seg_b, seg_c, seg_a[:1024]], [leaf] * 4, idx_bits)
        assert len(got[2]) == 1


def test_coordinates_at_the_edges(ctx, orc):
    """points on exact multiples of the leaf, negative coordinates, clouds near +-5 km, a one-voxel cloud, a flat cloud"""
    rng = np.random.default_rng(23)
    segs, leaves = [], []
    for leaf in LEAVES:
        lat = np.zeros((2000, 4), np.float32)
        lat[:, :3] = (rng.integers(-40, 40, size=(2000, 3)) * np.float32(leaf)).astype(np.float32)   # on voxel faces
        lat[:, 3] = rng.uniform(0, 1, 2000)
        segs.append(lat); leaves.append(leaf)
        neg = cluster_cloud(rng, 1500, centre=(-30.3, -12.7, -4.1), side=5.0, leaf=leaf)
        segs.append(neg); leaves.append(leaf)
        for sign in (1, -1):
            far = cluster_cloud(rng, 1500, centre=(sign * 4999.0, sign * -4998.5, sign * 37.0), side=6.0, leaf=leaf)
            segs.append(far); leaves.append(leaf)
    one = np.full((300, 4), 0.5, np.float32); one[:, :3] += rng.uniform(0, 0.04, size=(300, 3)).astype(np.float32)
    segs.append(one); leaves.append(0.1)
    flat = cluster_cloud(rng, 2000, side=10.0); flat[:, 2] = np.float32(1.3)
    segs.append(flat); leaves.append(0.2)
    for idx_bits in (31, 24):
        check(ctx, orc, segs, leaves, idx_bits)


def test_pcl_overflow_segment_passes_through(ctx, orc):
    """a segment whose index range overflows PCL's int comes back unchanged (bit for bit: -0.0 stays -0.0), without an
    error, between normal ones"""
    rng = np.random.default_rng(29)
    huge = cluster_cloud(rng, 3000, side=4.0)
    huge[:2] = [[-2000.0, -2000.0, -2000.0, 1.0], [2000.0, 2000.0, 2000.0, 2.0]]
    huge[2, 0] = huge[3, 1] = huge[4, 2] = np.float32(-0.0)
    assert index_range(huge, 0.1)[0] > INT_MAX
    segs = [cluster_cloud(rng, 2500, side=6.0), huge, cluster_cloud(rng, 1800, side=3.0)]
    for idx_bits in (31, 28):
        got = check(ctx, orc, segs, [0.2, 0.1, 0.4], idx_bits)
        assert np.array_equal(got[1], huge)


@pytest.mark.parametrize("idx_bits", [31, 24])
def test_key_overflow_segment_is_flagged(ctx, orc, idx_bits):
    """a segment whose voxel index needs more than idx_bits bits (but not more than PCL's int): err bit 0, that segment
    unchanged (bit for bit: -0.0 stays -0.0), every other segment still exact.  For 31 bits: a 25.79 m box at leaf 0.02 off
    the voxel lattice gives dxyz = 1290^3 <= INT_MAX but 1291^3 > 2^31 cells; aloam_voxel_filter, whose key is PCL's whole
    32-bit index, filters that cloud exactly"""
    rng = np.random.default_rng(31 + idx_bits)
    if idx_bits == 31:
        leaf, lo = 0.02, np.float32(-12.887)
        bad = (rng.uniform(0, 1, size=(2000, 4)) * [25.79, 25.79, 25.79, 1] + [lo, lo, lo, 0]).astype(np.float32)
        bad[0, :3] = lo; bad[1, :3] = np.float32(lo + np.float32(25.79))
    else:
        leaf = 0.1
        bad = cluster_cloud(rng, 2000, side=30.0, leaf=leaf)
    bad[2, 0] = bad[3, 1] = bad[4, 2] = np.float32(-0.0)
    dprod, cells = index_range(bad, leaf)
    assert dprod <= INT_MAX and cells > 2**idx_bits
    segs = [cluster_cloud(rng, 1200, side=5.0), bad, np.zeros((0, 4), np.float32), cluster_cloud(rng, 3000, side=8.0)]
    got = check(ctx, orc, segs, [0.2, leaf, 0.4, 0.1], idx_bits)
    assert np.array_equal(got[1], bad)
    if idx_bits == 31:
        assert cells <= 2**32
        ref = orc.voxel_grid(bad, leaf, orc.SORT_CANONICAL)
        one = ctx.voxel_filter(bad, leaf)
        assert one.shape == ref.shape and np.array_equal(one.view(np.uint32), ref.view(np.uint32))


def test_debug_filter_leaves_the_mapper_alone(aloam, orc):
    """mapper_step frames with debug filter and voxel_filter calls between them give the same results as without, and
    voxel_filter, which has a segmented filter of its own, stays exact between the mapper's filters"""
    rng = np.random.default_rng(37)
    frames = []
    for k in range(4):
        q = np.array([0.0, 0.0, np.sin(0.1 * k), np.cos(0.1 * k)])
        frames.append((cluster_cloud(rng, 40, side=20.0), cluster_cloud(rng, 4000, side=60.0, leaf=0.4), q, np.array([20.0 * k, -7.0 * k, 1.5 * k])))
    runs = []
    for interleave in (False, True):
        c = aloam.Aloam(n_scans=16, max_points=20000, max_map_points=50000)
        c.mapper_reset()
        out = []
        for corner, surf, q, t in frames:
            if interleave:
                one = c.voxel_filter(surf, 0.4)
                c.seg_voxel_filter([cluster_cloud(rng, 5000, side=9.0), surf[:3000]], [0.1, 0.2], 28)
                ref = orc.voxel_grid(surf, 0.4, orc.SORT_CANONICAL)
                assert np.array_equal(one.view(np.uint32), ref.view(np.uint32))
                ref = orc.voxel_grid(corner, 0.2, orc.SORT_CANONICAL)
                assert np.array_equal(c.voxel_filter(corner, 0.2).view(np.uint32), ref.view(np.uint32))
            out.append(np.concatenate(c.mapper_step(corner, surf, q, t)[:2]))
        st = c.mapper_state()
        out.append(np.concatenate([st["q_wmap_wodom"], st["t_wmap_wodom"]]))
        out += [c.mapper_cube(w, i) for i in st["valid"] for w in (0, 1)]
        runs.append(out)
        c.close()
    assert len(runs[0]) == len(runs[1])
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


def test_limits_are_capacity_errors(aloam, ctx):
    """more than 160 segments, or more points than the sort buffers hold: ALOAM_ERR_CAPACITY, nothing runs"""
    with pytest.raises(aloam.AloamError) as e:
        ctx.seg_voxel_filter([np.zeros((1, 4), np.float32)] * 161, [0.2] * 161)
    assert e.value.code == -4
    cap = 75 * (16384 + 20000)
    with pytest.raises(aloam.AloamError) as e:
        ctx.seg_voxel_filter([np.zeros((cap // 2 + 1, 4), np.float32)] * 2, [0.2, 0.2])
    assert e.value.code == -4
    got, err = ctx.seg_voxel_filter([np.ones((3, 4), np.float32)], [0.2])
    assert err == 0 and np.array_equal(got[0], np.ones((1, 4), np.float32))
