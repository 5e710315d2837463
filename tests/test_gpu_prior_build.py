"""GPU: building the prior map from two map-frame clouds (aloam_prior_map_build).  Checked here: the built map against the oracle's
build (prior_build_cases.oracle_build: the cube rule, then the oracle's VoxelGrid per cube) bit for bit -- the store clouds of mapped snapshots, shuffled, non-default leaves, 1 M and
8 M-point synthetic maps, a cube whose index range overflows int; the cube rule's edges, non-finite points, far centres, stride 8,
every kind of input memory, empty clouds; the refusals, which change nothing; the memory a build and a clear give back; a built map
against the same map loaded from a snapshot (export and localising poses byte for byte) and against itself rebuilt; localisation
on a built map against the oracle's frozen frames, and on a map joined from two sessions."""
import numpy as np
import pytest

import lane_refs as R
import prior_build_cases as P

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
IDLE, SCAN, START = 0, 1, 2
N_MAP = 10


def _ctx(aloam, maxpts, batch=1, ns=16, **cfg):
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, max_ring_points=4096, max_map_points=400000, **cfg)


def _entries(dev, i0, i1):
    return [(d.data_ptr(), d.shape[0], START if i == i0 else SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def _run(ctx, entries):
    """one lane through aloam_scan_stream_lanes (mapped) -> (odometry rows, map rows)"""
    n = len(entries)
    ptrs, counts, ops = np.zeros((n, 1), np.uint64), np.zeros((n, 1), np.int64), np.zeros((n, 1), np.int32)
    for k, (p, c, op) in enumerate(entries):
        ptrs[k, 0], counts[k, 0], ops[k, 0] = p, c, op
    o, m = ctx.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
    return o[:, 0], m[:, 0]


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def _perturbed(pose7, dt, deg):
    h = np.radians(deg) / 2
    dq = np.array([0, 0, np.sin(h), np.cos(h)])
    x, y, z, w = pose7[:4]
    q = np.array([dq[3] * x + dq[0] * w + dq[1] * z - dq[2] * y, dq[3] * y - dq[0] * z + dq[1] * w + dq[2] * x,
                  dq[3] * z + dq[0] * y - dq[1] * x + dq[2] * w, dq[3] * w - dq[0] * x - dq[1] * y - dq[2] * z])
    return q, pose7[4:] + dt * np.array([1.0, -1.0, 0.5]) / 1.5


def _free():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


_WORLD = {}


def _world(aloam, synth, sensor="VLP-16", s0=0, n=N_MAP, extra=12):
    """a trajectory, and the snapshot, map poses and export of the lane that mapped its scans s0 .. s0 + n - 1"""
    key = (sensor, s0, n, extra)
    if key not in _WORLD:
        ns = synth.SENSORS[sensor][0]
        scans = R.traj(synth, 0, s0 + n + extra, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)
        M = R.maxn([scans]) + 1024
        dev = R.to_device(scans)
        c = _ctx(aloam, M, 1, ns)
        o, m = _run(c, _entries(dev, s0, s0 + n))
        blob = c.lane_save(0)
        exported = c.mapper_export(aloam.EXPORT_MAP, 0).copy()
        c.close()
        _WORLD[key] = {"scans": scans, "dev": dev, "M": M, "ns": ns, "blob": blob, "odom": o, "map": m, "export": exported}
    return _WORLD[key]


def _build(aloam, ctx, corner, surf, centre=None):
    dropped = ctx.prior_map_build(corner, surf, centre)
    return ctx.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).copy(), dropped


def _oracle(corner, surf, leaves, centre=(10, 10, 5)):
    return P.oracle_build(corner, surf, leaves[0], leaves[1], centre)


def _same(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("sensor,leaves", [("VLP-16", None), ("HDL-64", None), ("VLP-16", (0.55, 1.1))])
def test_snapshot_clouds_build_equals_the_oracle(aloam, synth, sensor, leaves):
    W = _world(aloam, synth, sensor)
    split = aloam.snapshot_store_clouds(W["blob"])
    leaves = leaves or synth.SENSORS[sensor][3:5]
    c = _ctx(aloam, W["M"], 1, W["ns"], line_res=leaves[0], plane_res=leaves[1])
    got, dropped = _build(aloam, c, split["corner"], split["surf"], split["centre"])
    ref, ref_dropped = _oracle(split["corner"], split["surf"], leaves, split["centre"])
    assert dropped == ref_dropped == (0, 0)
    assert _same(got, ref.export())
    # shuffled: another input order, another map where a voxel holds several points, still the oracle's for that order
    perm = [np.random.default_rng(s).permutation(len(split[k])) for s, k in ((1, "corner"), (2, "surf"))]
    sc, ss = split["corner"][perm[0]], split["surf"][perm[1]]
    got2, _ = _build(aloam, c, sc, ss, split["centre"])
    assert _same(got2, _oracle(sc, ss, leaves, split["centre"])[0].export())
    if leaves != synth.SENSORS[sensor][3:5]:
        assert not _same(got2, got)
    c.close()


_MAPS = {}


def _synth_map(aloam, synth, n):
    if n not in _MAPS:
        fx = _ctx(aloam, 200000, 1, 64)
        def feats(raw):
            f = fx.extract_features(raw)
            return f["less_sharp"], f["less_flat"]
        _MAPS[n] = synth.build_map(feats, n)
        fx.close()
    return _MAPS[n]


@pytest.mark.parametrize("n,leaves", [(1_000_000, (0.4, 0.8)), (8_000_000, (0.8, 1.0))])
def test_synthetic_maps_equal_the_oracle(aloam, synth, n, leaves):
    import torch
    corner, surf = _synth_map(aloam, synth, n)
    c = _ctx(aloam, 200000, 1, 64, line_res=leaves[0], plane_res=leaves[1])
    if n > 2_000_000:   # from device memory
        got, dropped = _build(aloam, c, torch.from_numpy(corner).cuda(), torch.from_numpy(surf).cuda())
    else:
        got, dropped = _build(aloam, c, corner, surf)
    ref, ref_dropped = _oracle(corner, surf, leaves)
    assert dropped == ref_dropped
    assert _same(got, ref.export())
    assert c.mapper_export_size(aloam.EXPORT_MAP, aloam.PRIOR_MAP) == len(got) and 0 < len(got) < n
    c.close()
    if n > 2_000_000:
        # at the HDL-64 leaves a corner cube of this map keeps more than 65536 points: refused, as the oracle's count says
        ref, _ = _oracle(corner, surf, (0.4, 0.8))
        assert np.diff(ref.packed()["cube_start"], axis=1).max() > 65536
        c = _ctx(aloam, 200000, 1, 64)
        _expect(aloam, ERR_CAPACITY, lambda: c.prior_map_build(corner, surf))
        _expect(aloam, ERR_STATE, lambda: c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP))   # no map was made
        c.close()


def test_a_cube_whose_index_range_overflows_comes_back_unfiltered(aloam):
    rng = np.random.default_rng(5)
    corner = rng.uniform(-24, 24, (3000, 4)).astype(np.float32)          # one cube: 48 m / 1 mm per axis overflows int
    corner[:1000, :3] = np.round(corner[:1000, :3])                       # duplicates that a filter would merge
    surf = rng.uniform(-100, 100, (5000, 4)).astype(np.float32)
    c = _ctx(aloam, 20000, line_res=0.001, plane_res=0.4)
    got, dropped = _build(aloam, c, corner, surf)
    ref, ref_dropped = _oracle(corner, surf, (0.001, 0.4))
    assert dropped == ref_dropped == (0, 0) and _same(got, ref.export())
    assert _same(ref.packed()["corner"], corner)   # kept unfiltered, in input order
    c.close()


def test_edges_non_finite_far_centres_strides_and_memory_kinds(aloam):
    import torch
    c = _ctx(aloam, 20000, line_res=0.2, plane_res=0.4)
    corner, surf = P.edge_clouds()
    got, dropped = _build(aloam, c, corner, surf)
    ref, ref_dropped = _oracle(corner, surf, (0.2, 0.4))
    assert dropped == ref_dropped and dropped[0] >= 45 and _same(got, ref.export())
    model, model_dropped = P.build_model(corner, surf, 0.2, 0.4)
    assert model_dropped == dropped and _same(ref.packed()["surf"], model["surf"])
    # stride 8 (PCL's PointXYZI), pinned and device memory: the same bytes
    pad = lambda a: np.ascontiguousarray(np.concatenate([a, np.full((len(a), 4), 7.0, np.float32)], axis=1))
    assert _same(_build(aloam, c, pad(corner), pad(surf))[0], got)
    for conv in (lambda a: torch.from_numpy(a).pin_memory(), lambda a: torch.from_numpy(a).cuda(), lambda a: torch.from_numpy(pad(a)).cuda()):
        g, d = _build(aloam, c, conv(corner), conv(surf))
        assert d == dropped and _same(g, got)
    # far centres: x + 25 = +-50 000 inside the buffer, and points outside it for a non-default centre
    far = P.far_clouds()
    for centre in ((-990, 10, 5), (1010, 10, 5), (10, -990, 1005), (2**20, -2**20, 5)):
        g, d = _build(aloam, c, far, far[:, [1, 0, 2, 3]].copy(), centre)
        r, rd = _oracle(far, far[:, [1, 0, 2, 3]].copy(), (0.2, 0.4), centre)
        assert d == rd and _same(g, r.export()), centre
    g, d = _build(aloam, c, corner, surf, (3, 17, 9))
    r, rd = _oracle(corner, surf, (0.2, 0.4), (3, 17, 9))
    assert d == rd and d != dropped and _same(g, r.export())
    # empty clouds: a valid, empty map
    e = np.zeros((0, 4), np.float32)
    g, d = _build(aloam, c, e, e)
    assert d == (0, 0) and len(g) == 0
    assert c.mapper_export_size(aloam.EXPORT_MAP, aloam.PRIOR_MAP) == 0
    c.close()


def test_refusals_change_nothing_and_memory_comes_back(aloam, synth):
    W = _world(aloam, synth)
    c = _ctx(aloam, W["M"], 2)
    c.prior_map_load(W["blob"])
    before = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes()
    init = _perturbed(W["map"][2], 0.1, 1.0)
    c.lane_localise(0, *init)
    # a cube of 42^3 points 0.9 m apart: more than 65536 voxels at plane_res 0.4
    g = np.arange(42, dtype=np.float32) * 0.9 - 18.0
    big = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    big = np.concatenate([big, np.zeros((len(big), 1), np.float32)], 1).astype(np.float32)
    _expect(aloam, ERR_CAPACITY, lambda: c.prior_map_build(big[:10], big))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.prior_map_build(big[:10], big[:10], (2**20 + 1, 10, 5)))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.prior_map_build(big[:10], big[:10], (10, -2**20 - 1, 5)))
    assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == before
    # the arming survived the refusals: lane 0's START localises as on a context that never saw them
    ref = _ctx(aloam, W["M"], 2)
    ref.prior_map_load(W["blob"])
    ref.lane_localise(0, *init)
    a, b = _run(c, _entries(W["dev"], 2, 6)), _run(ref, _entries(W["dev"], 2, 6))
    assert np.array_equal(a[1], b[1])
    # while lane 0 localises: refused, nothing changes, the lane goes on
    _expect(aloam, ERR_STATE, lambda: c.prior_map_build(big[:10], big[:10]))
    assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == before
    ref.close()
    c.reset_odometry()
    # a successful build keeps an arming, as a load does: the START localises against the new map
    c.lane_localise(1, *init)
    split = aloam.snapshot_store_clouds(W["blob"])
    c.prior_map_build(split["corner"], split["surf"], split["centre"])
    ptrs = np.array([[0, W["dev"][k].data_ptr()] for k in (2, 3)], np.uint64)
    counts = np.array([[0, W["dev"][k].shape[0]] for k in (2, 3)], np.int64)
    ops = np.array([[IDLE, START], [IDLE, SCAN]], np.int32)
    c.scan_stream_lanes(ptrs, counts, ops, True, mapped=True)
    st = c.mapper_state(1)   # lane 1 localises: it answers with the new map's centre and totals
    assert st["centre"] == split["centre"] and st["total_corner"] + st["total_surf"] == c.mapper_export_size(aloam.EXPORT_MAP, aloam.PRIOR_MAP)
    c.reset_odometry()
    # an emulating context refuses
    e = _ctx(aloam, W["M"], 1)
    assert aloam.lib().aloam_debug_shard_emulate(e._h, 0, 2, 0, 0) == 0
    _expect(aloam, ERR_STATE, lambda: e.prior_map_build(big[:10], big[:10]))
    e.close()
    # a build and a clear give the device memory back
    c.prior_map_clear()
    corner, surf = _synth_map(aloam, synth, 1_000_000)
    free0 = _free()
    c.prior_map_build(corner, surf)
    assert _free() < free0
    c.prior_map_clear()
    assert abs(_free() - free0) < (64 << 20), (free0, _free())
    c.close()


def _split_export(export, cube_start):
    """an export back into its corner and surf clouds, by the cube table"""
    cs = np.asarray(cube_start, np.int64)
    n = cs[:, 1:] - cs[:, :-1]
    kind = np.repeat(np.tile(np.array([0, 1], np.int8), P.NCUBE), n.T.ravel())
    return export[kind == 0], export[kind == 1]


def test_built_equals_loaded_and_a_rebuild_changes_nothing(aloam, synth, orc):
    W = _world(aloam, synth)
    split = aloam.snapshot_store_clouds(W["blob"])
    centre = (8, 11, 4)   # another window of the same map frame: the built map is not the snapshot's store
    built = _ctx(aloam, W["M"])
    got, dropped = _build(aloam, built, split["corner"], split["surf"], centre)
    ref, _ = _oracle(split["corner"], split["surf"], synth.SENSORS["VLP-16"][3:5], centre)
    packed = ref.packed()
    assert _same(got, ref.export())
    counts = P.store_counts(packed)
    assert (counts >= 0).sum(axis=1).max() <= 1024 and counts[0].max() <= 16384   # it fits snapshot format v1
    loaded = _ctx(aloam, W["M"])
    loaded.prior_map_load(P.snapshot_with_store(W["blob"], centre, counts, got))
    assert loaded.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == got.tobytes()
    init = _perturbed(np.array([0, 0, 0, 1.0, 0, 0, 0]), 0.2, 2.0)
    runs = []
    for c in (built, loaded):
        c.lane_localise(0, *init)
        runs.append(_run(c, _entries(W["dev"], 0, len(W["scans"]))))
        st = c.mapper_state(0)
        assert st["centre"] == centre
    assert runs[0][0].tobytes() == runs[1][0].tobytes() and runs[0][1].tobytes() == runs[1][1].tobytes()
    # the oracle's frozen frames on the oracle-built map
    import pyfrozen
    ns, _, mr, line_res, plane_res = synth.SENSORS["VLP-16"]
    odom, _ = R.oracle(orc, synth, W["scans"], ("localise", "VLP-16"), False, 0, "VLP-16")
    R.assert_near(runs[0][0], odom, "odometry")
    loc = pyfrozen.Localiser(ref.frozen(), *init)
    poses = []
    for k, raw in enumerate(W["scans"]):
        f = orc.Features(raw, ns, mr)
        pose, info = loc.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], line_res, plane_res)
        poses.append(pose)
    R.assert_near(runs[0][1], np.array(poses), "map poses on a built map")
    # idempotence: the built map's own clouds build the same map
    built.reset_odometry()
    c_again, s_again = _split_export(got, packed["cube_start"])
    again, d2 = _build(aloam, built, c_again, s_again, centre)
    assert d2 == (0, 0) and again.tobytes() == got.tobytes()
    built.close(); loaded.close()


def _moved(cloud, R3, t):
    out = cloud.copy()
    out[:, :3] = (cloud[:, :3].astype(np.float64) @ R3.T + t).astype(np.float32)
    return out


def _compose(R3, t, pose7):
    """(R3, t) * pose7 as a pose7 (xyzw quaternion)"""
    from scipy.spatial.transform import Rotation
    r = Rotation.from_matrix(R3) * Rotation.from_quat(pose7[:4])
    return np.concatenate([r.as_quat(), R3 @ pose7[4:] + t])


def test_a_map_joined_from_two_sessions(aloam, synth):
    """session A maps scans 0-9, session B scans 10-21 from its own origin; B's clouds are moved into A's frame by the ground truth
    and the two are built into one map; a third drive over scans 5-21 localises from A's area into B's"""
    A = _world(aloam, synth, "VLP-16", 0, 10, 12)
    B = _world(aloam, synth, "VLP-16", 10, 12, 0)
    qa, ta = synth.pose(0)
    qb, tb = synth.pose(10)
    Ra, Rb = synth.rotation_matrix(qa), synth.rotation_matrix(qb)
    R_ab, t_ab = Ra.T @ Rb, Ra.T @ (tb - ta)          # B's map frame (its scan 10) in A's
    sa, sb = aloam.snapshot_store_clouds(A["blob"]), aloam.snapshot_store_clouds(B["blob"])
    corner = np.concatenate([sa["corner"], _moved(sb["corner"], R_ab, t_ab)])
    surf = np.concatenate([sa["surf"], _moved(sb["surf"], R_ab, t_ab)])
    c = _ctx(aloam, max(A["M"], B["M"]))
    dropped = c.prior_map_build(corner, surf)
    assert dropped == (0, 0)
    init = _perturbed(A["map"][5], 0.15, 1.5)
    c.lane_localise(0, *init)
    _, m = _run(c, _entries(A["dev"], 5, 22))
    expect = np.concatenate([A["map"][5:10], np.array([_compose(R_ab, t_ab, p) for p in B["map"]])])
    dt, dr = R.deviation(m[2:], expect[2:])   # after two scans the initial error is gone
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    c.close()
