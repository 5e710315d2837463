"""GPU: localisation against a prior map (aloam_prior_map_load, aloam_lane_localise).  The prior map is the store a mapping lane
saved; lanes armed with an initial T_wmap_wodom register their scans against it through the persistent index and never change it.
Checked here: every localising frame against the mapping frame of the existing device path started from the same store and
T_wmap_wodom (bit for bit); many lanes on one map against their solo runs; lanes of all three modes in one context; the prior map's
bytes before and after; the registered sink; mapping_skip_frame; launch counts; refusals that leave the state untouched."""
import struct

import numpy as np
import pytest

import lane_refs as R
import pyclouds

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_STATE, ERR_SNAPSHOT = -1, -9, -11
IDLE, SCAN, START = 0, 1, 2
N_MAP = 10   # scans the prior map is built from


def _ctx(aloam, maxpts, batch=1, ns=16, **cfg):
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, max_ring_points=4096, max_map_points=400000, **cfg)


def _entries(dev, i0, i1):
    """scans i0 .. i1-1 of a device-resident trajectory as lane entries; the first one STARTs the lane's trajectory"""
    return [(d.data_ptr(), d.shape[0], START if i == i0 else SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def _call(ctx, batch, lanes, mapped=True, first_step=None):
    """one aloam_scan_stream_lanes call; lanes = {lane: entries}, lane l idle for first_step[l] steps before them and after them
    -> {lane: (odometry rows, map rows)} of its entries"""
    first_step = first_step or {}
    steps = max(first_step.get(l, 0) + len(e) for l, e in lanes.items())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for lane, entries in lanes.items():
        for k, (p, n, op) in enumerate(entries, first_step.get(lane, 0)):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    o, m = ctx.scan_stream_lanes(ptrs, counts, ops, True, mapped=mapped)
    out = {}
    for lane, e in lanes.items():
        s = slice(first_step.get(lane, 0), first_step.get(lane, 0) + len(e))
        out[lane] = (o[s, lane], m[s, lane] if mapped else None)
    return out


def _perturbed(pose7, dt, deg):
    """pose7 moved by dt metres along (1, -1, 0.5) / 1.5 and turned by deg degrees about z, as (q, t)"""
    h = np.radians(deg) / 2
    dq = np.array([0, 0, np.sin(h), np.cos(h)])
    x, y, z, w = pose7[:4]
    q = np.array([dq[3] * x + dq[0] * w + dq[1] * z - dq[2] * y, dq[3] * y - dq[0] * z + dq[1] * w + dq[2] * x,
                  dq[3] * z + dq[0] * y - dq[1] * x + dq[2] * w, dq[3] * w - dq[0] * x - dq[1] * y - dq[2] * z])
    return q, pose7[4:] + dt * np.array([1.0, -1.0, 0.5]) / 1.5


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


_WORLD = {}


def _world(aloam, synth, sensor="VLP-16", **cfg):
    """a trajectory, the snapshot of the lane that mapped its first N_MAP scans, that lane's map poses and exported map"""
    key = (sensor, tuple(sorted(cfg.items())))
    if key not in _WORLD:
        ns = synth.SENSORS[sensor][0]
        scans = R.traj(synth, 0, N_MAP + 12, sensor=sensor, n_az=900 if sensor == "VLP-16" else 600)
        M = R.maxn([scans]) + 1024
        dev = R.to_device(scans)
        c = _ctx(aloam, M, 1, ns, **cfg)
        o, m = _call(c, 1, {0: _entries(dev, 0, N_MAP)})[0]
        blob = c.lane_save(0)
        exported = c.mapper_export(aloam.EXPORT_MAP, 0).copy()
        state = c.mapper_state(0)
        c.close()
        _WORLD[key] = {"scans": scans, "dev": dev, "M": M, "ns": ns, "blob": blob, "odom": o, "map": m, "export": exported, "state": state}
    return _WORLD[key]


def _localiser(aloam, W, batch=1, **cfg):
    c = _ctx(aloam, W["M"], batch, W["ns"], **cfg)
    c.prior_map_load(W["blob"])
    return c


def _rebased(W, s):
    """the initial T_wmap_wodom of a vehicle whose first scan is scan s of the mapped trajectory: its map pose there"""
    return W["map"][s].copy()


def test_every_frame_equals_the_mapping_frame_from_the_same_store(aloam, synth):
    """frame j of a localising lane == aloam_mapper_step on a scratch context whose lane 0 was restored from the prior snapshot
    with the lane's T_wmap_wodom patched in at the documented offsets, fed the same clouds and odometry pose"""
    W = _world(aloam, synth)
    s0, n = 2, 8
    loc = _localiser(aloam, W)
    before = loc.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes()
    assert before == W["export"].tobytes()   # the prior map is the source lane's store, in its export order
    q0, t0 = _perturbed(_rebased(W, s0), 0.25, 3.0)
    loc.lane_localise(0, 2.0 * q0, t0)       # a finite quaternion is normalised: q / sqrt(q . q), summed in index order
    n2 = 0.0
    for v in 2.0 * q0:
        n2 += float(v) * float(v)
    q0 = 2.0 * q0 / np.sqrt(n2)
    scratch, feats = _ctx(aloam, W["M"]), _ctx(aloam, W["M"])
    blob = bytearray(W["blob"].tobytes())
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    S = 256 + 16 * (nls + nlf)
    T = np.concatenate([q0, t0])
    entries = _entries(W["dev"], s0, s0 + n)
    for j in range(n):
        o, m = _call(loc, 1, {0: [entries[j]]})[0]
        struct.pack_into("<4d", blob, S + 536, *T[:4])
        struct.pack_into("<3d", blob, S + 568, *T[4:])
        scratch.lane_restore(0, np.frombuffer(bytes(blob), np.uint8))
        f = feats.extract_features(W["scans"][s0 + j])
        q, t, st = scratch.mapper_step(f["less_sharp"], f["less_flat"], o[0][:4], o[0][4:])
        assert not st["flags"] & aloam.FLAG_MAP_TOO_THIN
        assert np.array_equal(m[0], np.concatenate([q, t])), "frame %d" % j
        sl, ss = loc.mapper_state(0), scratch.mapper_state(0)
        assert sl["centre"] == ss["centre"] == W["state"]["centre"] and sl["valid"] == ss["valid"], "frame %d" % j   # no shift happened
        assert np.array_equal(sl["q_wmap_wodom"], ss["q_wmap_wodom"]) and np.array_equal(sl["t_wmap_wodom"], ss["t_wmap_wodom"])
        assert (sl["total_corner"], sl["total_surf"]) == (W["state"]["total_corner"], W["state"]["total_surf"])
        T = np.concatenate([sl["q_wmap_wodom"], sl["t_wmap_wodom"]])
    # the initial error is gone: the last refined pose is the one the mapping lane had found for that scan, to a few centimetres
    dt, dr = R.deviation(m[:1], W["map"][s0 + n - 1:s0 + n])
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    assert loc.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == before   # never written
    for c in (loc, scratch, feats):
        c.close()


@pytest.mark.parametrize("sensor,cfg", [("VLP-16", {}), ("HDL-32", {}), ("VLP-16", {"distortion": 1, "mapping_skip_frame": 3})])
def test_a_localising_trajectory_follows_the_frozen_oracle(aloam, synth, orc, sensor, cfg):
    """22 scans from an initial pose 0.2 m and 2 degrees off: the map poses against the oracle's frozen frames (oracle features and
    odometry, the prior map parsed from the snapshot), and the window of the last registered scan"""
    import pyfrozen
    W = _world(aloam, synth, sensor, **cfg)
    skip, n = cfg.get("mapping_skip_frame", 1), len(W["scans"])
    init = _perturbed(np.array([0, 0, 0, 1.0, 0, 0, 0]), 0.2, 2.0)
    c = _localiser(aloam, W, 1, **cfg)
    c.lane_localise(0, *init)
    o, m = _call(c, 1, {0: _entries(W["dev"], 0, n)})[0]
    st = c.mapper_state(0)
    c.close()
    # the oracle's side
    blob = W["blob"].tobytes()
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    S = 256 + 16 * (nls + nlf)
    counts = np.frombuffer(blob, np.int32, 2 * 4851, S + 592).reshape(2, 4851)
    points = np.frombuffer(blob, np.float32, offset=S + 39424).reshape(-1, 4)
    frozen = pyfrozen.FrozenMap.from_export(struct.unpack_from("<3i", blob, S), counts, points)
    ns, _, mr, line_res, plane_res = synth.SENSORS[sensor]
    odom, _ = R.oracle(orc, synth, W["scans"], ("localise", sensor), False, cfg.get("distortion", 0), sensor)
    R.assert_near(o, odom, "odometry")
    loc = pyfrozen.Localiser(frozen, *init, skip=skip)
    ref = []
    for k, raw in enumerate(W["scans"]):
        f = orc.Features(raw, ns, mr)
        pose, info = loc.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], line_res, plane_res)
        assert info is None or info["optimised"] == 1
        ref.append(pose)
    R.assert_near(m, np.array(ref), "map poses of the localising lane")
    assert st["valid"] == loc.valid and st["centre"] == frozen.centre
    # and the lane found the mapped trajectory again
    dt, dr = R.deviation(m[N_MAP - 1:N_MAP], W["map"][N_MAP - 1:N_MAP])
    assert dt < 0.1 and dr < 0.02, (dt, dr)


_SOLO = {}


def _solo(aloam, W, s0, n, init, **cfg):
    key = (id(W), s0, n, init[0].tobytes(), init[1].tobytes(), tuple(sorted(cfg.items())))
    if key not in _SOLO:
        c = _localiser(aloam, W, 1, **cfg)
        c.lane_localise(0, *init)
        _SOLO[key] = _call(c, 1, {0: _entries(W["dev"], s0, s0 + n)})[0]
        c.close()
    return _SOLO[key]


@pytest.mark.parametrize("width", [5, 16])
def test_lanes_on_one_prior_map_equal_their_solo_runs(aloam, synth, width):
    W = _world(aloam, synth)
    c = _localiser(aloam, W, width)
    free0 = _free()
    plan = {}
    for l in range(width):
        s0, n = l % 5, 5 + l % 3
        plan[l] = (s0, n, _perturbed(_rebased(W, s0), 0.05 * (l % 4), 0.5 * (l % 5)))
        c.lane_localise(l, *plan[l][2])
    got = _call(c, width, {l: _entries(W["dev"], s0, s0 + n) for l, (s0, n, _) in plan.items()}, first_step={l: l % 3 for l in plan})
    for l, (s0, n, init) in plan.items():
        ref = _solo(aloam, W, s0, n, init)
        assert np.array_equal(got[l][0], ref[0]) and np.array_equal(got[l][1], ref[1]), "lane %d" % l
    assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == W["export"].tobytes()
    # lanes that only localise own no cube store (1.34 GB of slabs each): `width` of them stay far below one store
    assert free0 - _free() < (1 << 30), free0 - _free()
    _expect(aloam, ERR_STATE, lambda: c.mapper_export(aloam.EXPORT_MAP, width - 1))
    c.close()


def _free():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def test_mapping_localising_and_odometry_lanes_in_one_context_and_launch_counts(aloam, synth):
    W = _world(aloam, synth)
    n = 6
    init = _perturbed(_rebased(W, 2), 0.1, 1.0)
    c = _localiser(aloam, W, 3)
    od = _call(c, 3, {2: _entries(W["dev"], 0, n)}, mapped=False)[2]   # odometry only
    c.lane_localise(1, *init)
    r = _call(c, 3, {0: _entries(W["dev"], 0, n), 1: _entries(W["dev"], 2, 2 + n)})   # lane 0 maps, lane 1 localises
    ref_loc = _solo(aloam, W, 2, n, init)
    assert np.array_equal(r[1][0], ref_loc[0]) and np.array_equal(r[1][1], ref_loc[1])
    assert np.array_equal(r[0][0], W["odom"][:n]) and np.array_equal(r[0][1], W["map"][:n])   # the mapping lane: its solo run
    assert np.array_equal(od[0], W["odom"][:n])
    assert c.mapper_state(0)["total_surf"] > 0 and c.mapper_state(1)["total_surf"] == W["state"]["total_surf"]
    c.close()

    def launches(mode, batch=1):
        """launches of one call of n steps; the call is made twice, the first creating what the lanes own (a store's reset is a launch)"""
        x = _localiser(aloam, W, batch)
        for _ in range(2):
            x.reset_odometry()
            for l in range(batch):
                if mode == "loc" or (mode == "mixed" and l == 1):
                    x.lane_localise(l, *init)
            a = x.launch_count()
            _call(x, batch, {l: _entries(W["dev"], 2, 2 + n) for l in range(batch)}, mapped=mode != "odo")
            a = x.launch_count() - a
        x.close()
        return a
    odo, mp, loc1, loc16, mixed = launches("odo"), launches("map"), launches("loc"), launches("loc", 16), launches("mixed", 2)
    assert mp - odo == 38 * n                      # the mapping frame issues what it issued before localisation existed
    assert loc1 == loc16 and 0 < loc1 - odo < mp - odo   # one locate frame serves 1 or 16 lanes, with fewer launches
    assert mixed == mp + (loc1 - odo)              # side by side: each group's frame once per step


def test_skip_frames_registered_sink_and_deskew(aloam, synth):
    import torch
    W = _world(aloam, synth, mapping_skip_frame=3, distortion=1)
    n, s0 = 8, 1
    init = _perturbed(_rebased(W, s0), 0.1, 1.0)
    c = _localiser(aloam, W, 2, mapping_skip_frame=3, distortion=1)
    sink = torch.zeros((n * W["M"], 4), dtype=torch.float32, device="cuda")
    c.set_registered_sink(sink)
    c.lane_localise(1, *init)
    o, m = _call(c, 2, {1: _entries(W["dev"], s0, s0 + n)})[1]
    begin, count = c.registered_rows(2 * n)
    feats = _ctx(aloam, W["M"], distortion=1)
    for j in range(n):
        r = 2 * j + 1
        if j % 3 == 0:   # registered: its row is the full cloud moved by the refined pose
            full = feats.extract_features(W["scans"][s0 + j])["full"]
            assert count[r] == full.shape[0]
            assert np.array_equal(sink[begin[r]:begin[r] + count[r]].cpu().numpy(), pyclouds.associate_to_map(m[j], full))
        else:
            assert count[r] == 0
    # skipped scans: the high-frequency pose composed from the T_wmap_wodom of the lane's latest registered scan
    st = c.mapper_state(1)
    ref = _solo(aloam, W, s0, n, init, mapping_skip_frame=3, distortion=1)
    assert np.array_equal(m, ref[1]) and np.array_equal(o, ref[0])
    assert not np.array_equal(m[1, 4:], o[1, 4:]) and not np.array_equal(m[7], m[6])
    assert st["valid"] and len(st["valid"]) <= 75
    c.close(); feats.close()


def test_refusals_leave_the_state_untouched(aloam, synth):
    W = _world(aloam, synth)
    ident = (np.array([0, 0, 0, 1.0]), np.zeros(3))
    c = _ctx(aloam, W["M"], 2)
    _expect(aloam, ERR_STATE, lambda: c.lane_localise(0, *ident))                      # no prior map
    _expect(aloam, ERR_STATE, lambda: c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP))
    c.prior_map_clear()                                                                # nothing to release: fine
    unmapped = _ctx(aloam, W["M"], 1)
    _call(unmapped, 1, {0: _entries(W["dev"], 0, 2)}, mapped=False)
    _expect(aloam, ERR_SNAPSHOT, lambda: c.prior_map_load(unmapped.lane_save(0)))      # an unmapped snapshot
    unmapped.close()
    _expect(aloam, ERR_SNAPSHOT, lambda: c.prior_map_load(W["blob"][:-16]))
    nls, nlf = struct.unpack_from("<ii", W["blob"].tobytes(), 28)
    bad = bytearray(W["blob"].tobytes())
    struct.pack_into("<i", bad, 256 + 16 * (nls + nlf) + 12, 126)                      # a valid list of 126 entries
    _expect(aloam, ERR_SNAPSHOT, lambda: c.prior_map_load(bytes(bad)))
    other = _ctx(aloam, W["M"], 1, line_res=0.3)
    _expect(aloam, ERR_SNAPSHOT, lambda: other.prior_map_load(W["blob"]))              # another configuration
    other.close()
    c.prior_map_load(W["blob"])
    for q, t in ((np.zeros(4), np.zeros(3)), (np.array([0, 0, np.nan, 1.0]), np.zeros(3)), (ident[0], np.array([0, np.inf, 0]))):
        _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_localise(0, q, t))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_localise(2, *ident))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.mapper_export(aloam.EXPORT_SURROUND, aloam.PRIOR_MAP))
    # aloam_reset_odometry drops an arming: the next mapped START maps
    c.lane_localise(0, *ident)
    c.reset_odometry()
    r = _call(c, 2, {0: _entries(W["dev"], 0, 3)})[0]
    assert np.array_equal(r[1], W["map"][:3])
    # while a lane localises: no load, no clear, no snapshot of that lane; the lane goes on as if nothing had been asked
    init = _perturbed(_rebased(W, 0), 0.1, 1.0)
    c.lane_localise(1, *init)
    a = _call(c, 2, {1: _entries(W["dev"], 0, 3)})[1]
    _expect(aloam, ERR_STATE, lambda: c.prior_map_load(W["blob"]))
    _expect(aloam, ERR_STATE, lambda: c.prior_map_clear())
    _expect(aloam, ERR_STATE, lambda: c.lane_save(1))
    b = _call(c, 2, {1: [(p, k, SCAN) for p, k, _ in _entries(W["dev"], 3, 6)]})[1]
    ref = _solo(aloam, W, 0, 6, init)
    assert np.array_equal(np.concatenate([a[1], b[1]]), ref[1])
    # its trajectory over (the call above left lane 1 idle at no step, so end it), the map may be replaced and cleared
    c.reset_odometry()
    c.prior_map_load(W["blob"])
    c.prior_map_clear()
    _expect(aloam, ERR_STATE, lambda: c.lane_localise(0, *ident))
    # a rank of a sharded job does not localise
    assert aloam.lib().aloam_debug_shard_emulate(c._h, 0, 2, 0, 0) == 0
    _expect(aloam, ERR_STATE, lambda: c.prior_map_load(W["blob"]))
    c.close()


def test_a_refused_call_keeps_the_arming(aloam, synth):
    """a call that STARTs the armed lane 0 at step 0 and is refused at step 1 (a SCAN on lane 1, which runs nothing) consumes
    nothing: lane 0's next accepted START localises, as its solo run"""
    W = _world(aloam, synth)
    n = 6
    init = _perturbed(_rebased(W, 2), 0.1, 1.0)
    c = _localiser(aloam, W, 2)
    c.lane_localise(0, *init)
    stray = (W["dev"][2].data_ptr(), W["dev"][2].shape[0], SCAN)
    _expect(aloam, ERR_STATE, lambda: _call(c, 2, {0: _entries(W["dev"], 2, 2 + n), 1: [stray]}, first_step={1: 1}))
    r = _call(c, 2, {0: _entries(W["dev"], 2, 2 + n)})[0]
    ref = _solo(aloam, W, 2, n, init)
    assert np.array_equal(r[0], ref[0]) and np.array_equal(r[1], ref[1])
    c.close()


def test_create_load_destroy_returns_the_memory(aloam, synth):
    W = _world(aloam, synth)
    _localiser(aloam, W).close()   # first use: the process's one-time allocations
    free0 = _free()
    for _ in range(3):
        c = _localiser(aloam, W)
        c.prior_map_load(W["blob"])   # replaces the first
        c.lane_localise(0, np.array([0, 0, 0, 1.0]), np.zeros(3))
        _call(c, 1, {0: _entries(W["dev"], 0, 2)})
        c.close()
    assert _free() >= free0 - (8 << 20), (free0, _free())
