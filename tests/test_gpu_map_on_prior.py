"""GPU: mapping trajectories that start on a copy of the prior map (aloam_lane_map_on_prior).  A seeded lane is an ordinary mapping
lane whose store, at its START, is the prior map's and whose T_wmap_wodom is the armed init.  Checked here: every row against
aloam_mapper_step on a lane restored from the prior snapshot with the init patched in (bit for bit, through a ring-buffer shift); an
empty prior at the identity against an unarmed lane; the START frame against a localising lane's; seeded lanes beside fresh-mapping,
localising and odometry-only lanes against their solo runs, with launch counts; a second session that extends the first one's map;
suspend and resume without a prior map; refusals and the arming's lifecycle."""
import struct

import numpy as np
import pytest

import lane_refs as R
from test_gpu_localise import N_MAP, _call, _ctx, _entries, _expect, _perturbed, _solo, _world

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
IDLE, SCAN, START = 0, 1, 2
NCUBE = 4851


def _normalised(q, t):
    """(q, t) as the library normalises an init: q / sqrt(q . q), summed in index order"""
    n2 = 0.0
    for v in q:
        n2 += float(v) * float(v)
    return np.concatenate([np.asarray(q, np.float64) / np.sqrt(n2), np.asarray(t, np.float64)])


def _store_offset(blob):
    nls, nlf = struct.unpack_from("<ii", blob, 28)
    return 256 + 16 * (nls + nlf)


def _edge_blob(W, T, dx=8):
    """W's snapshot with its store moved dx cubes down in i and the centre offset with it (cube i of centre 10 covers what cube
    i - dx of centre 10 - dx covers: the same points, re-indexed), T_wmap_wodom = T, frames = 0 and an empty valid list.  A lane
    near the map's origin then lies in cube 10 - dx, so its first frame shifts the ring buffer."""
    b = bytearray(W["blob"].tobytes())
    S = _store_offset(b)
    counts = np.frombuffer(bytes(b), np.int32, 2 * NCUBE, S + 592).reshape(2, NCUBE)
    pts = np.frombuffer(bytes(b), np.float32, offset=S + 39424).reshape(-1, 4)
    blocks, off = {}, 0
    for c in range(NCUBE):
        for t in range(2):
            n = max(int(counts[t, c]), 0)
            blocks[c, t] = pts[off:off + n]
            off += n
    assert all(counts[t, c] <= 0 for c in range(NCUBE) if c % 21 < dx for t in range(2)), "no point leaves the buffer"
    new, out = np.full((2, NCUBE), -1, np.int32), []
    for c in range(NCUBE):
        for t in range(2):
            if c % 21 + dx <= 20:
                new[t, c] = counts[t, c + dx]
                out.append(blocks[c + dx, t])
    cen = struct.unpack_from("<3i", b, S)
    struct.pack_into("<3i", b, S, cen[0] - dx, cen[1], cen[2])
    struct.pack_into("<i", b, S + 12, 0)
    b[S + 16:S + 528] = bytes(512)
    struct.pack_into("<i", b, S + 528, 0)
    struct.pack_into("<4d", b, S + 536, *T[:4])
    struct.pack_into("<3d", b, S + 568, *T[4:])
    b[S + 592:S + 592 + new.nbytes] = new.tobytes()
    b[S + 39424:] = np.concatenate(out).tobytes()
    return np.frombuffer(bytes(b), np.uint8)


def _store_section(blob):
    b = blob.tobytes()
    return b[_store_offset(b):]


def _row_stats(rows, j):
    return {k: (list(rows[k][j]) if k == "termination" else rows[k][j]) for k in R.STAT_KEYS}


def test_every_row_equals_mapper_step_on_the_restored_prior(aloam, synth):
    """12 scans from a perturbed pose on a prior map whose cubes lie near the buffer's low edge: the first frame shifts the ring
    buffer.  Every map pose and row == aloam_mapper_step on a scratch lane restored once from the prior snapshot with the
    normalised init and frames = 0, fed the same clouds and odometry poses; the lanes' saved stores are the same bytes."""
    W = _world(aloam, synth)
    s0, n = 1, 12
    q0, t0 = _perturbed(W["map"][s0], 0.2, 2.0)
    T = _normalised(3.0 * q0, t0)
    prior = _edge_blob(W, T)
    c = _ctx(aloam, W["M"])
    c.prior_map_load(prior)
    before = c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes()
    c.set_map_rows(True)
    c.lane_map_on_prior(0, 3.0 * q0, t0)
    o, m = _call(c, 1, {0: _entries(W["dev"], s0, s0 + n)})[0]
    rows = c.map_rows(n)
    assert (rows["kind"] == aloam.ROW_MAPPED).all()
    assert c.mapper_state(0)["centre"] == (3, 10, 5)   # the first frame shifted the ring buffer one cube up in i
    scratch, feats = _ctx(aloam, W["M"]), _ctx(aloam, W["M"])
    scratch.lane_restore(0, prior)
    for j in range(n):
        f = feats.extract_features(W["scans"][s0 + j])
        q, t, st = scratch.mapper_step(f["less_sharp"], f["less_flat"], o[j][:4], o[j][4:])
        assert np.array_equal(m[j], np.concatenate([q, t])), "frame %d" % j
        assert _row_stats(rows, j) == {k: st[k] for k in R.STAT_KEYS}, "frame %d" % j
    assert not (rows["flags"] & aloam.FLAG_MAP_TOO_THIN).any()   # every frame registered against the seeded map
    assert _store_section(c.lane_save(0)) == _store_section(scratch.lane_save(0))
    assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == before   # the prior map is never written
    dt, dr = R.deviation(m[N_MAP - 1 - s0:N_MAP - s0], W["map"][N_MAP - 1:N_MAP])   # the initial error is gone
    assert dt < 0.1 and dr < 0.02, (dt, dr)
    for x in (c, scratch, feats):
        x.close()


def test_an_empty_prior_at_the_identity_is_an_unarmed_start(aloam, synth):
    W = _world(aloam, synth)
    n = 6
    c = _ctx(aloam, W["M"], 2)
    c.prior_map_build(np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))
    c.set_map_rows(True)
    c.lane_map_on_prior(0, np.array([0, 0, 0, 1.0]), np.zeros(3))
    r = _call(c, 2, {0: _entries(W["dev"], 0, n), 1: _entries(W["dev"], 0, n)})
    rows = c.map_rows(2 * n)
    assert np.array_equal(r[0][0], r[1][0]) and np.array_equal(r[0][1], r[1][1])
    assert np.array_equal(r[0][1], W["map"][:n])
    for k, v in rows.items():
        assert np.array_equal(v[0::2], v[1::2]), k
    assert c.mapper_export(aloam.EXPORT_MAP, 0).tobytes() == c.mapper_export(aloam.EXPORT_MAP, 1).tobytes()
    c.close()


def test_the_start_frame_is_the_localising_frame(aloam, synth):
    """a START that neither shifts nor exceeds max_map_points returns the pose a localising START returns from the same init;
    the next rows differ, because the seeded lane inserted its scan"""
    W = _world(aloam, synth)
    init = _perturbed(W["map"][2], 0.1, 1.0)
    c = _ctx(aloam, W["M"], 2)
    c.prior_map_load(W["blob"])
    c.lane_map_on_prior(0, *init)
    c.lane_localise(1, *init)
    r = _call(c, 2, {0: _entries(W["dev"], 2, 5), 1: _entries(W["dev"], 2, 5)})
    assert np.array_equal(r[0][1][0], r[1][1][0])
    assert not np.array_equal(r[0][1][1:], r[1][1][1:])
    c.close()


@pytest.mark.parametrize("sensor,cfg", [("VLP-16", {}), ("HDL-32", {}), ("VLP-16", {"distortion": 1, "mapping_skip_frame": 3})])
def test_a_seeded_trajectory_follows_the_seeded_oracle(aloam, synth, orc, sensor, cfg):
    """scans 2 .. of the mapped trajectory as a new session from a pose 0.2 m and 2 degrees off its map pose: the map poses against
    the oracle's CubeMap seeded with the snapshot's store (oracle features and odometry); skipped scans get the high-frequency pose
    from the seeded T_wmap_wodom.  The stores' cubes with the tolerances of test_gpu_cubemap.py."""
    from cube_edge_cases import associate
    from map_on_prior_seed import seed_cubemap
    W = _world(aloam, synth, sensor, **cfg)
    # full-size slabs (16 384 corner / 65 536 surf points) and leaves of 0.4 / 0.8 m, so that no cube of this dense synthetic scene
    # overflows its slab: the oracle's cubes have no bound
    maxpts, ns, leaves = 70000, W["ns"], (0.4, 0.8)
    cfg = dict(cfg, line_res=leaves[0], plane_res=leaves[1])
    src = _ctx(aloam, maxpts, 1, ns, **cfg)
    map_rows = _call(src, 1, {0: _entries(W["dev"], 0, N_MAP)})[0][1]
    blob = src.lane_save(0)
    src.close()
    skip, s0 = cfg.get("mapping_skip_frame", 1), 2
    scans = W["scans"][s0:]
    init = _perturbed(map_rows[s0], 0.2, 2.0)
    c = _ctx(aloam, maxpts, 1, ns, **cfg)
    c.prior_map_load(blob)
    c.set_map_rows(True)
    c.lane_map_on_prior(0, *init)
    o, m = _call(c, 1, {0: _entries(W["dev"], s0, len(W["scans"]))})[0]
    assert not (c.map_rows(len(scans))["flags"] & aloam.FLAG_CUBE_OVERFLOW).any()
    b = blob.tobytes()
    S = _store_offset(b)
    counts = np.frombuffer(b, np.int32, 2 * NCUBE, S + 592).reshape(2, NCUBE)
    T = _normalised(*init)
    cm = orc.CubeMap()
    seed_cubemap(cm, struct.unpack_from("<3i", b, S), T[:4], T[4:], counts, np.frombuffer(b, np.float32, offset=S + 39424))
    mr, (line_res, plane_res) = synth.SENSORS[sensor][2], leaves
    odom, _ = R.oracle(orc, synth, scans, ("seeded", sensor, s0), False, cfg.get("distortion", 0), sensor)
    R.assert_near(o, odom, "odometry")
    ref = []
    for k, raw in enumerate(scans):
        if k % skip:
            st = cm.state()
            ref.append(np.array(associate((tuple(st["q_wmap_wodom"]), tuple(st["t_wmap_wodom"])), odom[k, :4], odom[k, 4:])))
            continue
        f = orc.Features(raw, ns, mr)
        ref.append(cm.step(f.less_sharp, f.less_flat, odom[k, :4], odom[k, 4:], line_res, plane_res)[0])
    R.assert_near(m, np.array(ref), "map poses of the seeded lane")
    sg, so = c.mapper_state(0), cm.state()
    assert sg["centre"] == so["centre"] and sg["valid"] == so["valid"]
    assert abs(sg["total_corner"] - so["total_corner"]) <= 5 and abs(sg["total_surf"] - so["total_surf"]) <= 20
    c.close()


_SEEDED = {}


def _seeded_solo(aloam, W, s0, n, init):
    """a seeded trajectory on W's map alone on a fresh context: (odometry rows, map rows)"""
    key = (id(W), s0, n, init[0].tobytes(), init[1].tobytes())
    if key not in _SEEDED:
        c = _ctx(aloam, W["M"])
        c.prior_map_load(W["blob"])
        c.lane_map_on_prior(0, *init)
        _SEEDED[key] = _call(c, 1, {0: _entries(W["dev"], s0, s0 + n)})[0]
        c.close()
    return _SEEDED[key]


@pytest.mark.parametrize("width", [1, 5, 16])
def test_seeded_lanes_beside_other_modes_equal_their_solo_runs(aloam, synth, width):
    """lane l: seeded (l % 4 == 0 or width 1), fresh-mapping (1), localising (2), odometry-only in a call of its own (3).  The
    seeded STARTs fall at different steps; lane 0 (width > 1) first runs a fresh-mapping trajectory whose last SCAN its seeded
    START follows directly"""
    W = _world(aloam, synth)
    c = _ctx(aloam, W["M"], width)
    c.prior_map_load(W["blob"])
    modes = {l: ("seed" if width == 1 or l % 4 == 0 else ("map", "loc", "odo")[l % 4 - 1]) for l in range(width)}
    odo = [l for l in modes if modes[l] == "odo"]
    if odo:
        got = _call(c, width, {l: _entries(W["dev"], 0, 4) for l in odo}, mapped=False)
        for l in odo:
            assert np.array_equal(got[l][0], W["odom"][:4])
    lanes, first, plan = {}, {}, {}
    if width > 1:   # lane 0 maps scans 0 .. 2 in a call of their own, then SCANs 3, 4 and STARTs seeded at once
        _call(c, width, {0: _entries(W["dev"], 0, 3)})
        plan[0] = (1, 6, _perturbed(W["map"][1], 0.1, 1.0))
        c.lane_map_on_prior(0, *plan[0][2])
        lanes[0] = [(p, k, SCAN) for p, k, _ in _entries(W["dev"], 3, 5)] + _entries(W["dev"], 1, 7)
    for l, mode in modes.items():
        if l in lanes or mode == "odo":
            continue
        s0, n = l % 5, 5 + l % 3
        first[l] = l % 3
        init = _perturbed(W["map"][s0], 0.05 * (l % 4), 0.5 * (l % 5))
        if mode == "seed":
            c.lane_map_on_prior(l, *init)
        elif mode == "loc":
            c.lane_localise(l, *init)
        plan[l] = (s0, n, init)
        lanes[l] = _entries(W["dev"], s0, s0 + n)
    got = _call(c, width, lanes, first_step=first)
    for l, (s0, n, init) in plan.items():
        o, m = got[l]
        if l == 0 and width > 1:
            o, m = o[2:], m[2:]
        if modes[l] == "seed":
            ref = _seeded_solo(aloam, W, s0, n, init)
        elif modes[l] == "loc":
            ref = _solo(aloam, W, s0, n, init)
        else:
            ref = (W["odom"][s0:s0 + n] if s0 == 0 else None, W["map"][s0:s0 + n] if s0 == 0 else None)
            if s0 != 0:
                continue
        assert np.array_equal(o, ref[0]) and np.array_equal(m, ref[1]), "lane %d (%s)" % (l, modes[l])
    assert c.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == W["export"].tobytes()
    c.close()


def test_launch_counts(aloam, synth):
    """a call with no seeded START issues what it issues on a context that was never armed; a step with seeded STARTs issues 2
    more launches, for any number of them"""
    W = _world(aloam, synth)
    n = 4
    init = _perturbed(W["map"][2], 0.1, 1.0)

    def launches(arm, lanes, mapped=True, first_step=None):
        x = _ctx(aloam, W["M"], 2)
        x.prior_map_load(W["blob"])
        for _ in range(2):   # the first call creates what the lanes own
            x.reset_odometry()
            for l in arm:
                x.lane_map_on_prior(l, *init)
            a = x.launch_count()
            _call(x, 2, {l: _entries(W["dev"], 2, 2 + n) for l in lanes}, mapped=mapped, first_step=first_step)
            a = x.launch_count() - a
        x.close()
        return a
    assert launches([0], [0], mapped=False) == launches([], [0], mapped=False)   # an odometry-only START keeps the arming
    assert launches([0], [1]) == launches([], [1])                               # armed, but idle all call
    fresh = launches([], [0, 1])
    assert launches([0], [0, 1]) == fresh + 2
    assert launches([0, 1], [0, 1]) == fresh + 2
    assert launches([0, 1], [0, 1], first_step={1: 1}) == launches([], [0, 1], first_step={1: 1}) + 4


def test_a_second_session_extends_the_first_sessions_map(aloam, synth):
    """session 1 = W (scans 0 .. N_MAP-1 mapped and saved).  Session 2 = scans s0 .. of the same ground, its first scan placed on
    session 1's map by aloam_prior_relocalise, mapped on a copy of it and driven beyond it.  Its snapshot, loaded as the new prior
    map, exports the seeded lane's store, holds more points, and keeps a localising lane tracking where session 1's map was thin."""
    W = _world(aloam, synth)
    s0, n = 6, 34
    scans = R.traj(synth, 0, s0 + n)
    dev = R.to_device(scans)
    M = max(W["M"], R.maxn([scans]) + 1024)
    c = _ctx(aloam, M)
    c.prior_map_load(W["blob"])
    hyps = np.array([np.concatenate(_perturbed(W["map"][s0], d, a)) for d in (0.0, 0.3, 0.6) for a in (-2.0, 0.0, 2.0)])
    hyps[:, 4:] += np.array([0.3, -0.2, 0.0])
    out, _ = c.prior_relocalise(hyps, raw=scans[s0], refine=3)
    pose = out[0]["pose"]
    c.lane_map_on_prior(0, pose[:4], pose[4:])
    _call(c, 1, {0: [(d.data_ptr(), d.shape[0], START if i == s0 else SCAN) for i, d in enumerate(dev[s0:], s0)]})
    blob2 = c.lane_save(0)
    exported = c.mapper_export(aloam.EXPORT_MAP, 0).tobytes()
    c.close()
    info1, info2 = aloam.snapshot_info(W["blob"]), aloam.snapshot_info(blob2)
    assert info2["map_points"] > info1["map_points"]
    scores = {}
    for name, blob in (("old", W["blob"]), ("new", blob2)):
        x = _ctx(aloam, M)
        x.prior_map_load(blob)
        if name == "new":
            assert x.mapper_export(aloam.EXPORT_MAP, aloam.PRIOR_MAP).tobytes() == exported
        x.set_map_rows(True, 1.0, 512)
        x.lane_localise(0, pose[:4], pose[4:])
        _call(x, 1, {0: [(d.data_ptr(), d.shape[0], START if i == s0 else SCAN) for i, d in enumerate(dev[s0:], s0)]})
        rows = x.map_rows(n)
        scores[name] = rows["score"] / np.maximum(rows["n_score"], 1)
        x.close()
    far = slice(n - 8, n)   # the last scans, beyond session 1's last mapped scan
    assert scores["new"][far].mean() > scores["old"][far].mean() and scores["new"][-1] > scores["old"][-1], (scores["new"][far], scores["old"][far])


def test_a_seeded_lane_resumes_without_a_prior_map(aloam, synth):
    W = _world(aloam, synth)
    s0, n, k = 1, 10, 5
    init = _perturbed(W["map"][s0], 0.1, 1.0)
    ref = _seeded_solo(aloam, W, s0, n, init)
    c = _ctx(aloam, W["M"])
    c.prior_map_load(W["blob"])
    c.lane_map_on_prior(0, *init)
    a = _call(c, 1, {0: _entries(W["dev"], s0, s0 + k)})[0]
    blob = c.lane_save(0)
    c.close()
    d = _ctx(aloam, W["M"], 2)   # no prior map; lane 1 of a wider context
    d.lane_restore(1, blob)
    b = _call(d, 2, {1: [(p, q, SCAN) for p, q, _ in _entries(W["dev"], s0 + k, s0 + n)]})[1]
    d.close()
    assert np.array_equal(np.concatenate([a[0], b[0]]), ref[0]) and np.array_equal(np.concatenate([a[1], b[1]]), ref[1])


def test_refusals_arm_nothing_and_the_arming_lifecycle(aloam, synth):
    W = _world(aloam, synth)
    ident = (np.array([0, 0, 0, 1.0]), np.zeros(3))
    n = 4
    init = _perturbed(W["map"][2], 0.1, 1.0)
    c = _ctx(aloam, W["M"], 2)
    _expect(aloam, ERR_STATE, lambda: c.lane_map_on_prior(0, *ident))   # no prior map
    c.prior_map_load(W["blob"])
    # every refusal leaves an earlier arming (here: localise) in place
    c.lane_localise(0, *init)
    for q, t in ((np.zeros(4), np.zeros(3)), (np.array([0, 0, np.nan, 1.0]), np.zeros(3)), (ident[0], np.array([0, np.inf, 0]))):
        _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_map_on_prior(0, q, t))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_map_on_prior(2, *ident))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_map_on_prior(-1, *ident))
    # centre cube of x: int((x + 25) / 50) - 1 + 10 -- -16 at x = -1300 (allowed), -18 at x = -1400
    _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_map_on_prior(0, ident[0], np.array([-1400.0, 0, 0])))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.lane_map_on_prior(0, ident[0], np.array([0, 0, 1e300])))
    r = _call(c, 2, {0: _entries(W["dev"], 2, 2 + n)})[0]
    assert np.array_equal(r[1], _solo(aloam, W, 2, n, init)[1])
    # the slack bound itself arms; aloam_reset_odometry drops it
    c.lane_map_on_prior(0, ident[0], np.array([-1300.0, 0, 0]))
    c.reset_odometry()
    assert np.array_equal(_call(c, 2, {0: _entries(W["dev"], 0, n)})[0][1], W["map"][:n])
    seeded = _seeded_solo(aloam, W, 2, n, init)
    # an odometry-only START keeps it
    c.lane_map_on_prior(0, *init)
    _call(c, 2, {0: _entries(W["dev"], 0, 2)}, mapped=False)
    assert np.array_equal(_call(c, 2, {0: _entries(W["dev"], 2, 2 + n)})[0][1], seeded[1])
    # the later arming wins, both ways
    c.lane_map_on_prior(0, *init)
    c.lane_localise(0, *init)
    assert np.array_equal(_call(c, 2, {0: _entries(W["dev"], 2, 2 + n)})[0][1], _solo(aloam, W, 2, n, init)[1])
    c.lane_localise(0, *init)
    c.lane_map_on_prior(0, *init)
    assert np.array_equal(_call(c, 2, {0: _entries(W["dev"], 2, 2 + n)})[0][1], seeded[1])
    # load, build and clear drop it: the next mapped START is a fresh one, as an unarmed lane's
    for drop in (lambda: c.prior_map_load(W["blob"]), lambda: c.prior_map_build(np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32)),
                 lambda: c.prior_map_clear()):
        c.prior_map_load(W["blob"])
        c.lane_map_on_prior(0, *init)
        drop()
        assert np.array_equal(_call(c, 2, {0: _entries(W["dev"], 0, n)})[0][1], W["map"][:n])
    # a rank of a sharded job (here an emulating context) does not seed
    c.prior_map_load(W["blob"])
    assert aloam.lib().aloam_debug_shard_emulate(c._h, 0, 2, 0, 0) == 0
    _expect(aloam, ERR_STATE, lambda: c.lane_map_on_prior(0, *ident))
    c.close()
    # a built map with a corner cube above the corner slab capacity (min(16384, max_points) = 4096 here)
    g = np.stack(np.meshgrid(np.arange(80) * 0.3, np.arange(80) * 0.3, indexing="ij"), -1).reshape(-1, 2)
    dense = np.concatenate([g, np.zeros((len(g), 2))], 1).astype(np.float32)
    small = aloam.Aloam(n_scans=16, max_points=4096, max_ring_points=4096, max_map_points=100000)
    small.prior_map_build(dense, np.zeros((0, 4), np.float32))
    assert small.mapper_export_size(aloam.EXPORT_MAP, aloam.PRIOR_MAP) == len(dense)
    _expect(aloam, ERR_CAPACITY, lambda: small.lane_map_on_prior(0, *ident))
    small.prior_map_build(dense[:4096], np.zeros((0, 4), np.float32))
    small.lane_map_on_prior(0, *ident)
    small.close()
