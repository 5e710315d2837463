"""GPU: suspending and resuming localising lanes (aloam_lane_save_localising, aloam_lane_restore of snapshot format version 2) and the
digest that names a prior map (aloam_prior_map_digest).  A localising trajectory saved mid-way and resumed -- in the same lane after
another trajectory ran there, in another lane of a context of another width that loaded the same map from device, pinned or
pageable memory, time-sliced with many others, at skipped and registered scans, with de-skewing, after a recovery adopted a
candidate, right after its START -- must equal its uninterrupted solo run bit for bit: odometry poses, map poses, per-row records
(scores included) and registered clouds.  The digest equals its host recomputation and follows every change of the map; restores
against another map or configuration are refused and change no other lane."""
import numpy as np
import pytest

from test_gpu_localise import _perturbed, _rebased, _world

pytestmark = pytest.mark.gpu

ERR_STATE, ERR_SNAPSHOT = -9, -11
IDLE, SCAN, START = 0, 1, 2
ISQ, PTS = 1.0, 400   # row scoring: inliers at d2 < 1 m^2, at most 400 stack points per type
NCUBE, STORE = 4851, 39424


def _ctx(aloam, W, batch=1, prior="device", max_map_points=400000, **cfg):
    """a context of `batch` lanes with the world's configuration, row records with scores, a registered sink, and the world's map
    loaded as `prior` (None: no map; "device" / "pinned" / "pageable": the copy kind of the load)"""
    import torch
    c = aloam.Aloam(n_scans=W["ns"], max_points=W["M"], max_batch=batch, max_ring_points=4096, max_map_points=max_map_points, **cfg)
    c.set_map_rows(True, ISQ, PTS)
    c.sink = torch.zeros((12 * batch * W["M"], 4), dtype=torch.float32, device="cuda")
    c.set_registered_sink(c.sink)
    if prior is not None:
        b = np.ascontiguousarray(W["blob"])
        blob = {"device": lambda: torch.from_numpy(b).cuda(), "pinned": lambda: torch.from_numpy(b).pin_memory(), "pageable": lambda: b}[prior]()
        c.prior_map_load(blob)
    return c


def _call(c, batch, lanes):
    """one mapped lanes call; lanes = {lane: entries (address, points, op)}; a lane idles after its entries -> {lane: (odometry,
    map poses, rows (dict of per-row arrays), registered clouds)} of its entries"""
    steps = max(len(e) for e in lanes.values())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for lane, entries in lanes.items():
        for k, (p, n, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    o, m = c.scan_stream_lanes(ptrs, counts, ops, True)
    rows = c.map_rows(steps * batch)
    begin, count = c.registered_rows(steps * batch)
    out = {}
    for lane, e in lanes.items():
        r = np.arange(len(e)) * batch + lane
        clouds = [c.sink[begin[i]:begin[i] + count[i]].cpu().numpy().copy() for i in r]
        out[lane] = (o[:len(e), lane], m[:len(e), lane], {k: v[r] for k, v in rows.items()}, clouds)
    return out


def _scans(W, s0, n, start=True):
    return [(d.data_ptr(), d.shape[0], START if start and i == s0 else SCAN) for i, d in enumerate(W["dev"][s0:s0 + n], s0)]


def _cat(parts):
    """the pieces of one trajectory's results, in order, as one result"""
    o = np.concatenate([p[0] for p in parts])
    m = np.concatenate([p[1] for p in parts])
    rows = {k: np.concatenate([p[2][k] for p in parts]) for k in parts[0][2]}
    return o, m, rows, [x for p in parts for x in p[3]]


def _same(got, ref, what):
    assert np.array_equal(got[0], ref[0]), (what, "odometry poses")
    assert np.array_equal(got[1], ref[1]), (what, "map poses")
    for k in ref[2]:
        assert np.array_equal(got[2][k], ref[2][k]), (what, "rows", k)
    assert (got[2]["kind"] == 2).any() and (got[2]["score"] >= 0).any(), what   # localised rows, scored
    assert len(got[3]) == len(ref[3]) and all(np.array_equal(a, b) for a, b in zip(got[3], ref[3])), (what, "registered clouds")


_SOLO = {}


def _solo(aloam, W, s0, n, init, **cfg):
    """the trajectory alone on a fresh one-lane context, one call"""
    key = (id(W), s0, n, np.concatenate(init).tobytes(), tuple(sorted(cfg.items())))
    if key not in _SOLO:
        c = _ctx(aloam, W, 1, **cfg)
        c.lane_localise(0, *init)
        _SOLO[key] = _call(c, 1, {0: _scans(W, s0, n)})[0]
        c.close()
    return _SOLO[key]


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def host_digest(centre, counts, corner, surf):
    """aloam_prior_map_digest recomputed from the documented formula (numpy's uint64 arithmetic wraps mod 2^64)"""
    cs = [np.concatenate([[0], np.cumsum(np.maximum(counts[t], 0))]) for t in range(2)]
    head = np.concatenate([np.array(centre, np.int64), cs[0], cs[1]]).astype(np.int64) & 0xFFFFFFFF
    pts = np.concatenate([np.ascontiguousarray(corner, np.float32).ravel(), np.ascontiguousarray(surf, np.float32).ravel()])
    w = np.concatenate([head.astype(np.uint64), pts.view(np.uint32).astype(np.uint64)])
    k = np.arange(w.size, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = (k * np.uint64(0x9E3779B97F4A7C15)) ^ w
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        return int(z.sum(dtype=np.uint64))


def _digest_of_blob(aloam, blob):
    s = aloam.snapshot_store_clouds(blob)
    return host_digest(s["centre"], s["counts"], s["corner"], s["surf"])


# ---- save, run something else in the lane, restore, continue

@pytest.mark.parametrize("cfg,k", [({}, 4), ({}, 1), ({"mapping_skip_frame": 3}, 5), ({"mapping_skip_frame": 3}, 4), ({"distortion": 1}, 3)])
def test_save_run_another_trajectory_restore_and_continue(aloam, synth, cfg, k):
    """lane 1 localises scans 2 .. 11, is saved after k of them (k = 1: the first scan after START; at mapping_skip_frame 3 the
    scan before the save is skipped at k = 5 and registered at k = 4), runs another localising trajectory while lane 0 maps, is
    restored from the snapshot and continues; save -> restore -> save gives the same bytes"""
    import torch
    W = _world(aloam, synth, **cfg)
    s0, n = 2, 10
    init = _perturbed(_rebased(W, s0), 0.15, 1.5)
    c = _ctx(aloam, W, 2, **cfg)
    c.lane_localise(1, *init)
    first = _call(c, 2, {1: _scans(W, s0, k)})[1]
    buf = torch.empty(int(c.lane_save_localising(1).size), dtype=torch.uint8, device="cuda")
    blob = c.lane_save_localising(1, buf)
    host = blob.cpu().numpy().copy()
    info = aloam.snapshot_info(host)
    assert info["localising"] and info["version"] == 2 and info["scan_index"] == k and info["bytes"] == host.size
    assert info["map_digest"] == c.prior_map_digest() and info["map_centre"] == tuple(W["state"]["centre"])
    assert info["map_points_prior"] == (W["state"]["total_corner"], W["state"]["total_surf"])
    _expect(aloam, ERR_STATE, lambda: c.lane_save(1))   # format 1 has no section for it
    # another trajectory in lane 1 (localising from elsewhere) beside a mapping lane 0
    c.lane_localise(1, *_perturbed(_rebased(W, 0), 0.05, 0.5))
    _call(c, 2, {0: _scans(W, 0, 3), 1: _scans(W, 0, 3)})
    c.lane_restore(1, blob)
    assert c.lane_save_localising(1).tobytes() == host.tobytes()
    _expect(aloam, ERR_STATE, lambda: c.prior_map_clear())   # the restored lane localises
    rest = _call(c, 2, {1: _scans(W, s0 + k, n - k, start=False)})[1]
    _same(_cat([first, rest]), _solo(aloam, W, s0, n, init, **cfg), "cfg %s, saved after %d" % (cfg, k))
    c.close()


@pytest.mark.parametrize("width,lane,kind", [(3, 2, "device"), (16, 11, "pinned"), (5, 0, "pageable")])
def test_restore_into_another_lane_of_another_context(aloam, synth, width, lane, kind):
    """saved from lane 0 of a one-lane context into pageable memory, restored into `lane` of a `width`-lane context that loaded the
    same map from `kind` memory, beside a localising lane of its own; the digest is the same in both contexts"""
    W = _world(aloam, synth)
    s0, n, k = 1, 9, 5
    init = _perturbed(_rebased(W, s0), 0.2, 2.0)
    a = _ctx(aloam, W, 1)
    a.lane_localise(0, *init)
    first = _call(a, 1, {0: _scans(W, s0, k)})[0]
    blob = a.lane_save_localising(0)
    b = _ctx(aloam, W, width, prior=kind)
    assert b.prior_map_digest() == a.prior_map_digest() == _digest_of_blob(aloam, W["blob"])
    a.close()
    other = (lane + 1) % width
    oinit = _perturbed(_rebased(W, 3), 0.1, 1.0)
    b.lane_localise(other, *oinit)
    b.lane_restore(lane, blob)
    got = _call(b, width, {lane: _scans(W, s0 + k, n - k, start=False), other: _scans(W, 3, n - k)})
    _same(_cat([first, got[lane]]), _solo(aloam, W, s0, n, init), "lane %d of %d" % (lane, width))
    _same(got[other], _solo(aloam, W, 3, n - k, oinit), "the other lane")
    b.close()


def _solo_mapping(aloam, W, s0, n):
    key = ("map", id(W), s0, n)
    if key not in _SOLO:
        c = _ctx(aloam, W, 1, prior=None)
        _SOLO[key] = _call(c, 1, {0: _scans(W, s0, n)})[0]
        c.close()
    return _SOLO[key]


def test_time_slicing_localising_and_mapping_trajectories(aloam, synth):
    """24 localising trajectories (format-2 snapshots) and 4 mapping ones (format-1 snapshots) round-robin over 8 lanes in slices
    of 5 scans: each equals its solo run"""
    W = _world(aloam, synth)
    lanes, L, S = 8, 10, 5
    trajs = {}
    for t in range(24):
        s0 = t % 8
        trajs[t] = ("loc", s0, _perturbed(_rebased(W, s0), 0.03 * (t % 5), 0.4 * (t % 4)))
    for t in range(24, 28):
        trajs[t] = ("map", t - 24, None)
    c = _ctx(aloam, W, lanes)
    pos, saved, parts, order = {t: 0 for t in trajs}, {}, {t: [] for t in trajs}, list(trajs)
    kinds = set()
    while any(p < L for p in pos.values()):
        group = [t for t in order if pos[t] < L][:lanes]
        plan = {}
        for i, t in enumerate(group):
            mode, s0, init = trajs[t]
            if t in saved:
                c.lane_restore(i, saved.pop(t))
                plan[i] = _scans(W, s0 + pos[t], min(S, L - pos[t]), start=False)
            else:
                if mode == "loc":
                    c.lane_localise(i, *init)
                plan[i] = _scans(W, s0, min(S, L))
        res = _call(c, lanes, plan)
        for i, t in enumerate(group):
            parts[t].append(res[i])
            pos[t] += len(plan[i])
            if pos[t] < L:
                saved[t] = (c.lane_save_localising(i) if trajs[t][0] == "loc" else c.lane_save(i))
                kinds.add(aloam.snapshot_info(saved[t])["version"])
        order = order[len(group):] + group
    assert kinds == {1, 2}
    for t, (mode, s0, init) in trajs.items():
        got = _cat(parts[t])
        if mode == "loc":
            _same(got, _solo(aloam, W, s0, L, init), "trajectory %d" % t)
        else:
            ref = _solo_mapping(aloam, W, s0, L)
            assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), "mapping trajectory %d" % t
            assert all(np.array_equal(x, y) for x, y in zip(got[3], ref[3])), "mapping trajectory %d" % t
    c.close()


def test_restore_after_a_recovery_adopted_a_candidate(aloam, synth):
    """recovery on: a mis-armed lane adopts a candidate; saved right after the adopting row and restored into another context, it
    continues from the adopted T_wmap_wodom exactly as the uninterrupted run"""
    import recovery_cases as RV
    import track_cases as TC
    from test_gpu_map_rows import _world as rows_world
    Wr = rows_world(aloam, synth)
    W = {"ns": Wr["ns"], "M": Wr["M"], "blob": Wr["blob"], "dev": Wr["dev"]}
    D = RV.deltas(aloam)
    init7 = TC.mis_armed(Wr["map"][TC.START])
    init = (init7[:4], init7[4:])
    n = 6

    def ctx():
        c = _ctx(aloam, W, 2)
        c.set_map_rows(True, TC.ISQ, TC.PTS)   # the scoring the recovery scenario is laid out for
        c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
        return c

    ref_c = ctx()
    ref_c.lane_localise(0, *init)
    steps, adopted = [], None
    for j in range(n):
        steps.append(_call(ref_c, 2, {0: _scans(Wr, TC.START + j, 1, start=j == 0)})[0])
        if adopted is None and ref_c.recovery_rows(2)["adopted"][0]:
            adopted = j
    ref_c.close()
    assert adopted is not None and adopted < n - 1, adopted
    c = ctx()
    c.lane_localise(1, *init)
    first = _call(c, 2, {1: _scans(Wr, TC.START, adopted + 1)})[1]
    assert c.recovery_rows(2 * (adopted + 1))["adopted"].reshape(-1, 2)[adopted, 1]
    blob = c.lane_save_localising(1)
    T = aloam.snapshot_info(blob)["t_wmap_wodom"]
    st = c.mapper_state(1)
    assert np.array_equal(T, np.concatenate([st["q_wmap_wodom"], st["t_wmap_wodom"]]))   # the adopted T_wmap_wodom
    c.close()
    d = ctx()
    d.lane_restore(0, blob)
    rest = _call(d, 2, {0: _scans(Wr, TC.START + adopted + 1, n - adopted - 1, start=False)})[0]
    d.close()
    _same(_cat([first, rest]), _cat(steps), "recovered lane")


# ---- the digest

def test_digest_equals_the_host_recomputation_and_follows_the_map(aloam, synth):
    import struct
    W = _world(aloam, synth)
    c = _ctx(aloam, W, 1, prior=None)
    _expect(aloam, ERR_STATE, lambda: c.prior_map_digest())
    c.profile_enable(True)
    n0 = c.launch_count()
    c.prior_map_load(W["blob"])
    load_launches = c.launch_count() - n0
    assert "k_prior_digest" not in c.profile_read()      # load issues no digest launch
    n0 = c.launch_count()
    d = c.prior_map_digest()
    assert c.launch_count() - n0 == 1 and c.profile_read()["k_prior_digest"][1] == 1
    n0 = c.launch_count()
    assert c.prior_map_digest() == d and c.launch_count() == n0   # kept with the map
    assert d == _digest_of_blob(aloam, W["blob"])
    n0 = c.launch_count()
    c.prior_map_load(W["blob"])                          # a new map: its digest is computed again, on demand
    assert c.launch_count() - n0 == load_launches
    assert c.prior_map_digest() == d and c.launch_count() - n0 == load_launches + 1
    # one point's bit, one cube count (a point moved to another cube), one centre offset
    b = W["blob"].tobytes()
    nls, nlf = struct.unpack_from("<ii", b, 28)
    S = 256 + 16 * (nls + nlf)
    counts = np.frombuffer(b, np.int32, 2 * NCUBE, S + 592).reshape(2, NCUBE)
    full = [i for i in range(NCUBE) if counts[1, i] > 1]
    bit = bytearray(b); bit[S + STORE + 16 * 7 + 3] ^= 0x01
    cnt = bytearray(b)
    struct.pack_into("<i", cnt, S + 592 + 4 * (NCUBE + full[0]), int(counts[1, full[0]]) - 1)
    struct.pack_into("<i", cnt, S + 592 + 4 * (NCUBE + full[1]), int(counts[1, full[1]]) + 1)
    cen = bytearray(b); struct.pack_into("<i", cen, S, struct.unpack_from("<i", b, S)[0] + 1)
    seen = {d}
    for what, blob in (("point bit", bit), ("cube count", cnt), ("centre", cen)):
        c.prior_map_load(bytes(blob))
        got = c.prior_map_digest()
        assert got == _digest_of_blob(aloam, bytes(blob)) and got not in seen, what
        seen.add(got)
    # two builds from the same clouds agree; a build issues no digest launch either
    s = aloam.snapshot_store_clouds(W["blob"])
    c.profile_enable(False); c.profile_enable(True)
    c.prior_map_build(s["corner"], s["surf"], s["centre"])
    assert "k_prior_digest" not in c.profile_read()
    b1 = c.prior_map_digest()
    c.prior_map_build(s["corner"], s["surf"], s["centre"])
    assert c.prior_map_digest() == b1
    c.close()


# ---- refusals

def test_refused_restores_end_the_lane_and_change_no_other(aloam, synth):
    W = _world(aloam, synth)
    s0, n, k = 2, 8, 3
    init = _perturbed(_rebased(W, s0), 0.1, 1.0)
    oinit = _perturbed(_rebased(W, 1), 0.1, -1.0)
    src = _ctx(aloam, W, 1)
    src.lane_localise(0, *init)
    _call(src, 1, {0: _scans(W, s0, k)})
    blob = src.lane_save_localising(0)
    src.close()
    s = aloam.snapshot_store_clouds(W["blob"])
    moved = s["corner"].copy()
    moved[0, 0] = np.nextafter(moved[0, 0], np.float32(np.inf))

    # a different map (one corner coordinate one ulp off): the restore into lane 0 is refused while lane 1 runs a localising
    # trajectory whose halves bracket it; lane 1 equals the same calls on a context where no restore was tried
    runs = []
    for attempt in (True, False):
        c = _ctx(aloam, W, 2, prior=None)
        c.prior_map_build(moved, s["surf"], s["centre"])
        c.lane_localise(1, *oinit)
        a = _call(c, 2, {1: _scans(W, 1, 3)})[1]
        c.lane_localise(0, *init)
        b = _call(c, 2, {0: _scans(W, s0, 1), 1: _scans(W, 4, 1, start=False)})[1]   # lane 0 runs something the refusal ends
        if attempt:
            _expect(aloam, ERR_SNAPSHOT, lambda: c.lane_restore(0, blob))
            _expect(aloam, ERR_STATE, lambda: c.lane_save_localising(0))   # not running
        runs.append(_cat([a, b, _call(c, 2, {1: _scans(W, 5, 3, start=False)})[1]]))
        c.close()
    _same(runs[0], runs[1], "the other lane")
    c = _ctx(aloam, W, 2, prior=None, max_map_points=0)     # no scan-to-map at all (a map can still be built)
    c.prior_map_build(s["corner"], s["surf"], s["centre"])
    _expect(aloam, ERR_SNAPSHOT, lambda: c.lane_restore(0, blob))
    c.close()
    c = _ctx(aloam, W, 2, prior=None, line_res=0.3)         # another leaf of the corner stack
    c.prior_map_build(s["corner"], s["surf"], s["centre"])
    _expect(aloam, ERR_SNAPSHOT, lambda: c.lane_restore(0, blob))
    c.close()
    c = _ctx(aloam, W, 2, prior=None)                       # no prior map
    _expect(aloam, ERR_STATE, lambda: c.lane_restore(0, blob))
    _expect(aloam, ERR_STATE, lambda: c.lane_save_localising(0))
    c.prior_map_load(W["blob"])
    c.lane_restore(0, blob)                                 # and with the map loaded it restores
    # a mapping lane and an odometry-only lane have no localising snapshot
    _call(c, 2, {1: _scans(W, 0, 2)})
    _expect(aloam, ERR_STATE, lambda: c.lane_save_localising(1))
    c.close()
    c = _ctx(aloam, W, 1)
    c.scan_stream_lanes(np.array([[W["dev"][0].data_ptr()]], np.uint64), np.array([[W["dev"][0].shape[0]]]),
                            np.array([[START]], np.int32), True, mapped=False)
    _expect(aloam, ERR_STATE, lambda: c.lane_save_localising(0))
    assert aloam.snapshot_info(c.lane_save(0))["version"] == 1
    _expect(aloam, ERR_SNAPSHOT, lambda: c.prior_map_load(blob))   # a localising snapshot holds no store
    c.close()
