"""GPU: loop verification (aloam_set_loops, aloam_loop_rows, aloam_loop_verify, aloam_place_keyframe_cloud).  Keyframe clouds
against the subsample of the voxel-filtered stacks, bit for bit; on a return trip every verified row against the host API run on
the host gather of the exported clouds (aloam_map_upload + aloam_mapping_register in an outer_iters = 1 context), the brute-force
score, the Eigen-order constraint and the oracle registration; its accuracy against the ground truth; loops changing nothing else
and issuing the documented launches; batched and scheduled lanes; thin submaps; refusals."""
import numpy as np
import pytest

import lane_refs as R
import pyloop as L
import pyoracle
import reloc_cases as RC

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
IDLE, SCAN, START = 0, 1, 2
LOOP = dict(max_distance=2.0, window=5, cloud_points=1000, outer_iters=4, inlier_sq=1.0)
STAT_KEYS = ("n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps", "flags", "termination", "init_cost", "final_cost")


def _ctx(aloam, maxpts, batch=1, ns=32, **cfg):
    kw = {"max_ring_points": 4096, "max_map_points": 400000, **cfg}
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, **kw)


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _same_row(a, b):
    for k in ("query", "cand", "verified", "shift", "n_sub", "score", "n_score"):
        assert a[k] == b[k], (k, a[k], b[k])
    for k in ("pose", "rel"):
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    for k in STAT_KEYS:
        assert np.array_equal(_bits(np.float64(a["stats"][k])) if "cost" in k else a["stats"][k],
                              _bits(np.float64(b["stats"][k])) if "cost" in k else b["stats"][k]), k


def _lanes_run(c, dev, ops):
    n, b = ops.shape
    ptrs = np.array([[dev[j][k].data_ptr() for j in range(b)] for k in range(n)], np.uint64)
    counts = np.array([[dev[j][k].shape[0] for j in range(b)] for k in range(n)], np.int64)
    return c.scan_stream_lanes(ptrs, counts, ops, True)


# ---- the return trip of test_gpu_place.py: 40 scans out, 39 back over the same places
@pytest.fixture(scope="module")
def trip(aloam, synth):
    out = R.traj(synth, 0, 40, sensor="HDL-32", n_az=600)
    back = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 50, n_az=700) for k in range(38, -1, -1)]
    scans = out + back
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M)
    c.set_place(True, keyframe_gap=0.0, exclude_recent=10, max_keyframes=200)
    c.set_loops(True, **LOOP)
    ops = np.full((len(scans), 1), SCAN, np.int32); ops[0] = START
    _, m = _lanes_run(c, [dev], ops)
    rows = c.loop_rows(len(scans))
    place = c.place_rows(len(scans))
    rec = c.place_keyframes(0)
    clouds = [c.keyframe_cloud(0, k) for k in range(len(rec))]
    yield dict(c=c, M=M, rows=rows, place=place, rec=rec, clouds=clouds, n=len(scans))
    c.close()


def test_keyframe_clouds_are_the_subsampled_stacks(aloam, synth):
    scans = R.traj(synth, 1, 12, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    fx = _ctx(aloam, M)
    stacks = []
    for s in scans:
        f = fx.extract_features(s)
        stacks.append((fx.voxel_filter(f["less_sharp"], fx.cfg.line_res), fx.voxel_filter(f["less_flat"], fx.cfg.plane_res)))
    fx.close()
    small = min(min(a.shape[0], b.shape[0]) for a, b in stacks)
    for P in (max(1, small // 3), M):
        c = _ctx(aloam, M)
        c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
        c.set_loops(True, max_distance=0.0, window=0, cloud_points=P)
        c.scan_stream_mapped([d.data_ptr() for d in dev], [d.shape[0] for d in dev], True)
        kf = c.place_rows(len(scans))["keyframe"]
        assert (kf >= 0).sum() > 3
        for k in range(len(scans)):
            if kf[k] < 0:
                continue
            got = c.keyframe_cloud(0, int(kf[k]))
            for t in range(2):
                assert np.array_equal(_bits(got[t]), _bits(L.subsample(stacks[k][t], P))), (P, k, t)
        c.close()


def test_return_trip_rows_equal_the_host_api(aloam, trip):
    c, rows, rec, clouds = trip["c"], trip["rows"], trip["rec"], trip["clouds"]
    H = _ctx(aloam, trip["M"], outer_iters=1)
    R_ = LOOP["outer_iters"]
    checked = 0
    for r, row in enumerate(rows):
        pr = trip["place"]
        trig = pr["keyframe"][r] >= 0 and pr["loop"][r] >= 0 and pr["distance"][r] <= LOOP["max_distance"]
        assert bool(row["verified"]) == bool(trig), r
        if not trig:
            assert (row["query"], row["cand"], row["shift"]) == (-1, -1, -1)
            continue
        q, cd, s = int(pr["keyframe"][r]), int(pr["loop"][r]), int(pr["shift"][r])
        assert (row["query"], row["cand"], row["shift"]) == (q, cd, s)
        _same_row(row, c.loop_verify(0, q, cd, s))                       # in-stream == on request after the call
        lo, hi = L.window(q, cd, LOOP["window"], 10)
        sc, ss = L.gather(clouds, rec["pose"], lo, hi)
        assert row["n_sub"] == (sc.shape[0], ss.shape[0])
        qc, qs = clouds[q]
        assert row["n_score"] == qc.shape[0] + qs.shape[0]
        x0 = L.init_pose(rec["pose"][cd], s)
        H.map_upload(sc, ss)
        x, st = x0.copy(), None
        for _ in range(R_):
            x, st = H.mapping_register(qc, qs, x)
        assert np.array_equal(_bits(row["pose"]), _bits(x)), r
        for k in STAT_KEYS:
            assert np.array_equal(np.asarray(row["stats"][k]), np.asarray(st[k])), (r, k)
        assert row["score"] == L.score(qc, qs, row["pose"], sc, ss, LOOP["inlier_sq"]), r
        assert np.array_equal(_bits(row["rel"]), _bits(L.rel(rec["pose"][cd], row["pose"]))), r
        if not row["stats"]["flags"] & aloam.FLAG_MAP_TOO_THIN:
            m = pyoracle.Mapping(); m.set_map(sc, ss)
            xr, _ = m.register(qc, qs, x0, outer=R_)
            dq = abs(float(np.dot(xr[:4], row["pose"][:4])))
            assert np.abs(xr[4:] - row["pose"][4:]).max() < 1e-7 and 2 * np.arccos(min(1.0, dq)) < 1e-7, r
        checked += 1
    assert checked > 20
    H.close()


def _rel_err(a, b):
    dq = abs(float(np.dot(a[:4], b[:4])))
    return float(np.linalg.norm(a[4:] - b[4:])), 2 * float(np.arccos(min(1.0, dq)))


def test_return_trip_accuracy_and_wrong_pairs(aloam, synth, trip):
    c, rows, rec = trip["c"], trip["rows"], trip["rec"]
    gt = [np.concatenate(synth.pose(k)) for k in range(40)]
    checked = 0
    for i, k in enumerate(range(38, -1, -1)):
        row = rows[40 + i]
        if not row["verified"] or abs(row["cand"] - k) > 1:
            continue
        dt, dr = _rel_err(row["rel"], L.rel(gt[row["cand"]], gt[k]))
        assert dt < RC.NEAR_M and dr < RC.NEAR_RAD, (k, row["cand"], dt, dr)
        q = row["query"]
        far = [w for w in range(0, q - 10) if w < 40 and np.linalg.norm(gt[w][4:] - gt[k][4:]) >= 20.0]
        if far:
            wrong = c.loop_verify(0, q, far[0], 0)
            assert wrong["score"] < row["score"], (k, far[0], wrong["score"], row["score"])
        checked += 1
    assert checked > 10


def _stream(aloam, synth, loops, sink=True, place=True, setup=None, n=12):
    import torch
    scans = R.traj(synth, 2, n, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M)
    if place:
        c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    if setup:
        setup(c)
    if loops:
        c.set_loops(True, **LOOP)
    c.set_map_rows(True)
    s = torch.zeros((sum(d.shape[0] for d in dev), 4), dtype=torch.float32, device="cuda") if sink else None
    if sink:
        c.set_registered_sink(s)
    n0 = c.launch_count()
    ops = np.full((n, 1), SCAN, np.int32); ops[0] = START
    o, m = _lanes_run(c, [dev], ops)
    out = dict(launches=c.launch_count() - n0, odom=o, map=m, rows=c.map_rows(n), reg=s.cpu().numpy() if sink else None,
               snap=bytes(c.lane_save(0)))
    if place:
        out.update(place=c.place_rows(n), rec=c.place_keyframes(0).tobytes())
    out["c"] = c
    return out


def test_loops_change_nothing_else(aloam, synth):
    a = _stream(aloam, synth, False)
    b = _stream(aloam, synth, True)
    for k in ("odom", "map", "reg"):
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    for k in a["rows"]:
        assert np.array_equal(a["rows"][k], b["rows"][k]), k
    for k in a["place"]:
        assert np.array_equal(a["place"][k], b["place"][k]), k
    assert a["rec"] == b["rec"] and a["snap"] == b["snap"]
    lrows = b["c"].loop_rows(12)
    assert sum(r["verified"] for r in lrows) > 0
    for x in (a, b):
        x["c"].close()


def test_launch_counts(aloam, synth):
    base = _stream(aloam, synth, False, sink=False)
    off = _stream(aloam, synth, False, sink=False, setup=lambda c: (c.set_loops(True, **LOOP), c.set_loops(False, **LOOP)))
    on = _stream(aloam, synth, True, sink=False)
    assert off["launches"] == base["launches"]
    # the place table's bound on the keyframes a record queries (max_keyframes 64, exclude_recent 2), per mapping frame
    extra, upper = 0, 0
    for k in range(12):
        if k == 0:
            upper = 0
        n_upper = min(upper, 63) - 2
        upper = min(64, upper + 1)
        extra += 1 + (8 + 3 * LOOP["outer_iters"] if n_upper > 0 else 0)
    assert on["launches"] - base["launches"] == extra
    for x in (base, off, on):
        x["c"].close()


def test_batched_lanes_equal_solo_runs(aloam, synth):
    B, n = 16, 12
    scans = [R.traj(synth, t, n, sensor="HDL-32", n_az=600) for t in range(B)]
    M = R.maxn(scans) + 1024
    dev = [R.to_device(tr) for tr in scans]
    c = _ctx(aloam, M, B)
    c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    c.set_loops(True, **LOOP)
    ptrs = np.array([[dev[b][k].data_ptr() for b in range(B)] for k in range(n)], np.uint64)
    counts = np.array([[dev[b][k].shape[0] for b in range(B)] for k in range(n)], np.int64)
    c.scan_stream_mapped_batch(ptrs, counts, True)
    rows = c.loop_rows(n * B)
    c.close()
    assert sum(r["verified"] for r in rows) > B
    S = _ctx(aloam, M)
    S.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    S.set_loops(True, **LOOP)
    for b in range(B):
        ops = np.full((n, 1), SCAN, np.int32); ops[0] = START   # a lanes START: a fresh cube store and table
        _lanes_run(S, [dev[b]], ops)
        solo = S.loop_rows(n)
        for k in range(n):
            _same_row(rows[k * B + b], solo[k])
    S.close()


def test_lanes_with_a_mid_call_start(aloam, synth):
    n = 16
    scans = [R.traj(synth, t, n, sensor="HDL-32", n_az=600) for t in range(2)]
    M = R.maxn(scans) + 1024
    dev = [R.to_device(tr) for tr in scans]
    c = _ctx(aloam, M, 2)
    c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    c.set_loops(True, **LOOP)
    ops = np.full((n, 2), SCAN, np.int32); ops[0] = START; ops[7, 1] = START
    _lanes_run(c, dev, ops)
    rows = c.loop_rows(n * 2)
    place = c.place_rows(n * 2)
    first = int(place["keyframe"][7 * 2 + 1])
    assert first == 0   # the START cleared lane 1's table
    seen = 0
    for k in range(n):
        for b in range(2):
            r = rows[k * 2 + b]
            if not r["verified"] or (b == 1 and k < 7):   # lane 1's rows before its START: that table is gone
                continue
            if b == 1:
                assert r["query"] <= k - 7 and r["cand"] < r["query"]
            _same_row(r, c.loop_verify(b, r["query"], r["cand"], r["shift"]))
            seen += 1
    assert seen > 0
    c.close()


def test_skip_frame_verifies_mapped_keyframe_rows_only(aloam, synth):
    n = 30
    scans = R.traj(synth, 3, n, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M, mapping_skip_frame=3)
    c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    c.set_loops(True, **LOOP)
    c.scan_stream_mapped([d.data_ptr() for d in dev], [d.shape[0] for d in dev], True)
    rows = c.loop_rows(n)
    seen = 0
    for k, r in enumerate(rows):
        if k % 3:
            assert not r["verified"] and r["query"] == -1
        elif r["verified"]:
            _same_row(r, c.loop_verify(0, r["query"], r["cand"], r["shift"]))
            seen += 1
    assert seen > 0
    c.close()


def test_thin_submap_rows(aloam, synth):
    scans = R.traj(synth, 4, 20, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M)
    c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    c.set_loops(True, max_distance=2.0, window=0, cloud_points=8, outer_iters=2)
    c.scan_stream_mapped([d.data_ptr() for d in dev], [d.shape[0] for d in dev], True)
    rows = c.loop_rows(20)
    rec = c.place_keyframes(0)
    seen = 0
    for r in rows:
        if not r["verified"]:
            continue
        assert r["stats"]["flags"] & aloam.FLAG_MAP_TOO_THIN and r["n_sub"][0] <= 8
        x0 = L.init_pose(rec["pose"][r["cand"]], r["shift"])
        assert np.array_equal(_bits(r["pose"]), _bits(x0))
        qc, qs = c.keyframe_cloud(0, r["query"])
        sc, ss = L.gather([c.keyframe_cloud(0, k) for k in range(len(rec))], rec["pose"], r["cand"], r["cand"])
        assert r["score"] == L.score(qc, qs, x0, sc, ss, 1.0)
        seen += 1
    assert seen > 0
    c.close()


def test_refusals_leave_the_context_unchanged(aloam, synth):
    scans = R.traj(synth, 2, 12, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M, max_map_points=20000)
    _expect(aloam, ERR_STATE, lambda: c.set_loops(True, **LOOP))                 # place recording off
    _expect(aloam, ERR_STATE, lambda: c.loop_verify(0, 1, 0, 0))
    _expect(aloam, ERR_STATE, lambda: c.keyframe_cloud(0, 0))
    c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=64)
    bad = [dict(max_distance=-1.0), dict(max_distance=float("nan")), dict(window=-1), dict(window=65), dict(cloud_points=0),
           dict(cloud_points=M + 1), dict(outer_iters=0), dict(outer_iters=17), dict(inlier_sq=0.0), dict(inlier_sq=1.5)]
    for kw in bad:
        _expect(aloam, ERR_INVALID_ARG, lambda: c.set_loops(True, **{**LOOP, **kw}))
    _expect(aloam, ERR_CAPACITY, lambda: c.set_loops(True, **{**LOOP, "window": 10, "cloud_points": 1000}))   # 21000 > 20000
    c.set_loops(True, **LOOP)
    c.scan_stream_mapped([d.data_ptr() for d in dev], [d.shape[0] for d in dev], True)
    rows = c.loop_rows(12)
    r = next(r for r in rows if r["verified"])
    before = c.loop_verify(0, r["query"], r["cand"], r["shift"])
    n_kf = len(c.place_keyframes(0))
    q, cd = r["query"], r["cand"]
    for args in ((-1, q, cd, 0), (1, q, cd, 0), (0, n_kf, cd, 0), (0, q, q - 2, 0), (0, q, -1, 0), (0, q, cd, 60), (0, q, cd, -1)):
        _expect(aloam, ERR_INVALID_ARG, lambda: c.loop_verify(*args))
    for init in ([0, 0, 0, 0, 1, 2, 3], [0, 0, 0, 1, np.nan, 0, 0], [np.inf, 0, 0, 1, 0, 0, 0]):
        _expect(aloam, ERR_INVALID_ARG, lambda: c.loop_verify(0, q, cd, init=init))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.keyframe_cloud(0, n_kf))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.keyframe_cloud(1, 0))
    _same_row(before, c.loop_verify(0, q, cd, r["shift"]))
    _same_row(rows[0], c.loop_rows(12)[0])
    # init instead of the shift: normalised as aloam_lane_localise normalises, shift ignored
    x0 = L.init_pose(c.place_keyframes(0)["pose"][cd], r["shift"])
    w = c.loop_verify(0, q, cd, init=x0 * np.array([2, 2, 2, 2, 1, 1, 1.0]))
    assert w["shift"] == -1 and w["verified"] == 1
    c.debug_shard_emulate(0, 2)
    _expect(aloam, ERR_STATE, lambda: c.set_loops(True, **LOOP))
    _expect(aloam, ERR_STATE, lambda: c.loop_verify(0, q, cd, 0))
    c.close()
    # aloam_set_place turns loops off; a call made with loops off cannot be read
    c = _ctx(aloam, M)
    c.set_place(True, keyframe_gap=0.5)
    c.set_loops(True, **LOOP)
    c.set_place(True, keyframe_gap=0.5)
    _expect(aloam, ERR_STATE, lambda: c.loop_verify(0, 1, 0, 0))
    c.scan_stream_mapped([d.data_ptr() for d in dev], [d.shape[0] for d in dev], True)
    _expect(aloam, ERR_STATE, lambda: c.loop_rows(12))
    c.close()
