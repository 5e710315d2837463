"""GPU: place recognition (aloam_set_place, aloam_place_*) against the oracle of oracle/place.cc -- descriptors bit for bit on
real and crafted scans, query distances, shifts and order, headings of rotated scans, keyframes and loop candidates recorded by
the mapped stream calls (from the device's own map poses), recording off changing nothing, relocalisation without a pose guess
through place hypotheses, and refusals that leave the context unchanged."""
import numpy as np
import pytest

import lane_refs as R
import pyplace as P
import reloc_cases as RC

pytestmark = pytest.mark.gpu

ERR_INVALID_ARG, ERR_CAPACITY, ERR_STATE = -1, -4, -9
IDLE, SCAN, START = 0, 1, 2


def _ctx(aloam, maxpts, batch=1, ns=32, **cfg):
    kw = {"max_ring_points": 4096, "max_map_points": 400000, **cfg}
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, **kw)


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if np.asarray(a).dtype == np.float32 else np.uint64)


def _records(descs, poses=None):
    r = np.zeros(len(descs), P.RECORD_DTYPE)
    r["pose"][:, 3] = 1.0
    if poses is not None:
        r["pose"] = poses
    r["max_range"], r["z_offset"], r["desc"] = 80.0, 2.0, descs
    return r


@pytest.mark.parametrize("sensor", ["VLP-16", "HDL-32", "HDL-64"])
def test_descriptors_equal_the_oracle(aloam, synth, sensor):
    ns = synth.SENSORS[sensor][0]
    scans = [synth.scan(sensor, k) for k in (0, 7)]
    c = _ctx(aloam, max(s.shape[0] for s in scans) + 1024, ns=ns)
    for s in scans:
        f = c.extract_features(s)
        d = c.place_describe(f["less_sharp"], f["less_flat"])
        assert np.array_equal(_bits(d), _bits(P.describe(f["less_sharp"], f["less_flat"])))
        assert np.array_equal(_bits(c.place_describe(raw=s)), _bits(d))
        # the whole raw scan as one cloud, and other descriptor parameters
        c.set_place(False, max_range=35.5, z_offset=-1.25)
        assert np.array_equal(_bits(c.place_describe(s, np.zeros((0, 4), np.float32))), _bits(P.describe(s, np.zeros((0, 4)), 35.5, -1.25)))
        c.set_place(False)
    c.close()


def test_descriptor_of_a_128_ring_scan(aloam, synth):
    s = synth.scan_rings("OS128", 3)
    c = aloam.Aloam(n_scans=128, max_points=s.shape[0] + 1024, wide=True, ring_source=aloam.RING_FIELD, max_ring_points=2048)
    f = c.extract_features(s)
    assert np.array_equal(_bits(c.place_describe(f["less_sharp"], f["less_flat"])), _bits(P.describe(f["less_sharp"], f["less_flat"])))
    c.close()


def test_descriptors_of_crafted_edge_clouds(aloam):
    mr = np.float32(80.0)
    edge = [(4.0, 0, 1.0), (np.nextafter(np.float32(4.0), np.float32(0)), 0, 2.0), (80.0, 0, 3.0), (np.nextafter(mr, np.float32(0)), 0, 5.0),
            (0.0, 10.0, -1.0), (0.0, -10.0, -3.5), (-10.0, -0.0, -2.0), (-10.0, 0.0, -2.0), (10, 0, -2.0), (10.1, 0, -2.0),
            (0.0, 0.0, 7.0), (1e-30, -1e-30, 1.0), (79.99, 0.01, 100.0), (-0.0, -0.0, 0.5)]
    a = np.zeros((len(edge), 4), np.float32); a[:, :3] = np.asarray(edge, np.float32)
    rng = np.random.default_rng(5)
    b = (rng.normal(size=(20000, 4)) * 40).astype(np.float32)
    c = _ctx(aloam, 30000)
    for z_off in (2.0, 0.0, -0.0, -2.0):
        c.set_place(False, z_offset=z_off)
        for x, y in ((a, np.zeros((0, 4), np.float32)), (a, b), (np.zeros((0, 4), np.float32), np.zeros((0, 4), np.float32))):
            assert np.array_equal(_bits(c.place_describe(x, y)), _bits(P.describe(x, y, 80.0, z_off)))
    c.close()


@pytest.mark.parametrize("M", [1, 63, 1000, 20000])
def test_queries_equal_the_oracle(aloam, M):
    rng = np.random.default_rng(M)
    base = rng.uniform(-1, 6, (max(M // 2, 1), 1200)).astype(np.float32)
    base[:, rng.integers(0, 1200, 200)] = 0.0
    db = base[rng.integers(0, base.shape[0], M)]             # duplicate records
    q = np.concatenate([db[rng.integers(0, M, 3)], rng.uniform(-1, 6, (2, 1200)).astype(np.float32)])
    q[0] = np.roll(q[0].reshape(20, 60), 11, axis=1).ravel()
    k = min(10, M)
    c = _ctx(aloam, 1000)
    c.place_db_load(_records(db))
    got = c.place_query(q, k)
    idx, sh, dist = P.query(q, db, k)
    assert np.array_equal(got["keyframe"], idx) and np.array_equal(got["shift"], sh)
    assert np.array_equal(_bits(got["distance"]), _bits(dist))
    c.close()


def test_a_rotated_scan_matches_at_its_shift(aloam, synth):
    s = synth.scan("HDL-32", 4)
    c = _ctx(aloam, s.shape[0] + 1024)
    f = c.extract_features(s)
    descs = []
    for k in range(0, 60, 7):
        th = np.deg2rad(6.0 * k + 0.5)
        rot = lambda a: np.column_stack([np.cos(th) * a[:, 0] - np.sin(th) * a[:, 1], np.sin(th) * a[:, 0] + np.cos(th) * a[:, 1], a[:, 2], a[:, 3]]).astype(np.float32)
        descs.append(c.place_describe(rot(f["less_sharp"]), rot(f["less_flat"])))
    c.place_db_load(_records(np.stack(descs)))
    q = c.place_describe(f["less_sharp"], f["less_flat"])
    got = c.place_query(q, len(descs))
    for j, k in enumerate(range(0, 60, 7)):
        pos = list(got["keyframe"][0]).index(j)
        assert got["shift"][0][pos] == k, (k, got)
    c.close()


def _mapped_run(aloam, synth, skip, batch, lanes_call):
    scans = [R.traj(synth, t, 12, sensor="HDL-32", n_az=600) for t in range(batch)]
    M = R.maxn(scans) + 1024
    c = _ctx(aloam, M, batch, mapping_skip_frame=skip)
    c.set_place(True, keyframe_gap=0.5, exclude_recent=2, max_keyframes=6)
    fx = _ctx(aloam, M)
    feats = [[fx.extract_features(s) for s in tr] for tr in scans]
    fx.close()
    dev = [R.to_device(tr) for tr in scans]
    n = len(scans[0])
    ptrs = np.array([[dev[b][k].data_ptr() for b in range(batch)] for k in range(n)], np.uint64)
    counts = np.array([[dev[b][k].shape[0] for b in range(batch)] for k in range(n)], np.int64)
    if lanes_call:
        ops = np.full((n, batch), SCAN, np.int32); ops[0] = START; ops[7] = START   # a second START clears the tables
        _, m = c.scan_stream_lanes(ptrs, counts, ops, True)
    else:
        ops = np.full((n, batch), SCAN, np.int32); ops[0] = START
        _, m = c.scan_stream_mapped_batch(ptrs, counts, True) if batch > 1 else c.scan_stream_mapped([p[0] for p in ptrs], counts[:, 0], True)
        m = m.reshape(n, batch, 7)
    rows = c.place_rows(n * batch)
    for b in range(batch):
        T = P.KeyframeTable(b, keyframe_gap=0.5, exclude_recent=2, max_keyframes=6)
        j = 0
        for k in range(n):
            r = k * batch + b
            if ops[k, b] == START:
                j = 0
            if j % skip:
                assert (rows["keyframe"][r], rows["loop"][r], rows["distance"][r]) == (-1, -1, -1.0)
            else:
                e = T.add(feats[b][k]["less_sharp"], feats[b][k]["less_flat"], m[k, b], j, start=ops[k, b] == START)
                got = {key: rows[key][r] for key in ("keyframe", "loop", "shift", "full")}
                assert got == {key: e[key] for key in got}, (b, k, got, e)
                assert _bits(np.float64(rows["distance"][r])) == _bits(np.float64(e["distance"]))
            j += 1
        rec = c.place_keyframes(b)
        assert rec.tobytes() == T.records.tobytes()
    return c


@pytest.mark.parametrize("skip", [1, 3])
def test_recording_in_the_mapped_stream(aloam, synth, skip):
    _mapped_run(aloam, synth, skip, 1, False).close()


def test_recording_in_a_16_lane_batch(aloam, synth):
    _mapped_run(aloam, synth, 1, 16, False).close()


def test_recording_in_lanes_and_what_clears_a_table(aloam, synth):
    c = _mapped_run(aloam, synth, 1, 2, True)
    assert len(c.place_keyframes(0)) > 0
    blob = c.lane_save(0)
    c.lane_restore(0, blob)
    assert len(c.place_keyframes(0)) == 0 and len(c.place_keyframes(1)) > 0
    c.reset_odometry()
    assert len(c.place_keyframes(1)) == 0
    c.close()


def test_recording_off_issues_what_a_context_without_it_issues(aloam, synth):
    scans = R.traj(synth, 0, 6, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    outs = []
    for setup in (lambda c: None, lambda c: (c.set_place(True), c.set_place(False))):
        c = _ctx(aloam, M)
        setup(c)
        n0 = c.launch_count()
        o, m = c.scan_stream_mapped([d.data_ptr() for d in dev], [d.shape[0] for d in dev], True)
        outs.append((c.launch_count() - n0, o, m))
        c.close()
    assert outs[0][0] == outs[1][0]
    assert np.array_equal(outs[0][1], outs[1][1]) and np.array_equal(outs[0][2], outs[1][2])


def test_loop_candidates_of_a_return_trip(aloam, synth):
    out = R.traj(synth, 0, 40, sensor="HDL-32", n_az=600)
    back = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 50, n_az=700) for k in range(38, -1, -1)]
    scans = out + back
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M)
    c.set_place(True, keyframe_gap=0.0, exclude_recent=10, max_keyframes=200)
    ops = np.full((len(scans), 1), SCAN, np.int32); ops[0] = START
    ptrs = np.array([[d.data_ptr()] for d in dev], np.uint64); counts = np.array([[d.shape[0]] for d in dev], np.int64)
    _, m = c.scan_stream_lanes(ptrs, counts, ops, True)
    rows = c.place_rows(len(scans))
    fx = _ctx(aloam, M)
    T = P.KeyframeTable(0, keyframe_gap=0.0, exclude_recent=10, max_keyframes=200)
    for k, s in enumerate(scans):
        f = fx.extract_features(s)
        e = T.add(f["less_sharp"], f["less_flat"], m[k, 0], k, start=k == 0)
        assert (rows["keyframe"][k], rows["loop"][k], rows["shift"][k]) == (e["keyframe"], e["loop"], e["shift"])
    fx.close()
    for i, k in enumerate(range(38, -1, -1)):
        if k <= 33:
            assert abs(int(rows["loop"][40 + i]) - k) <= 1, (k, rows["loop"][40 + i])
    c.close()


def test_relocalisation_without_a_pose_guess(aloam, synth):
    import struct
    scans = R.traj(synth, 0, 60, sensor="HDL-32", n_az=600)
    dev = R.to_device(scans)
    M = R.maxn([scans]) + 1024
    c = _ctx(aloam, M)
    c.set_place(True, keyframe_gap=2.0, max_keyframes=64)
    ops = np.full((60, 1), SCAN, np.int32); ops[0] = START
    _, m = c.scan_stream_lanes(np.array([[d.data_ptr()] for d in dev], np.uint64), np.array([[d.shape[0]] for d in dev], np.int64), ops, True)
    rows = c.place_rows(60)
    rec = c.place_keyframes(0)
    blob = c.lane_save(0)
    c.close()
    L = _ctx(aloam, M)
    L.prior_map_load(blob)
    L.place_db_load(rec)
    n_scored = 0
    checked = 0
    for k in range(60):
        if rows["keyframe"][k] >= 0:
            continue
        f = L.extract_features(scans[k])
        match = L.place_query(L.place_describe(f["less_sharp"], f["less_flat"]), 3)
        hyps = aloam.place_hypotheses({"keyframe": match["keyframe"][0], "shift": match["shift"][0]}, rec, 2.0, 1.0, np.deg2rad(10), np.deg2rad(5))
        n_scored = max(n_scored, hyps.shape[0])
        res, _ = L.prior_relocalise(hyps, f["less_sharp"], f["less_flat"], refine=1, scores=False)
        p = res[0]["pose"]
        dq = abs(float(np.dot(p[:4], m[k, 0, :4])))
        assert np.linalg.norm(p[4:] - m[k, 0, 4:]) < RC.NEAR_M and 2 * np.arccos(min(1.0, dq)) < RC.NEAR_RAD, k
        checked += 1
    assert checked > 0 and n_scored * 10 < 31752
    L.close()


def test_refusals_leave_the_context_unchanged(aloam):
    c = _ctx(aloam, 1000)
    bad = [dict(max_range=0.0), dict(max_range=float("nan")), dict(z_offset=float("inf")), dict(keyframe_gap=-1.0),
           dict(exclude_recent=-1), dict(max_keyframes=0), dict(max_keyframes=65537)]
    for kw in bad:
        _expect(aloam, ERR_INVALID_ARG, lambda: c.set_place(True, **kw))
    _expect(aloam, ERR_STATE, lambda: c.place_keyframes(0))
    _expect(aloam, ERR_STATE, lambda: c.place_rows(1))
    _expect(aloam, ERR_STATE, lambda: c.place_query(np.zeros(1200, np.float32), 1))
    rng = np.random.default_rng(0)
    db = _records(rng.uniform(0, 5, (5, 1200)).astype(np.float32))
    c.place_db_load(db)
    before = c.place_query(db["desc"][:2], 5)
    for mutate in (lambda r: r["max_range"].__setitem__(0, 80.5), lambda r: r["z_offset"].__setitem__(1, -2.0),
                   lambda r: r["desc"].__setitem__((2, 7), np.inf), lambda r: r["pose"].__setitem__((3, 4), np.nan)):
        r = db.copy(); mutate(r)
        _expect(aloam, ERR_INVALID_ARG, lambda: c.place_db_load(r))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.place_query(db["desc"][:2], 6))
    _expect(aloam, ERR_INVALID_ARG, lambda: c.place_query(db["desc"][:2], 0))
    _expect(aloam, ERR_CAPACITY, lambda: c.place_describe(np.zeros((1001, 4), np.float32), np.zeros((0, 4), np.float32)))
    after = c.place_query(db["desc"][:2], 5)
    assert all(np.array_equal(before[k], after[k]) for k in before)
    c.debug_shard_emulate(0, 2)
    _expect(aloam, ERR_STATE, lambda: c.set_place(True))
    c.close()
