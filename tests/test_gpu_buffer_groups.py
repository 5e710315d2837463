"""GPU: the buffers a later call replaces (place recognition's tables, database and scratch, loop verification's per-lane sets,
recovery's candidates, the relocaliser's hypotheses, the prior map and its build scratch).  Three contexts in a row, each driven
through every replacement, give identical results and give back their memory at close; replacing a group again and again does
not hold on to the groups it replaced; a loop setting refused for want of memory leaves the earlier one as it was."""
import numpy as np
import pytest

import lane_refs as R
import recovery_cases as RV
import track_cases as TC

pytestmark = pytest.mark.gpu

ERR_CUDA = -5
IDLE, SCAN, START = 0, 1, 2
LOOP = dict(max_distance=2.0, window=5, cloud_points=1000, outer_iters=4, inlier_sq=1.0)
MIB = 1 << 20
# free device memory after each close() of the lifecycle test moves by at most this much: one 2 MiB page of the driver's
# accounting (measured on an H100 80GB HBM3: no drift at all over the three rounds, before and after the buffers moved into
# groups); the replacement cycles move by up to 4 MiB between cycles, far below one leaked group (21 MB or more)
LIFECYCLE_DRIFT = 2 * MIB
CYCLE_DRIFT = 8 * MIB


def _ctx(aloam, maxpts, batch=1, **cfg):
    kw = {"max_ring_points": 4096, "max_map_points": 400000, **cfg}
    return aloam.Aloam(n_scans=32, max_points=maxpts, max_batch=batch, **kw)


def _lanes(c, batch, lanes):
    """one mapped aloam_scan_stream_lanes call; lanes = {lane: [(device scan, op)]} -> (odometry, map) poses"""
    steps = max(len(e) for e in lanes.values())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for lane, entries in lanes.items():
        for k, (d, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = d.data_ptr(), d.shape[0], op
    return c.scan_stream_lanes(ptrs, counts, ops, True)


def _run(dev, first=True):
    return [(d, START if first and i == 0 else SCAN) for i, d in enumerate(dev)]


def _free():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def _flat(x):
    """every array of a result, in order"""
    if isinstance(x, dict):
        return [a for k in sorted(x) for a in _flat(x[k])]
    if isinstance(x, (list, tuple)):
        return [a for v in x for a in _flat(v)]
    return [np.asarray(x)]


# ---- HDL-32 trajectory 0 out and back over the same places, and the features of its first scans
@pytest.fixture(scope="module")
def trip(aloam, synth):
    out = R.traj(synth, 0, 40, sensor="HDL-32", n_az=600)
    back = [synth.scan("HDL-32", k, seed=synth.BASE_SEED + 50, n_az=700) for k in range(38, -1, -1)]
    scans = out + back
    M = R.maxn([scans]) + 1024
    fx = _ctx(aloam, M)
    feats = [fx.extract_features(s) for s in scans[:6]]
    fx.close()
    return dict(dev=R.to_device(scans), M=M, feats=feats, n=len(scans))


def _round(aloam, trip):
    """one context through every replaceable buffer group -> every output, in order"""
    dev, feats, n = trip["dev"], trip["feats"], trip["n"]
    c = _ctx(aloam, trip["M"], batch=2)
    out = []
    for mk in (16, 64, 200):                                  # larger keyframe tables and pair scratch
        c.set_place(True, keyframe_gap=0.0, exclude_recent=10, max_keyframes=mk)
    c.set_loops(True, **{**LOOP, "cloud_points": 500})
    c.set_loops(True, **LOOP)                                 # the per-lane sets replaced
    out += list(_lanes(c, 2, {0: _run(dev)}))
    out += [c.loop_rows(2 * n), c.place_rows(2 * n)]
    rec = c.place_keyframes(0)
    out += [rec.tobytes(), c.loop_verify(0, 30, 5, 0), c.keyframe_cloud(0, 12)]
    c.place_db_load(rec[:10])
    c.place_db_load(rec)                                      # the database replaced
    descs = np.stack([c.place_describe(f["less_sharp"], f["less_flat"]) for f in feats])
    for nq in (1, 3, len(descs)):                             # larger query scratch
        out.append(c.place_query(descs[:nq], 3))
    c.prior_map_load(c.lane_save(0))
    corner = np.concatenate([f["less_sharp"] for f in feats])
    surf = np.concatenate([f["less_flat"] for f in feats])
    out.append(c.prior_map_build(corner, surf))               # the map replaced, through the build's scratch
    out.append(c.prior_map_digest())
    D = RV.deltas(aloam)
    f = feats[0]
    for nh in (8, 200, len(D)):                               # larger hypothesis buffers
        out.append(c.prior_relocalise(D[:nh], f["less_sharp"], f["less_flat"], inlier_sq=0.5, max_score_points=256, refine=2))
    c.set_place(False)
    c.set_loops(False)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    for nd in (50, 500, len(D)):                              # larger candidate buffers
        c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D[:nd])
    c.lane_localise(1, np.array([0, 0, 0, 1.0]), np.zeros(3))
    out += list(_lanes(c, 2, {1: _run(dev[:6])}))
    out += [c.map_rows(12), c.recovery_rows(12)]
    c.close()
    return _flat(out)


def test_three_contexts_through_every_group(aloam, trip):
    _round(aloam, trip)   # warm-up: module loads and the caching allocator's first blocks
    free, rounds = [], []
    for _ in range(3):
        rounds.append(_round(aloam, trip))
        free.append(_free())
    print("free MiB after each close:", [f / MIB for f in free])
    for later in rounds[1:]:
        assert len(later) == len(rounds[0])
        for a, b in zip(rounds[0], later):
            assert a.shape == b.shape and a.tobytes() == b.tobytes()
    assert max(free) - min(free) <= LIFECYCLE_DRIFT, [f / MIB for f in free]


def test_replacements_free_what_they_replace(aloam, trip):
    dev = trip["dev"]
    c = _ctx(aloam, trip["M"])
    c.set_place(True, keyframe_gap=0.0, exclude_recent=10, max_keyframes=1000)
    _lanes(c, 1, {0: _run(dev[:10])})
    small = c.lane_save(0)
    _lanes(c, 1, {0: _run(dev[10:40], first=False)})
    large = c.lane_save(0)
    rec = c.place_keyframes(0)
    db = [np.resize(rec, 4000), np.resize(rec, 8000)]        # 21 and 43 MB of records
    free = []
    for cycle in range(10):
        for i in (0, 1):
            c.set_loops(True, **{**LOOP, "cloud_points": 2000 * (i + 1)})   # 64 and 128 MB of keyframe clouds
            c.place_db_load(db[i])
            c.prior_map_load((small, large)[i])
        free.append(_free())
    print("free MiB after each cycle:", [f / MIB for f in free])
    assert abs(free[-1] - free[1]) <= CYCLE_DRIFT, [f / MIB for f in free]
    c.close()


def test_a_refused_loop_setting_leaves_the_earlier_one(aloam, trip):
    dev = trip["dev"]
    P = 131072
    c = _ctx(aloam, P)
    c.set_place(True, keyframe_gap=0.0, exclude_recent=10, max_keyframes=65536)
    c.set_loops(True, **LOOP)
    _lanes(c, 1, {0: _run(dev)})
    before = _flat([c.loop_verify(0, 30, 5, 0), c.keyframe_cloud(0, 12), c.keyframe_cloud(0, 30)])
    free0 = _free()
    with pytest.raises(aloam.AloamError) as e:   # a cloud pool of 65536 x 2 x 131072 points: 275 GB
        c.set_loops(True, max_distance=2.0, window=0, cloud_points=P)
    assert e.value.code == ERR_CUDA, e.value.code
    free1 = _free()
    print("free MiB before / after the refusal:", free0 / MIB, free1 / MIB)
    assert free0 - free1 <= 32 * MIB
    after = _flat([c.loop_verify(0, 30, 5, 0), c.keyframe_cloud(0, 12), c.keyframe_cloud(0, 30)])
    assert len(after) == len(before)
    for a, b in zip(before, after):
        assert a.shape == b.shape and a.tobytes() == b.tobytes()
    c.close()
