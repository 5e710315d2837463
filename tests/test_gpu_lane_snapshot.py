"""GPU: lane snapshots (aloam_lane_save / aloam_lane_restore).  A trajectory suspended to a snapshot and resumed -- in the same
lane after other trajectories ran there, in another lane of another context, from device, pinned or pageable memory, or time-
sliced with many others over fewer lanes -- must equal its uninterrupted solo run bit for bit: odometry poses, map poses, stats,
registered clouds and the final cube store (its state and the ALOAM_EXPORT_MAP / _SURROUND bytes).  Refused restores end the
target lane and change no other."""
import struct
from collections import deque

import numpy as np
import pytest

import lane_refs as R

pytestmark = pytest.mark.gpu

ERR_CAPACITY, ERR_NOT_RING_MAJOR, ERR_STATE, ERR_SNAPSHOT = -4, -8, -9, -11
IDLE, SCAN, START = 0, 1, 2


def _ctx(aloam, maxpts, batch=1, mapped=True, ns=16, **cfg):
    extra = {"max_map_points": 400000} if mapped else {}
    return aloam.Aloam(n_scans=ns, max_points=maxpts, max_batch=batch, max_ring_points=4096, **extra, **cfg)


def _entries(dev, i0, i1):
    """the lane entries (address, points, op) of scans i0 .. i1-1 of a device-resident trajectory; scan 0 STARTs it"""
    return [(d.data_ptr(), d.shape[0], START if i == 0 else SCAN) for i, d in enumerate(dev[i0:i1], i0)]


def _call(ctx, batch, lanes, mapped=True):
    """one aloam_scan_stream_lanes call; lanes = {lane: entries} (a lane idles after its entries, absent lanes all call) ->
    {lane: (odometry rows, map rows or None)} of its entries"""
    steps = max(len(e) for e in lanes.values())
    ptrs, counts, ops = np.zeros((steps, batch), np.uint64), np.zeros((steps, batch), np.int64), np.zeros((steps, batch), np.int32)
    for lane, entries in lanes.items():
        for k, (p, n, op) in enumerate(entries):
            ptrs[k, lane], counts[k, lane], ops[k, lane] = p, n, op
    o, m = ctx.scan_stream_lanes(ptrs, counts, ops, True, mapped=mapped)
    return {lane: (o[:len(e), lane], m[:len(e), lane] if mapped else None) for lane, e in lanes.items()}


def _store(aloam, ctx, lane):
    """the cube store of a lane: its state and both exports, as bytes"""
    s = ctx.mapper_state(lane)
    return (s["centre"], s["valid"], s["q_wmap_wodom"].tobytes(), s["t_wmap_wodom"].tobytes(), s["total_corner"], s["total_surf"],
            ctx.mapper_export(aloam.EXPORT_MAP, lane).tobytes(), ctx.mapper_export(aloam.EXPORT_SURROUND, lane).tobytes())


_SOLO = {}


def _solo(aloam, key, dev, maxpts, mapped=True, ns=16, **cfg):
    """the whole trajectory alone on a fresh one-lane context, one call: {odom, map, stats, store}, cached"""
    ck = (key, len(dev), maxpts, mapped, ns, tuple(sorted(cfg.items())))
    if ck not in _SOLO:
        c = _ctx(aloam, maxpts, 1, mapped, ns, **cfg)
        o, m = _call(c, 1, {0: _entries(dev, 0, len(dev))}, mapped)[0]
        _SOLO[ck] = {"odom": o, "map": m, "stats": c.last_batch_stats[0], "store": _store(aloam, c, 0) if mapped else None}
        c.close()
    return _SOLO[ck]


def _same_as_solo(aloam, ref, parts, ctx=None, lane=None, what=""):
    """the rows of a trajectory gathered from several calls (and, given ctx / lane, the store it left) against its solo run"""
    odom = np.concatenate([p[0] for p in parts])
    assert np.array_equal(odom, ref["odom"]), "odometry " + what
    if ref["map"] is not None:
        assert np.array_equal(np.concatenate([p[1] for p in parts]), ref["map"]), "map poses " + what
    if ctx is not None:
        got = _store(aloam, ctx, lane)
        assert got[:6] == ref["store"][:6], "store state " + what
        assert got[6] == ref["store"][6] and got[7] == ref["store"][7], "exported clouds " + what
        assert got[4] + got[5] > 0


def _expect(aloam, code, fn):
    with pytest.raises(aloam.AloamError) as e:
        fn()
    assert e.value.code == code, (e.value.code, code)


def test_save_run_others_in_the_lane_restore_continue(aloam, synth):
    A, B, Cc = R.traj(synth, 0, 10), R.traj(synth, 1, 12), R.traj(synth, 2, 4)
    M = R.maxn([A, B, Cc]) + 1024
    dA, dB, dC = R.to_device(A), R.to_device(B), R.to_device(Cc)
    ctx = _ctx(aloam, M, 2)
    r1 = _call(ctx, 2, {0: _entries(dA, 0, 4), 1: _entries(dB, 0, 4)})
    blob = ctx.lane_save(0)
    info = aloam.snapshot_info(blob)
    assert info["mapped"] and info["scan_index"] == 4 and info["bytes"] == len(blob) and info["n_scans"] == 16 and info["map_points"] > 0
    assert np.array_equal(info["world"], r1[0][0][-1])   # the world pose of its last scan
    assert ctx.lane_save(0).tobytes() == blob.tobytes()   # saving changes nothing
    r2 = _call(ctx, 2, {0: _entries(dC, 0, 4), 1: _entries(dB, 4, 8)})   # another trajectory in lane 0 meanwhile
    ctx.lane_restore(0, blob)
    assert ctx.lane_save(0).tobytes() == blob.tobytes()   # save -> restore -> save: the same bytes
    r3 = _call(ctx, 2, {0: _entries(dA, 4, 10), 1: _entries(dB, 8, 12)})
    _same_as_solo(aloam, _solo(aloam, "A", dA, M), [r1[0], r3[0]], ctx, 0, "of the resumed trajectory")
    _same_as_solo(aloam, _solo(aloam, "B", dB, M), [r1[1], r2[1], r3[1]], ctx, 1, "of the lane beside it")
    _same_as_solo(aloam, _solo(aloam, "C", dC, M), [r2[0]], what="of the trajectory that ran in between")
    ctx.close()


def test_restore_into_another_context_from_device_pinned_and_pageable_memory(aloam, synth):
    import torch
    A = R.traj(synth, 0, 10)
    M = R.maxn([A]) + 1024
    dA = R.to_device(A)
    ctx = _ctx(aloam, M, 2)
    r1 = _call(ctx, 2, {1: _entries(dA, 0, 5)})
    pageable = ctx.lane_save(1)
    n = len(pageable)
    dev = ctx.lane_save(1, torch.empty(n + 64, dtype=torch.uint8, device="cuda"))
    pinned = ctx.lane_save(1, torch.empty(n, dtype=torch.uint8).pin_memory())
    assert dev.numel() == pinned.numel() == n
    assert dev.cpu().numpy().tobytes() == pinned.numpy().tobytes() == pageable.tobytes()
    _expect(aloam, ERR_CAPACITY, lambda: ctx.lane_save(1, torch.zeros(n - 1, dtype=torch.uint8, device="cuda")))
    other = _ctx(aloam, M, 3)   # another width; every lane resumes the same trajectory from its own copy
    other.lane_restore(2, dev)
    other.lane_restore(0, pinned)
    other.lane_restore(1, pageable)
    r2 = _call(other, 3, {lane: _entries(dA, 5, 10) for lane in range(3)})
    ref = _solo(aloam, "A", dA, M)
    for lane in range(3):
        _same_as_solo(aloam, ref, [r1[1], r2[lane]], other, lane, "restored into lane %d" % lane)
    ctx.close(); other.close()


@pytest.mark.parametrize("sensor", ["VLP-16", "HDL-32"])
def test_time_sliced_trajectories_equal_their_solo_runs(aloam, synth, sensor):
    """24 trajectories over 8 lanes in slices of 5 scans: at the end of a slice every unfinished trajectory is saved and goes to
    the back of the queue, the next slice restores the next 8 into the lanes, rotated so a trajectory changes lanes"""
    ns = synth.SENSORS[sensor][0]
    n_traj, lanes, per = 24, 8, 5
    lengths = [7 + (5 * t) % 7 for t in range(n_traj)]   # 7 .. 13 scans
    trajs = [R.traj(synth, 100 + t, lengths[t], sensor=sensor, n_az=600) for t in range(n_traj)]
    M = R.maxn(trajs) + 1024
    dev = [R.to_device(tr) for tr in trajs]
    ctx = _ctx(aloam, M, lanes, ns=ns)
    queue, pos, saved = deque(range(n_traj)), [0] * n_traj, {}
    parts = {t: [] for t in range(n_traj)}
    stores, swaps, rnd = {}, 0, 0
    while queue:
        group = [queue.popleft() for _ in range(min(lanes, len(queue)))]
        lane_of = {t: (i + rnd) % lanes for i, t in enumerate(group)}
        for t in group:
            if t in saved:
                ctx.lane_restore(lane_of[t], saved.pop(t))
                swaps += 1
        res = _call(ctx, lanes, {lane_of[t]: _entries(dev[t], pos[t], min(pos[t] + per, lengths[t])) for t in group})
        for t in group:
            parts[t].append(res[lane_of[t]])
            pos[t] += len(res[lane_of[t]][0])
            if pos[t] < lengths[t]:
                saved[t] = ctx.lane_save(lane_of[t])
                queue.append(t)
            else:
                stores[t] = _store(aloam, ctx, lane_of[t])
        rnd += 1
    assert swaps >= n_traj and not saved
    for t in range(n_traj):
        ref = _solo(aloam, (sensor, t), dev[t], M, ns=ns)
        _same_as_solo(aloam, ref, parts[t], what="of trajectory %d" % t)
        assert stores[t] == ref["store"], "store of trajectory %d" % t
    ctx.close()


def test_mapping_skip_frame_saved_at_a_skipped_and_at_a_mapped_scan(aloam, synth):
    A = R.traj(synth, 3, 12)
    M = R.maxn([A]) + 1024
    dA = R.to_device(A)
    ref = _solo(aloam, "A3", dA, M, mapping_skip_frame=3)
    for cut in (5, 7):   # the last scan run before the save: 4 (skipped), 6 (mapped)
        ctx = _ctx(aloam, M, 1, mapping_skip_frame=3)
        r1 = _call(ctx, 1, {0: _entries(dA, 0, cut)})
        blob = ctx.lane_save(0)
        assert aloam.snapshot_info(blob)["scan_index"] == cut
        _expect(aloam, ERR_SNAPSHOT, lambda: _ctx(aloam, M, 1).lane_restore(0, blob))   # mapping_skip_frame 1
        other = _ctx(aloam, M, 2, mapping_skip_frame=3)
        other.lane_restore(1, blob)
        r2 = _call(other, 2, {1: _entries(dA, cut, 12)})
        _same_as_solo(aloam, ref, [r1[0], r2[1]], other, 1, "cut after %d scans" % cut)
        ctx.close(); other.close()


def test_odometry_only_lane_distortion_and_a_save_right_after_start(aloam, synth):
    A = R.traj(synth, 4, 8)
    M = R.maxn([A]) + 1024
    dA = R.to_device(A)
    # an odometry-only trajectory: it moves into a context that maps (the scan-to-map fields do not count for it)
    ctx = _ctx(aloam, M, 1, mapped=False)
    r1 = _call(ctx, 1, {0: _entries(dA, 0, 3)}, mapped=False)
    blob = ctx.lane_save(0)
    assert not aloam.snapshot_info(blob)["mapped"] and aloam.snapshot_info(blob)["map_points"] == 0
    other = _ctx(aloam, M, 2, line_res=0.3)
    other.lane_restore(1, blob)
    _expect(aloam, ERR_STATE, lambda: _call(other, 2, {1: _entries(dA, 3, 4)}))   # it continues in its own mode only
    r2 = _call(other, 2, {1: _entries(dA, 3, 8)}, mapped=False)
    ref = _solo(aloam, "A4", dA, M, mapped=False)
    _same_as_solo(aloam, ref, [r1[0], r2[1]], what="odometry only")
    assert R.same_stats(other.last_batch_stats[1], ref["stats"])
    # DISTORTION build, saved right after its START (the snapshot of a trajectory that has only initialised)
    src = _ctx(aloam, M, 1, distortion=1)
    r1 = _call(src, 1, {0: _entries(dA, 0, 1)})
    blob = src.lane_save(0)
    assert aloam.snapshot_info(blob)["scan_index"] == 1
    dst = _ctx(aloam, M, 1, distortion=1)
    dst.lane_restore(0, blob)
    r2 = _call(dst, 1, {0: _entries(dA, 1, 8)})
    _same_as_solo(aloam, _solo(aloam, "A4", dA, M, distortion=1), [r1[0], r2[0]], dst, 0, "distortion 1")
    ctx.close(); other.close(); src.close(); dst.close()


def test_registered_rows_of_a_resumed_trajectory(aloam, synth):
    import torch
    A = R.traj(synth, 5, 9)
    M = R.maxn([A]) + 1024
    dA = R.to_device(A)

    def rows_of_second_call(ctx, batch, lane):
        """scans 4 .. 8 with a sink set: the registered cloud of each, in scan order"""
        sink = torch.zeros((5 * M, 4), dtype=torch.float32, device="cuda")
        ctx.set_registered_sink(sink)
        _call(ctx, batch, {lane: _entries(dA, 4, 9)})
        begin, count = ctx.registered_rows(5 * batch)
        out = [sink[begin[r]:begin[r] + count[r]].cpu().numpy() for r in range(lane, 5 * batch, batch)]
        assert all(len(x) > 0 for x in out)
        return out

    solo = _ctx(aloam, M, 1)
    _call(solo, 1, {0: _entries(dA, 0, 4)})
    ref = rows_of_second_call(solo, 1, 0)
    src = _ctx(aloam, M, 1)
    _call(src, 1, {0: _entries(dA, 0, 4)})
    dst = _ctx(aloam, M, 2)
    dst.lane_restore(1, src.lane_save(0))
    got = rows_of_second_call(dst, 2, 1)
    assert all(a.view(np.int32).tobytes() == b.view(np.int32).tobytes() for a, b in zip(got, ref))
    solo.close(); src.close(); dst.close()


def test_refusals_end_the_target_lane_and_change_no_other(aloam, synth):
    A, B = R.traj(synth, 6, 8), R.traj(synth, 7, 8)
    M = R.maxn([A, B]) + 1024
    dA, dB = R.to_device(A), R.to_device(B)
    src = _ctx(aloam, M, 1)
    r1 = _call(src, 1, {0: _entries(dA, 0, 4)})
    blob = src.lane_save(0)
    tgt = _ctx(aloam, M, 2)
    _expect(aloam, ERR_STATE, lambda: tgt.lane_save(0))   # before any lanes call
    rb = [_call(tgt, 2, {0: _entries(dA, 0, 2), 1: _entries(dB, 0, 4)})[1]]
    _expect(aloam, ERR_STATE, lambda: tgt.lane_save(0))   # an idle lane (its trajectory ended at step 2)
    # a configuration that changes results: the target lane (running again after a restore) ends, lane 1 is untouched
    wrong_cfg = _ctx(aloam, M, 1, line_res=0.25)
    _call(wrong_cfg, 1, {0: _entries(dA, 0, 4)})
    wrong = wrong_cfg.lane_save(0)
    tgt.lane_restore(0, blob)
    _expect(aloam, ERR_SNAPSHOT, lambda: tgt.lane_restore(0, wrong))
    _expect(aloam, ERR_STATE, lambda: _call(tgt, 2, {0: _entries(dA, 4, 5), 1: _entries(dB, 4, 5)}))   # lane 0 has ended
    # malformed: a count changed, a truncated blob, a ring order the association cannot use
    bad = blob.copy()
    S = 256 + 16 * sum(struct.unpack_from("<ii", blob.tobytes(), 28))
    counts = np.frombuffer(blob.tobytes(), np.int32, 2 * 4851, S + 592)
    bad[S + 592 + 4 * int(np.argmax(counts >= 0)):][:4] = np.array([-1], np.int32).view(np.uint8)
    _expect(aloam, ERR_SNAPSHOT, lambda: tgt.lane_restore(0, bad))
    _expect(aloam, ERR_SNAPSHOT, lambda: tgt.lane_restore(0, blob[:-16]))
    unordered = blob.copy()
    unordered[256 + 12:256 + 16] = np.array([70.5], np.float32).view(np.uint8)   # intensity of the first less-sharp point: ring 70
    _expect(aloam, ERR_NOT_RING_MAJOR, lambda: tgt.lane_restore(0, unordered))
    # a "last" cloud beyond max_points (an odometry-only snapshot: no slab capacity in its fingerprint)
    odo = _ctx(aloam, M, 1, mapped=False)
    _call(odo, 1, {0: _entries(dA, 0, 3)}, mapped=False)
    oblob = odo.lane_save(0)
    nls, nlf = struct.unpack_from("<ii", oblob.tobytes(), 28)
    small = _ctx(aloam, max(nls, nlf) - 1, 1, mapped=False)
    _expect(aloam, ERR_CAPACITY, lambda: small.lane_restore(0, oblob))
    # a context that emulates a rank of a sharded job
    emu = _ctx(aloam, M, 1)
    emu.debug_shard_emulate(0, 2)
    _expect(aloam, ERR_STATE, lambda: emu.lane_restore(0, blob))
    # lane 1 went on through all of it; lane 0 resumes A from the good snapshot
    tgt.lane_restore(0, blob)
    r2 = _call(tgt, 2, {0: _entries(dA, 4, 8), 1: _entries(dB, 4, 8)})
    rb.append(r2[1])
    _same_as_solo(aloam, _solo(aloam, "A6", dA, M), [r1[0], r2[0]], tgt, 0, "after the refusals")
    _same_as_solo(aloam, _solo(aloam, "B7", dB, M), rb, tgt, 1, "of the lane beside the refusals")
    # a restore puts a context in lanes mode: the lockstep calls are refused until aloam_reset_odometry
    fresh = _ctx(aloam, M, 1)
    fresh.lane_restore(0, blob)
    p, c = np.array([dA[4].data_ptr()], np.uint64), np.array([A[4].shape[0]])
    _expect(aloam, ERR_STATE, lambda: fresh.scan_stream_mapped(p, c, True))
    _expect(aloam, ERR_STATE, lambda: fresh.scan_stream(p, c, True))
    fresh.reset_odometry()
    _expect(aloam, ERR_STATE, lambda: fresh.lane_save(0))   # the reset ended the lane
    o, m = fresh.scan_stream_mapped(p, c, True)
    assert np.isfinite(o).all() and np.isfinite(m).all()
    for x in (src, tgt, wrong_cfg, odo, small, emu, fresh):
        x.close()
