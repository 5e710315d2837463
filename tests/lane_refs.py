"""References shared by the lane-width and long-stream GPU tests: seeded trajectories, solo runs of one trajectory through
the single-trajectory stream calls on a fresh context, and the CPU oracle chain (ascanRegistration | alaserOdometry |
alaserMapping).  Both references are cached for the session, so every distinct trajectory is run solo and through the
oracle once, whichever test and lane it appears in."""
import numpy as np

from conftest import rot_angle

STAT_KEYS = ("n_corner_corr", "n_plane_corr", "lm_iters", "accepted_steps", "flags", "termination", "init_cost", "final_cost")
BAR = 1e-4   # north-star: metres / radians

_SCANS, _SOLO, _ORACLE = {}, {}, {}


def traj(synth, t, n, sensor="VLP-16", n_az=900):
    """scans 0 .. n-1 of trajectory t (seed BASE_SEED + 50 + t), cached"""
    out = []
    for k in range(n):
        key = (sensor, t, n_az, k)
        if key not in _SCANS:
            _SCANS[key] = synth.scan(sensor, k, seed=synth.BASE_SEED + 50 + t, n_az=n_az)
        out.append(_SCANS[key])
    return out


def maxn(trajs):
    return max(s.shape[0] for tr in trajs for s in tr)


def to_device(scans):
    import torch
    return [torch.from_numpy(s).cuda() for s in scans]


def splits_of(n, sizes):
    """consecutive slices of range(n) with the given call sizes (they must add up to n)"""
    assert sum(sizes) == n, (sizes, n)
    edges = np.cumsum([0] + list(sizes))
    return [slice(int(a), int(b)) for a, b in zip(edges[:-1], edges[1:])]


def snapshot(ctx, lane):
    """mapper state and every cube of its valid block, both cloud types, as bytes"""
    s = ctx.mapper_state(lane)
    cubes = {(c, w): ctx.mapper_cube(w, c, lane).view(np.int32).tobytes() for c in s["valid"] for w in (0, 1)}
    return s, cubes


def same_store(got, ref, what):
    """two snapshots: the same state and the same bits in every cube"""
    (sa, ca), (sb, cb) = got, ref
    assert sa["centre"] == sb["centre"] and sa["valid"] == sb["valid"], what
    assert np.array_equal(sa["q_wmap_wodom"], sb["q_wmap_wodom"]) and np.array_equal(sa["t_wmap_wodom"], sb["t_wmap_wodom"]), what
    assert (sa["total_corner"], sa["total_surf"]) == (sb["total_corner"], sb["total_surf"]), what
    bad = [k for k in ca if ca[k] != cb[k]]
    assert not bad, (what, "cubes (index, type) differ", bad[:4])
    assert sa["total_corner"] + sa["total_surf"] > 0


def same_stats(a, b):
    return all(a[k] == b[k] for k in STAT_KEYS)


def solo(aloam, scans, key, mapped, distortion=0, sizes=None, ns=16, max_ring=4096, maxpts=None):
    """the trajectory alone on a fresh context through aloam_scan_stream(_mapped), device-resident, in calls of `sizes`
    scans (default: one call).  Returns {odom, map (or None), stats (of the last call), store (snapshot or None)}; cached
    under (key, mapped, distortion, sizes)."""
    sizes = tuple(sizes or (len(scans),))
    ck = (key, bool(mapped), int(distortion), sizes, max_ring)
    if ck not in _SOLO:
        dev = to_device(scans)
        extra = {"max_map_points": 400000} if mapped else {}
        c = aloam.Aloam(n_scans=ns, max_points=(maxpts or maxn([scans])) + 1024, max_ring_points=max_ring, distortion=distortion, **extra)
        ptrs = np.array([d.data_ptr() for d in dev], np.uint64)
        counts = np.array([s.shape[0] for s in scans])
        odom, mp = [], []
        for s in splits_of(len(scans), sizes):
            if mapped:
                o, m = c.scan_stream_mapped(ptrs[s], counts[s], True)
                mp.append(m)
                st = None
            else:
                o, st = c.scan_stream(ptrs[s], counts[s], True)
                st = st.as_dict()
            odom.append(o)
        _SOLO[ck] = {"odom": np.concatenate(odom), "map": np.concatenate(mp) if mapped else None, "stats": st,
                     "store": snapshot(c, 0) if mapped else None}
        c.close()
    return _SOLO[ck]


def oracle(orc, synth, scans, key, mapped, distortion=0, sensor="VLP-16", leaves=None):
    """the oracle chain over `scans`: (odometry world poses, map poses or None), (n, 7) each; the mapping stage filters
    with the sensor's leaf sizes unless `leaves` = (line_res, plane_res) is given.  The chain is causal, so a cached longer
    run of the same trajectory answers a shorter one."""
    n = len(scans)
    ck = (key, bool(mapped), bool(distortion), leaves)
    if ck not in _ORACLE or len(_ORACLE[ck][0]) < n:
        ns, _, mr, line_res, plane_res = synth.SENSORS[sensor]
        if leaves is not None:
            line_res, plane_res = leaves
        od = orc.Odometry(distortion=bool(distortion))
        cm = orc.CubeMap() if mapped else None
        q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
        odom, mp = [], []
        for k, raw in enumerate(scans):
            f = orc.Features(raw, ns, mr)
            if k > 0:
                q, t, _ = od.register(f.sharp, f.flat, q, t)
                qw, tw = orc.integrate_pose(qw, tw, q, t)
            od.set_last(f.less_sharp, f.less_flat)
            odom.append(np.concatenate([qw, tw]))
            if mapped:
                pose, _ = cm.step(f.less_sharp, f.less_flat, qw, tw, line_res, plane_res)
                mp.append(pose)
        _ORACLE[ck] = (np.array(odom), np.array(mp) if mapped else None)
    o, m = _ORACLE[ck]
    return o[:n], (m[:n] if mapped else None)


def deviation(got, ref):
    """(largest translation deviation, largest rotation angle) over the rows of two (n, 7) pose arrays"""
    return float(np.abs(got[:, 4:] - ref[:, 4:]).max()), max(rot_angle(got[k, :4], ref[k, :4]) for k in range(len(got)))


def assert_near(got, ref, what):
    dt, dr = deviation(got, ref)
    assert dt < BAR and dr < BAR, "%s: %.3g m / %.3g rad from the oracle (bar %g)" % (what, dt, dr, BAR)
    return dt, dr
