"""Scenes for the stream paths of 128-wide contexts (aloam_create_wide above 64 rings), shared by
tests/test_oracle_wide_streams.py (CPU) and tests/test_gpu_wide_streams.py (GPU).  TEST INFRASTRUCTURE.

The stream calls run other code than the solo entry points: k_ring_features_batch (one CTA per ring and lane), k_compact into
fixed feature slots (ring_w x 12 sharp, 24 flat, 120 less-sharp per ring), the fused association k_odom_assoc<128> over 1536 sharp
+ 3072 flat query slots with the sharp / flat split at slot 1536, and the batched index build.  The scenes here reach those
slots to their ends:

* cap_scan: a field-mode scan of the polygon room of edge_scenes in which every ring it holds yields exactly its caps, 12 sharp,
  24 flat and 120 less-sharp.  Along a ring, runs of 20 returns whose range alternates by about +-0.16 m (every return a corner
  candidate; consecutive returns over 0.224 m apart, so a pick marks no neighbour) alternate with runs of 20 returns on the wall
  (flat candidates); 720 returns per ring give each of the six segments three of each run.  With all 128 rings present, every
  fused slot is occupied: sharp slot 1535 and flat slot 3071 included.
* SCENES: full-cap scans at 128, 96 and 65 rings (the slot table stays 128 wide), and 128-ring scans with features on rings
  64..127 only, on ring 127 only, and on rings {0, 127} only.
* band_rings: per-lane distinct content for a batch: lane j's rings are a band of 16 that moves with j.
* seam_scan: laser-major OS128 scans cut off the azimuth origin with reversed ring ids (synth.scan_rings), whose ratios s leave
  [0, 1] (DISTORTION 1 de-skews them)."""
import numpy as np

import edge_scenes as es
import wide_ring_oracle as WR

CAPS = {"sharp": 12, "flat": 24, "less_sharp": 120}   # per ring: 2 / 4 / 20 per segment, six segments (scanRegistration.cpp)
WIDTH = 128
SHARP_SLOTS, FLAT_SLOTS = WIDTH * CAPS["sharp"], WIDTH * CAPS["flat"]   # 1536, 3072: the fused query slots of a 128-wide context
PER_RING = 720
RUN = 20              # returns per zigzag run and per wall run
MIN_RANGE = 0.3       # synth.RING_RANGES
MOTION = (0.06, -0.04, 0.004)   # sensor motion per frame: x, y (m), yaw (rad)

# name -> (n_scans, rings holding returns, elevation span in degrees of those rings)
SCENES = {
    "full128": (128, tuple(range(128)), 40.0),
    "full96": (96, tuple(range(96)), 40.0),
    "full65": (65, tuple(range(65)), 40.0),
    "high64": (128, tuple(range(64, 128)), 20.0),
    "ring127": (128, (127,), 0.0),
    "ends": (128, (0, 127), 0.8),   # beams 0.8 degrees apart: within the 5 m search radius of each other (nearby_scan = inf)
}


def elevation(rank, n, span):
    """degrees: the rank-th of n rings, the n spread over `span` degrees around the horizon"""
    return span * (rank / max(n - 1, 1) - 0.5)


def band_rings(j, width=16):
    """the rings of lane j in a batch of distinct lanes: a band of `width` that moves by 7 rings per lane (lane 15: 105..120)"""
    return tuple(range(7 * j, 7 * j + width))


def band_scan(j, frame):
    """lane j's scan of a batch of distinct lanes: band_rings(j) over 12 degrees, its own motion and its own amplitudes"""
    return cap_scan(WIDTH, band_rings(j), 12.0, frame, motion=(0.03 + 0.01 * (j % 5), -0.02 + 0.006 * j, 0.002 * (j % 3)), seed=j)


def cap_scan(n_scans, rings, span, frame=0, motion=MOTION, per_ring=PER_RING, seed=0):
    """(n, 4) float32 field-mode raw scan in firing order, ring id in float 3: the rings `rings` of n_scans over `span` degrees
    of elevation, seen from the sensor after `frame` steps of `motion` (x, y, yaw).  Every ring's returns lie on the walls of
    edge_scenes' room (scaled 1.5), with runs of RUN returns pushed out and in by 0.15 .. 0.19 m alternately (a different
    amplitude per return, so that no curvatures tie) between runs of RUN returns on the wall."""
    rng = np.random.default_rng(seed)
    dx, dy, dyaw = (frame * m for m in motion)
    verts = es._ROOM * 1.5 - np.array([dx, dy])
    parts = []
    k = np.arange(per_ring)
    zig = (k // RUN) % 2 == 0
    sign = np.where(k % 2 == 0, 1.0, -1.0)
    for rank, r in enumerate(rings):
        amp = 0.15 + 0.04 * rng.random(per_ring)
        phi_s = np.pi - 2.0 * np.pi * (k + 0.37) / per_ring     # azimuth in the sensor frame, clockwise firing
        phi_w = phi_s + dyaw                                     # ... in the room
        rho = es._room_range(phi_w, verts)
        z = rho * np.tan(np.deg2rad(elevation(rank, len(rings), span)))
        rho = rho + np.where(zig, sign * amp, 0.0)
        p = np.stack([rho * np.cos(phi_s), rho * np.sin(phi_s), z], 1)
        parts.append((p, (k + 0.37) / per_ring + r * 1e-9, float(r)))
    return es._firing_order(parts)


def scene_scan(name, frame=0):
    ns, rings, span = SCENES[name]
    return cap_scan(ns, rings, span, frame)


def seam_scan(synth, frame, reverse=True):
    """a laser-major OS128 scan cut off the azimuth origin (0.6 turn from 45 degrees), ring ids reversed"""
    return WR.scan(synth, "OS128", frame, reverse=reverse, laser_major=True, cut=0.785, coverage=0.6)


def features(raw, n_scans):
    return WR.Features(raw, n_scans, MIN_RANGE)


def per_ring(cloud, n_scans):
    return np.bincount(np.asarray(cloud)[:, 3].astype(np.int64), minlength=n_scans)


def ratios(full):
    """the de-skew ratio s of every return of a ring-major cloud: intensity = ring + 0.1 s (scanPeriod 0.1), s within
    (-4.5, 5.5)"""
    i = np.asarray(full, np.float64)[:, 3]
    return (i - np.round(i - 0.05)) * 10.0


def oracle_chain(orc, raws, n_scans, distortion=False, nearby=2.5):
    """world poses (frames x 7), per-frame (corner, plane) correspondence counts and the features of the oracle's odometry
    over the wide oracle's features of `raws`"""
    od = orc.Odometry(distortion=distortion, nearby_scan=nearby)
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    poses, counts, feats = [], [], []
    for k, raw in enumerate(raws):
        f = features(raw, n_scans)
        feats.append(f)
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
            counts.append((info["corner_corr"], info["plane_corr"]))
        else:
            counts.append(None)
        od.set_last(f.less_sharp, f.less_flat)
        poses.append(np.concatenate([qw, tw]))
    return np.array(poses), counts, feats
