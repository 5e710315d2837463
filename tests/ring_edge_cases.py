"""Returns on the ring edges of scanRegistration.cpp:166-205, shared by tests/test_oracle_ring_edges.py (CPU) and
tests/test_gpu_ring_edges.py (GPU).  TEST INFRASTRUCTURE.

The ring of a return is decided by one line of mixed float / double arithmetic:
    float angle = atan(z / sqrt(x*x + y*y)) * 180 / M_PI      (double atan / sqrt over float products)
followed by the formula of the sensor (VLP-16: float (angle + 15) / 2, then + 0.5 in double, truncated; HDL-32: the 92/3
formula in double, truncated; HDL-64: the float compare angle > 2 and the double compare against -8.83).  The synthetic beams
of synth.scan() sit at the bin centres, where none of these details can change a ring.  Here:
  * ring_ids() restates the line and the three formulas in numpy, with MUTATIONS that a transcription could plausibly make;
  * edges() lists every decision of each formula as an angle, decision() finds the two adjacent float32 angles it falls
    between, and edge_scan() builds a sweep whose returns take every float angle within +-N ulps of every decision;
  * LAYOUTS are seeded beam tables for synth.scan_beams(): calibration offsets and lasers off the sensor origin, so the
    elevation of one laser's returns changes with range and crosses the edges, and (HDL-64) rings fed by two lasers or none."""
import math

import numpy as np

F32 = np.float32
MAX_RING_POINTS = 4096          # ALOAM_MAX_RING_POINTS
SENSOR_OF = {16: "VLP-16", 32: "HDL-32", 64: "HDL-64"}
MIN_RANGE = {16: 0.3, 32: 0.3, 64: 5.0}

# ------------------------------------------------------------------------------------------------ the line and the formulas
MUTATIONS = ("float_overloads", "fma", "vlp16_double", "floor")
APPLIES = {"float_overloads": (16, 32, 64), "fma": (16, 32, 64), "vlp16_double": (16,), "floor": (16, 32)}


def _f32(a):
    return np.asarray(a, np.float64).astype(F32)


def elevation(xyz, mutation=None):
    """the float angle of :166 for (n, >=3) float32 points.  libm through Python's math module (the C double functions of the
    host, as in oracle/features.cc), not numpy's vectorised kernels, whose float64 atan need not be glibc's"""
    p = np.ascontiguousarray(np.asarray(xyz)[:, :3], F32)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    xx, yy = x * x, y * y                                                       # float products (numpy never contracts)
    if mutation == "fma":                                                       # x*x + y*y contracted: fma(y, y, x*x)
        h2 = _f32(xx.astype(np.float64) + y.astype(np.float64) * y.astype(np.float64))
    else:
        h2 = xx + yy
    z64 = z.astype(np.float64)
    if mutation == "float_overloads":                                           # atan(float) / sqrt(float): float results
        s = _f32([math.sqrt(v) for v in h2.astype(np.float64)])
        r = z / s
        at = _f32([math.atan(v) for v in r.astype(np.float64)])
        return _f32((at * F32(180)).astype(np.float64) / math.pi)
    h = [math.sqrt(v) for v in h2.astype(np.float64)]
    return _f32([math.atan(zz / hh) * 180 / math.pi for zz, hh in zip(z64.tolist(), h)])


def ring_of_angle(angle, n_scans, mutation=None):
    """ring id of float32 angles by the formula of n_scans (-1: dropped), oracle/features.cc ring_of"""
    a = np.asarray(angle, F32)
    a64 = a.astype(np.float64)
    cut = np.floor if mutation == "floor" else np.trunc
    with np.errstate(invalid="ignore"):
        if n_scans == 16:
            v = (a64 + 15) / 2 if mutation == "vlp16_double" else ((a + F32(15)) / F32(2)).astype(np.float64)
            idf = cut(v + 0.5)
            return np.where((idf > 15) | (idf < 0), -1, idf).astype(np.int64)
        if n_scans == 32:
            idf = cut((a64 + 92.0 / 3.0) * 3.0 / 4.0)
            return np.where((idf > 31) | (idf < 0), -1, idf).astype(np.int64)
        up = cut((F32(2) - a).astype(np.float64) * 3.0 + 0.5)
        lo = 32 + cut((-8.83 - a64) * 2.0 + 0.5)
        idf = np.where(a64 >= -8.83, up, lo)
        drop = (a > F32(2)) | (a64 < -24.33) | (idf > 50) | (idf < 0)
        return np.where(drop, -1, idf).astype(np.int64)


def ring_ids(xyz, n_scans, mutation=None):
    return ring_of_angle(elevation(xyz, mutation), n_scans, mutation)


def branch_64(angle):
    """which HDL-64 formula decides (True: the upper one, angle >= -8.83 in double)"""
    return np.asarray(angle, F32).astype(np.float64) >= -8.83


# ------------------------------------------------------------------------------------------------ decisions
def edges(n_scans):
    """[(name, angle [deg])] of every decision of the formula, oracle/features.cc ring_of"""
    if n_scans == 16:
        return [("ring%d|%d" % (k - 1, k), 2.0 * k - 16) for k in range(1, 16)] + [("drop>=16", 16.0), ("drop<=-18", -18.0)]
    if n_scans == 32:
        return ([("ring%d|%d" % (k - 1, k), -92.0 / 3 + 4.0 * k / 3) for k in range(1, 32)]
                + [("drop>=12", 12.0), ("drop<=-32", -32.0)])
    return ([("drop>2", 2.0)] + [("ring%d|%d" % (k - 1, k), 2.0 - (k - 0.5) / 3) for k in range(1, 33)]
            + [("branch-8.83", -8.83)] + [("ring%d|%d" % (31 + m, 32 + m), -8.83 - (m - 0.5) / 2) for m in range(1, 19)]
            + [("drop<=-18.08", -8.83 - 18.5 / 2)])


def _outcome(a, n_scans):
    r = ring_of_angle(a, n_scans)
    return r * 2 + branch_64(a) if n_scans == 64 else r


def _ordered(a):
    """float32 -> an int64 that increases with the float (and back)"""
    i = np.asarray(a, F32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def _unordered(k):
    k = np.asarray(k, np.int64)
    return np.where(k < 0, (-k) | 0x80000000, k).astype(np.uint32).view(np.int32).view(F32)


def decision(angle, n_scans, width=0.01):
    """the largest float32 below the decision near `angle` and the smallest above it: ring_of_angle (and for HDL-64 the
    branch) differs between them and is constant on either side within `width` degrees"""
    lo, hi = _ordered(F32(angle - width)), _ordered(F32(angle + width))
    o_lo, o_hi = _outcome(_unordered(lo), n_scans), _outcome(_unordered(hi), n_scans)
    assert o_lo != o_hi, (angle, n_scans)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if _outcome(_unordered(mid), n_scans) == o_lo:
            lo = mid
        else:
            hi = mid
    return F32(_unordered(lo)), F32(_unordered(hi))


def angles_around(angle, n_scans, n_ulps):
    """the 2 n_ulps float32 angles nearest the decision, n_ulps on either side, ascending"""
    below, above = decision(angle, n_scans)
    k = _ordered(above)
    return _unordered(np.arange(k - n_ulps, k + n_ulps)), below, above


# ------------------------------------------------------------------------------------------------ the edge sweep
_ROOM = np.array([[8.0, 1.0], [4.0, 9.0], [-6.0, 7.5], [-9.0, -1.0], [-3.0, -8.0], [7.0, -6.5]])   # convex, around 0


def _room_range(phi, verts):
    d = np.stack([np.cos(phi), np.sin(phi)], 1)
    best = np.full(len(phi), np.inf)
    for i in range(len(verts)):
        a, b = verts[i], verts[(i + 1) % len(verts)]
        e = b - a
        den = d[:, 0] * (-e[1]) - d[:, 1] * (-e[0])
        with np.errstate(divide="ignore", invalid="ignore"):
            t = (a[0] * (-e[1]) - a[1] * (-e[0])) / den
            u = (d[:, 0] * a[1] - d[:, 1] * a[0]) / den
        best = np.where((t > 0) & (u >= -1e-12) & (u <= 1 + 1e-12) & (t < best), t, best)
    return best


SCALES = {16: (0.4, 1.0, 2.5, 5.0, 9.0), 32: (0.4, 1.0, 2.5, 5.0, 9.0), 64: (1.0, 2.0, 4.0, 7.0, 9.0)}


def copies(j, n_ulps):
    """returns per float angle: many on the two floats that straddle the decision and their neighbours (where float vs
    double arithmetic, FMA contraction and the libm overloads move a return across), a few elsewhere"""
    d = min(abs(j), abs(j + 1))
    return 48 if d == 0 else 16 if d <= 2 else 2


def _tune_z(x, y, target, max_steps=6):
    """z (float32) with elevation(x, y, z) == target where one exists near x, y; NaN where this (x, y) skips the target"""
    h = np.sqrt((x * x + y * y).astype(np.float64))
    z = _f32(h * np.tan(np.deg2rad(target.astype(np.float64))))
    for _ in range(max_steps):
        a = elevation(np.stack([x, y, z], 1))
        if np.all(a == target):
            break
        z = np.where(a < target, np.nextafter(z, F32(np.inf)), np.where(a > target, np.nextafter(z, F32(-np.inf)), z))
    a = elevation(np.stack([x, y, z], 1))
    return np.where(a == target, z, F32(np.nan))


def edge_scan(n_scans, seed=0, n_ulps=40, shift=(0.0, 0.0)):
    """One sweep whose returns sit on every decision of the n_scans formula: for each decision, every float32 angle within
    n_ulps of it (copies() returns each, at different azimuths and ranges).  Each decision owns one sector of the
    revolution; its returns lie on the walls of a polygon room scaled to put their horizontal range between ~2 and ~80 m.
    Returns in firing order (clockwise, -atan2(y, x) increasing), an odd number of azimuth slots so none sits half a turn
    from the first one.  Returns (raw (n, 4) float32, target float angle of every return, decision index of every return)."""
    rng = np.random.default_rng(1000 * n_scans + seed)
    ed = edges(n_scans)
    per_edge, targets = [], []
    for e, (_, ang) in enumerate(ed):
        around, _, _ = angles_around(ang, n_scans, n_ulps)
        reps = np.array([copies(j, n_ulps) for j in range(-n_ulps, n_ulps)])
        t = np.repeat(around, reps)
        per_edge.append(t[rng.permutation(len(t))])
    n = sum(len(t) for t in per_edge)
    n_slot = n + 1 - n % 2 + 2 * len(ed)                    # odd, a few spare slots between sectors
    phi_all = math.pi - 2 * math.pi * (np.arange(n_slot) + 0.37) / n_slot
    verts = _ROOM - np.asarray(shift)
    xs, ys, zs, ts, es = [], [], [], [], []
    slot = 0
    order = rng.permutation(len(ed))                        # sector order: neighbouring decisions not in neighbouring sectors
    for e in order:
        t = per_edge[e]
        phi = phi_all[slot:slot + len(t)]
        scale = SCALES[n_scans][e % len(SCALES[n_scans])]
        rho = _room_range(phi, verts * scale)
        x, y = _f32(rho * np.cos(phi)), _f32(rho * np.sin(phi))
        z = _tune_z(x, y, t)
        for k in range(1, 40):                              # move the misses 0.1 mm along their ray and try again
            miss = np.isnan(z)
            if not miss.any():
                break
            f = 1.0 + 1e-5 * k * (1 if k % 2 else -1)
            x[miss], y[miss] = _f32(rho[miss] * f * np.cos(phi[miss])), _f32(rho[miss] * f * np.sin(phi[miss]))
            z[miss] = _tune_z(x[miss], y[miss], t[miss])
        assert not np.isnan(z).any(), (n_scans, ed[e])
        xs.append(x); ys.append(y); zs.append(z); ts.append(t); es.append(np.full(len(t), e))
        slot += len(t) + 2
    raw = np.zeros((sum(len(x) for x in xs), 4), F32)
    raw[:, 0], raw[:, 1], raw[:, 2] = np.concatenate(xs), np.concatenate(ys), np.concatenate(zs)
    return raw, np.concatenate(ts), np.concatenate(es)


def check_edge_scan(raw, target, edge_of, n_scans, n_ulps=40):
    """what makes the sweep worth testing: every return has its target float angle, each decision is straddled (both of
    its outcomes occur, on the two adjacent floats), every ring fits ALOAM_MAX_RING_POINTS and no return is near an azimuth
    threshold of the sweep walk.  Returns {decision name: (returns, outcome below, outcome above)}."""
    a = elevation(raw)
    assert np.array_equal(a, target)
    out = {}
    for e, (name, ang) in enumerate(edges(n_scans)):
        below, above = decision(ang, n_scans)
        m = edge_of == e
        o = _outcome(a[m], n_scans)
        ob, oa = _outcome(below, n_scans), _outcome(above, n_scans)
        assert np.count_nonzero(a[m] == below) > 0 and np.count_nonzero(a[m] == above) > 0, name
        assert set(np.unique(o).tolist()) == {int(ob), int(oa)}, name
        assert np.count_nonzero(a[m] < below) == np.count_nonzero(a[m] > above), name        # symmetric
        vals = np.unique(a[m])
        assert len(vals) == 2 * n_ulps and np.all(np.diff(_ordered(vals)) == 1), name        # every float, none skipped
        out[name] = (int(m.sum()), int(ob), int(oa))
    rings = ring_ids(raw, n_scans)
    assert np.bincount(rings[rings >= 0], minlength=n_scans).max() <= MAX_RING_POINTS
    assert azimuth_margins_ok(raw, n_scans, MIN_RANGE[n_scans])
    return out


def azimuth_margins_ok(raw, n_scans, minimum_range, margin=1e-5):
    """synth.cc check_seam_margins: no surviving return within `margin` rad of an azimuth threshold of the reference's
    sweep walk (scanRegistration.cpp:141-153,208-236), where host and device atan2f may take different branches"""
    p = np.asarray(raw, F32)
    thres = F32(minimum_range)
    keep = np.flatnonzero(~((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]) < thres * thres))
    if len(keep) == 0:
        return True
    ori = (-np.arctan2(p[:, 1].astype(np.float64), p[:, 0].astype(np.float64))).astype(F32).astype(np.float64)
    pi = math.pi
    start = ori[keep[0]]
    end_raw = float(F32(ori[keep[-1]] + 2 * pi))
    near = lambda a, b: abs(a - b) < margin
    if near(end_raw - start, 3 * pi) or near(end_raw - start, pi):
        return False
    end = end_raw
    if end - start > 3 * pi:
        end = float(F32(end - 2 * pi))
    elif end - start < pi:
        end = float(F32(end + 2 * pi))
    rings = ring_ids(p[keep], n_scans)
    half = False
    for i, r in zip(keep, rings):
        if r < 0:
            continue
        o = ori[i]
        pre = near(o, start - pi / 2) or near(o, start + pi * 3 / 2)
        post = near(o + 2 * pi, end - pi * 3 / 2) or near(o + 2 * pi, end + pi / 2)
        if not half:
            if o < start - pi / 2:
                o = float(F32(o + 2 * pi))
            elif o > start + pi * 3 / 2:
                o = float(F32(o - 2 * pi))
            if pre or (near(o - start, pi) and post):
                return False
            half = o - start > pi
        elif post:
            return False
    return True


# ------------------------------------------------------------------------------------------------ beams off the bin centres
def _layout(name):
    """(sensor, elevations [deg], vertical laser origins [m]) of a seeded beam table"""
    rng = np.random.default_rng({"VLP-16-offset": 16, "HDL-32-offset": 32, "HDL-64-offset": 64}[name])
    if name == "VLP-16-offset":
        # even lasers: calibration offsets of up to 0.2 deg near the centres; odd lasers: 0.05-0.3 deg from the ring's
        # upper edge with an origin 3-10 cm off the sensor's, on the side that carries near returns across the edge
        el, dz = [], []
        for b in range(16):
            if b % 2 == 0 or b == 15:
                el.append(-15.0 + 2.0 * b + rng.uniform(-0.2, 0.2)); dz.append(rng.uniform(-0.02, 0.02))
            else:
                s = 1.0 if b % 4 == 1 else -1.0
                el.append(-14.0 + 2.0 * b - s * rng.uniform(0.05, 0.3)); dz.append(s * rng.uniform(0.03, 0.1))
        return "VLP-16", np.array(el), np.array(dz)
    if name == "HDL-32-offset":
        # every fourth laser sits on the edge above its ring and the laser of the next ring is left out, so the two rings
        # share one laser's returns (a ring holding two whole lasers would exceed 4096 returns at 2200 columns)
        el, dz = [], []
        for b in range(32):
            if b % 4 == 3:
                continue
            if b % 4 == 2:
                # below the edge by the shift its origin gives at the laser's typical range (the ground 1.8 m below the
                # sensor, or the walls ~14 m away): returns nearer or farther than that land on either side
                edge = -92.0 / 3 + 4.0 * (b + 1) / 3
                d = (1.0 if b % 8 == 2 else -1.0) * rng.uniform(0.01, 0.04)
                r_typ = 1.8 / math.tan(math.radians(-edge)) if edge < -7.0 else 14.0
                el.append(edge - math.degrees(d * math.cos(math.radians(edge)) / r_typ) + rng.uniform(-0.003, 0.003)); dz.append(d)
            else:
                el.append(-92.0 / 3 + (b + 0.5) * 4.0 / 3 + rng.uniform(-0.3, 0.3)); dz.append(rng.uniform(-0.02, 0.02))
        return "HDL-32", np.array(el), np.array(dz)
    # HDL-64: per-laser calibration offsets of 0.1 deg (rms) against bins of 1/3 deg, the upper block's origin 3 cm above
    # the sensor's and the lower block's 3 cm below; laser 10 fires into ring 11 (ring 10 left without a laser, ring 11 with
    # two) and lasers 20-23 sit on the edges of their rings
    up = 1.96 - np.arange(32) / 3.0 + rng.normal(0, 0.1, 32)
    up[10] = 2.0 - 11 / 3.0 + 0.05
    up[20:24] = 2.0 - (np.arange(20, 24) + 0.5) / 3.0 + rng.uniform(-0.03, 0.03, 4)
    lo = -8.87 - 0.5 * np.arange(32) + rng.normal(0, 0.12, 32)
    dz = np.concatenate([0.03 + rng.normal(0, 0.005, 32), -0.03 + rng.normal(0, 0.005, 32)])
    return "HDL-64", np.concatenate([up, lo]), dz


LAYOUTS = ("VLP-16-offset", "HDL-32-offset", "HDL-64-offset")
# fraction of a scan's returns within 0.02 deg of a ring edge, at least (measured on scans 0-4)
NEAR_EDGE_FRACTION = {"VLP-16-offset": 0.05, "HDL-32-offset": 0.15, "HDL-64-offset": 0.06}


def layout_scan(synth, name, index, return_beams=False):
    sensor, el, dz = _layout(name)
    return synth.scan_beams(sensor, index, el, dz, return_beams=return_beams)


def edge_distance(angle, n_scans):
    """distance [deg] of float angles to the nearest ring edge or drop edge of the formula"""
    e = np.array([a for _, a in edges(n_scans) if not _.startswith("branch")])
    return np.abs(np.asarray(angle, np.float64)[:, None] - e[None, :]).min(1)


def check_layout(synth, name, index):
    """the properties that make a layout worth testing; returns a summary dict"""
    sensor, el, _ = _layout(name)
    ns = synth.SENSORS[sensor][0]
    raw, beam = layout_scan(synth, name, index, return_beams=True)
    a = elevation(raw)
    rings = ring_of_angle(a, ns)
    near = float(np.mean(edge_distance(a, ns) < 0.02))
    assert near >= NEAR_EDGE_FRACTION[name], (name, index, near)
    counts = np.bincount(rings[rings >= 0], minlength=ns)
    assert counts.max() <= MAX_RING_POINTS, (name, index, counts.max())
    # lasers whose returns land in more than one ring (the edge crossings the layout is for)
    split = [b for b in range(len(el)) if len(np.unique(rings[(beam == b) & (rings >= 0)])) > 1]
    assert len(split) >= 3, (name, index, split)
    out = {"returns": len(raw), "near_edge": near, "max_ring": int(counts.max()), "split_lasers": len(split)}
    if ns == 64:
        major = {}
        for b in range(len(el)):
            r = rings[(beam == b) & (rings >= 0)]
            if len(r):
                major.setdefault(int(np.bincount(r).argmax()), []).append(b)
        two = [r for r, bs in major.items() if len(bs) >= 2]
        none = [r for r in range(51) if r not in major]
        assert two and none, (name, index, two, none)
        out.update(two_lasers=two, no_laser=none)
    return raw, out
