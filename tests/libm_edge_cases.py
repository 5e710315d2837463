"""Returns on the rounding edges of the two transcendentals behind scanRegistration.cpp's ring and sweep-walk decisions,
shared by tests/test_oracle_libm_edges.py (CPU) and tests/test_gpu_libm_edges.py (GPU).  TEST INFRASTRUCTURE.

  * Elevation midpoints (:166).  The float angle is (float)(atan(d) * 180 / M_PI) in double; between the two floats that
    straddle a ring decision (ring_edge_cases.decision) lies their midpoint m, and a return whose double angle lies within
    a few double ulps of m takes the float below or above depending on the last ulp of atan(d).  midpoint_triples() finds,
    exactly, float returns (x, y, z) whose d = (double)z / sqrt((double)(x*x + y*y)) has a correctly rounded double angle
    within BAND ulps of m, and a control set whose angle lies within BAND ulps of the float above.
  * Azimuth thresholds (:141-153,208-236).  threshold_scenes() builds sweeps whose returns take, for each comparison of the
    walk, every float within +-3 ulps of the threshold's float image, with the host libm's atan2f (called through ctypes,
    the function the oracle and the reference's compiled source call) deciding which float a return has.

The correctly rounded references come from mpmath at 200 bits.  Host expectations are computed here at run time."""
import ctypes as C
import ctypes.util
import math
import os
import subprocess
import tempfile

import mpmath
import numpy as np

import ring_edge_cases as E

F32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BAND = 16                    # double ulps around the midpoint: the band of libm_atan.cuh (kAngleBand)
H2_BINADES = (5, 13)         # horizontal range^2 in [2^5, 2^13): 5.7 - 90 m, beyond every sensor's minimum range
mpmath.mp.prec = 200

_LIBM = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_LIBM.atan2f.restype = C.c_float
_LIBM.atan2f.argtypes = [C.c_float, C.c_float]
_LIBM.atan.restype = C.c_double
_LIBM.atan.argtypes = [C.c_double]
_LC = None


def lc():
    """tests/cpp/libm_atan_check.cc, built once per session into a temporary directory"""
    global _LC
    if _LC is None:
        so = os.path.join(tempfile.mkdtemp(prefix="libm_atan_"), "liblibm_atan_check.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fopenmp", "-w",
                               "-I" + os.path.join(ROOT, "a-loam_b200", "csrc"), "-o", so,
                               os.path.join(ROOT, "tests", "cpp", "libm_atan_check.cc"), "-lm"])
        L = C.CDLL(so)
        fp = C.POINTER(C.c_float)
        L.lc_atan2f.restype = L.lc_libm_atan2f.restype = C.c_float
        L.lc_atan2f.argtypes = L.lc_libm_atan2f.argtypes = [C.c_float, C.c_float]
        L.lc_atan_correct.restype = C.c_double
        L.lc_atan_correct.argtypes = [C.c_double, C.c_double]
        L.lc_elevation_deg.restype = C.c_float
        L.lc_elevation_deg.argtypes = [C.c_float, C.c_float, C.c_float]
        L.lc_compare_atan2f_random.restype = C.c_long
        L.lc_compare_atan2f_random.argtypes = [C.c_long, C.c_uint64, fp]
        L.lc_compare_atan2f_pairs.restype = C.c_long
        L.lc_compare_atan2f_pairs.argtypes = [fp, fp, C.c_long]
        L.lc_compare_atanf_range.restype = C.c_long
        L.lc_compare_atanf_range.argtypes = [C.c_uint64, C.c_uint64, fp]
        L.lc_search_triples.restype = C.c_long
        L.lc_search_triples.argtypes = [C.c_double, C.c_double, C.c_double, C.c_uint32, C.c_uint32, fp, C.c_long]
        _LC = L
    return _LC


# ------------------------------------------------------------------------------------------------ host and exact models
def host_ori(x, y):
    """-atan2f(y, x) of the host libm, float32, per return"""
    return np.array([-_LIBM.atan2f(float(b), float(a)) for a, b in zip(np.asarray(x, F32).tolist(), np.asarray(y, F32).tolist())], F32)


def exact_atan2f(y, x):
    """atan2(y, x) rounded correctly to float32"""
    v = mpmath.atan2(mpmath.mpf(float(y)), mpmath.mpf(float(x)))
    f = F32(float(v))
    cands = [np.nextafter(f, F32(-np.inf)), f, np.nextafter(f, F32(np.inf))]
    return min(cands, key=lambda c: abs(mpmath.mpf(float(c)) - v))


def exact_atan(d):
    """atan(d) rounded correctly to double"""
    return float(mpmath.atan(mpmath.mpf(d)))


def angle_of_atan(a):
    """ring_of's two double roundings after atan: fl(fl(a * 180) / M_PI)"""
    return a * 180.0 / math.pi


def _dbits(v):
    return np.float64(v).view(np.int64)


def _dnext(v, k):
    return float(np.int64(_dbits(v) + (k if v > 0 else -k)).view(np.float64)) if v != 0 else float(np.nextafter(0.0, k))


# ------------------------------------------------------------------------------------------------ elevation midpoints
def _d_band(target):
    """[dlo, dhi] of the doubles d whose correctly rounded angle lies within BAND double ulps of `target` (same sign)"""
    d0 = float(mpmath.tan(mpmath.mpf(target) * mpmath.pi / 180))
    tb = int(_dbits(abs(target)))
    hits = []
    for k in range(-4 * BAND - 8, 4 * BAND + 9):
        d = float(np.int64(_dbits(d0) + k).view(np.float64))
        t = angle_of_atan(exact_atan(d))
        if np.sign(t) == np.sign(target) and abs(int(_dbits(abs(t))) - tb) <= BAND:
            hits.append(d)
    assert hits, target
    return min(hits), max(hits)


def _xy_on(h2, phi):
    """float (x, y) with f32(x*x + y*y) == h2 near azimuth phi (atan2 sense), or None"""
    r = math.sqrt(float(h2))
    x0, y0 = F32(r * math.cos(phi)), F32(r * math.sin(phi))
    steps = np.arange(-12, 13)
    xs = x0 + steps.astype(F32) * np.spacing(np.abs(x0))
    ys = y0 + steps.astype(F32) * np.spacing(np.abs(y0))
    X, Y = np.meshgrid(xs.astype(F32), ys.astype(F32))
    hit = (X * X + Y * Y) == F32(h2)
    if not hit.any():
        return None
    k = np.flatnonzero(hit.ravel())
    k = k[np.argmin(np.abs(X.ravel()[k] - x0) + np.abs(Y.ravel()[k] - y0))]
    return F32(X.ravel()[k]), F32(Y.ravel()[k])


def _search(dlo, dhi, binades, cap=64):
    lo, hi = (int(np.float32(2.0 ** binades[0]).view(np.uint32)), int(np.float32(2.0 ** binades[1]).view(np.uint32)))
    out = np.zeros(2 * cap, F32)
    dmid = 0.5 * (dlo + dhi)
    n = lc().lc_search_triples(dlo, dhi, dmid, lo, hi, out.ctypes.data_as(C.POINTER(C.c_float)), cap)
    zh2 = out[:2 * min(n, cap)].reshape(-1, 2)
    return zh2[np.lexsort((zh2[:, 0], zh2[:, 1]))]


_MID = {}


def midpoint_triples(n_scans):
    """{decision name: dict(below, above, mid, d=(dlo, dhi), zh2=(k, 2) midpoint (z, h2), control=(k, 2) (z, h2))} for every decision of the n_scans formula.  Exact: every (z, h2) has its d in the band by construction"""
    if n_scans in _MID:
        return _MID[n_scans]
    out = {}
    for name, ang in E.edges(n_scans):
        below, above = E.decision(ang, n_scans)
        mid = 0.5 * (float(below) + float(above))
        dlo, dhi = _d_band(mid)
        zh2 = _search(dlo, dhi, H2_BINADES)
        clo, chi = _d_band(float(above))
        control = _search(clo, chi, H2_BINADES, cap=2)
        out[name] = dict(below=below, above=above, mid=mid, d=(dlo, dhi), zh2=zh2, control=control)
    _MID[n_scans] = out
    return out


def d_of(x, y, z):
    return float(np.float64(F32(z)) / math.sqrt(float(F32(x) * F32(x) + F32(y) * F32(y))))


def midpoint_scan(n_scans, seed=0):
    """E.edge_scan(n_scans, n_ulps=4) with every midpoint and control triple of midpoint_triples() inserted between two
    returns of the sweep, at the azimuth half-way between them (an exact (x, y) for the triple's h2 there).  Returns
    (raw, kind) with kind 0 for the edge sweep's returns, 1 for midpoint triples, 2 for controls"""
    base, _, _ = E.edge_scan(n_scans, seed=seed, n_ulps=4)
    trip = midpoint_triples(n_scans)
    pts = [(z, h2, 1) for v in trip.values() for z, h2 in v["zh2"]] + [(z, h2, 2) for v in trip.values() for z, h2 in v["control"]]
    phi = np.arctan2(base[:, 1].astype(np.float64), base[:, 0].astype(np.float64))
    slots = np.linspace(len(base) * 0.03, len(base) * 0.97, len(pts)).astype(int)
    rows, kinds, last = [], [], 0
    for (z, h2, kind), s in zip(pts, slots):
        rows.append(base[last:s]); kinds.append(np.zeros(s - last, int))
        a, b = phi[s - 1], phi[s]
        p = None
        for f in (0.5, 0.3, 0.7, 0.2, 0.8):
            p = _xy_on(h2, a + f * ((b - a + math.pi) % (2 * math.pi) - math.pi))
            if p is not None:
                break
        assert p is not None, (n_scans, z, h2)
        rows.append(np.array([[p[0], p[1], z, 0.0]], F32)); kinds.append(np.array([kind]))
        last = s
    rows.append(base[last:]); kinds.append(np.zeros(len(base) - last, int))
    return np.concatenate(rows), np.concatenate(kinds)


# ------------------------------------------------------------------------------------------------ azimuth thresholds
PI = math.pi
TWO_PI = 2 * math.pi
ULPS = 3


def _f(v):
    return float(F32(v))


def _pre(o, s):
    o = float(o)
    if o < s - PI / 2:
        return _f(o + TWO_PI)
    if o > s + PI * 3 / 2:
        return _f(o - TWO_PI)
    return o


# name: (value(o, s, e) -> float compared, threshold(s, e) -> double, taken(value, threshold) -> bool, role)
#   role "pre": a first-half return, "post": a second-half return, "last": the sweep's last return
COMPARISONS = {
    "pre<start-pi/2": (lambda o, s, e: float(o), lambda s, e: s - PI / 2, lambda v, t: v < t, "pre"),
    "pre>start+3pi/2": (lambda o, s, e: float(o), lambda s, e: s + PI * 3 / 2, lambda v, t: v > t, "pre"),
    "half:ori-start>pi": (lambda o, s, e: _f(F32(_pre(o, s)) - F32(s)), lambda s, e: PI, lambda v, t: v > t, "pre"),
    "post<end-3pi/2": (lambda o, s, e: _f(float(o) + TWO_PI), lambda s, e: e - PI * 3 / 2, lambda v, t: v < t, "post"),
    "post>end+pi/2": (lambda o, s, e: _f(float(o) + TWO_PI), lambda s, e: e + PI / 2, lambda v, t: v > t, "post"),
    "end-start>3pi": (lambda o, s, e: _f(F32(_f(float(o) + TWO_PI)) - F32(s)), lambda s, e: 3 * PI, lambda v, t: v > t, "last"),
    "end-start<pi": (lambda o, s, e: _f(F32(_f(float(o) + TWO_PI)) - F32(s)), lambda s, e: PI, lambda v, t: v < t, "last"),
}


def _ori_near(v):
    """raw -atan2f value (in (-pi, pi]) whose comparison value is near v, by comparison"""
    return ((v + PI) % TWO_PI) - PI


def target_oris(name, s, e):
    """(raw float ori, value) for every raw float ori whose comparison value lies within +-ULPS ulps of the float image of
    the threshold: the floats around the analytic position, walked one by one"""
    value, thr, _, _ = COMPARISONS[name]
    T = thr(s, e)
    img = F32(T)
    lo = E._unordered(E._ordered(img) - ULPS)
    hi = E._unordered(E._ordered(img) + ULPS)
    # analytic raw ori for the threshold
    if name.startswith("pre<") or name.startswith("pre>"):
        o0 = T
    elif name.startswith("half"):
        o0 = _ori_near(s + PI)
    elif name.startswith("post"):
        o0 = _ori_near(T - TWO_PI)
    else:
        o0 = _ori_near(T + s - TWO_PI)
    k0 = int(E._ordered(F32(o0)))
    out = []
    for k in range(k0 - 4 * ULPS - 8, k0 + 4 * ULPS + 9):
        o = F32(E._unordered(k))
        if not (-PI < float(o) <= PI):
            continue
        v = value(o, s, e)
        if float(lo) <= v <= float(hi):
            out.append((o, v))
    return out, T


def pairs_for(o, radii=(6.5, 9.0, 13.0, 21.0, 34.0, 55.0, 78.0), per_radius=2):
    """float (x, y) with host -atan2f(y, x) == o, on a fan of rays around azimuth -o at 6.5 - 78 m"""
    phi = -float(o)
    out = []
    for r in radii:
        x0, y0 = F32(r * math.cos(phi)), F32(r * math.sin(phi))
        found = 0
        for i in range(-4, 5):
            for j in range(-4, 5):
                x = F32(x0 + F32(i) * np.spacing(abs(x0)))
                y = F32(y0 + F32(j) * np.spacing(abs(y0)))
                if F32(-_LIBM.atan2f(float(y), float(x))) == o:
                    out.append((x, y))
                    found += 1
                    if found >= per_radius:
                        break
            if found >= per_radius:
                break
    return out


def misrounded(x, y):
    """True when the host libm's atan2f(y, x) is not the correctly rounded float"""
    return F32(_LIBM.atan2f(float(y), float(x))) != exact_atan2f(y, x)


def _ring_z(x, y, ring, n_scans, elev):
    return F32(math.sqrt(float(x) ** 2 + float(y) ** 2) * math.tan(math.radians(elev[ring % len(elev)])))


def _arc(a0, a1, n, r, n_scans, elev, ring0):
    """n filler returns on the azimuths -phi from a0 to a1 (ori sense, increasing), range r, rings cycling"""
    out = []
    for k, o in enumerate(np.linspace(a0, a1, n)):
        phi = -o
        x, y = F32(r * math.cos(phi)), F32(r * math.sin(phi))
        out.append((x, y, _ring_z(x, y, ring0 + k, n_scans, elev)))
    return out


def _pt(o, r, ring, n_scans, elev):
    phi = -o
    x, y = F32(r * math.cos(phi)), F32(r * math.sin(phi))
    return (x, y, _ring_z(x, y, ring, n_scans, elev))


# starts (raw ori of the first return) per comparison: every quadrant and both sides of the +-pi cut where the comparison
# can fire there
STARTS = {
    "pre<start-pi/2": (-1.2, 0.4, 2.9),
    "pre>start+3pi/2": (-2.0, -3.1),
    "half:ori-start>pi": (-2.5, -0.3, 0.8, 2.6),
    "post<end-3pi/2": (2.0, 2.9),
    "post>end+pi/2": (-2.4, -0.6, 1.0),
    "end-start>3pi": (-2.2, -0.4),
    "end-start<pi": (0.5, 2.7),
}


def threshold_scenes(n_scans, elev):
    """[(name, start, raw (n, 4) float32, marks)] for every comparison and start: marks (n,) holds, per return, the index
    of the comparison's target value it was placed on (-1 for filler)"""
    scenes = []
    for name, (value, thr, taken, role) in COMPARISONS.items():
        for s0 in STARTS[name]:
            first = _pt(s0, 12.0, 0, n_scans, elev)
            s = float(host_ori([first[0]], [first[1]])[0])
            if role == "last":
                tg, T = target_oris(name, s, 0.0)
                for t_i, (o, v) in enumerate(tg):
                    pr = pairs_for(o, radii=(11.0,), per_radius=1)
                    if not pr:
                        continue
                    x, y = pr[0]
                    body = _arc(s + 0.05, s + 0.9 * PI, 60, 15.0, n_scans, elev, 1)
                    pts = [first] + body + [(x, y, _ring_z(x, y, 3, n_scans, elev))]
                    marks = [-1] * (len(pts) - 1) + [t_i]
                    scenes.append((name + "#%d" % t_i, s, _raw(pts), np.array(marks)))
                continue
            # the end of the sweep: a last return 0.95 turn clockwise from the start
            e_last = _pt(_ori_near(s + 0.95 * TWO_PI), 12.0, 2, n_scans, elev)
            o_last = float(host_ori([e_last[0]], [e_last[1]])[0])
            e = _f(o_last + TWO_PI)
            if _f(F32(e) - F32(s)) > 3 * PI:
                e = _f(e - TWO_PI)
            elif _f(F32(e) - F32(s)) < PI:
                e = _f(e + TWO_PI)
            tg, T = target_oris(name, s, e)
            assert tg, (name, s0)
            pairs = [(t_i, o, pairs_for(o)) for t_i, (o, v) in enumerate(tg)]
            if role == "post":
                pre = _arc(s + 0.05, s + 0.9 * PI, 50, 15.0, n_scans, elev, 1)
                flip = [_pt(_ori_near(s + 1.05 * PI), 15.0, 4, n_scans, elev)]
                pts, marks = [first] + pre + flip, [-1] * (len(pre) + 2)
                for t_i, o, pr in pairs:
                    for j, (x, y) in enumerate(pr):
                        pts.append((x, y, _ring_z(x, y, 5 + j, n_scans, elev))); marks.append(t_i)
                post = _arc(s + 1.1 * PI, s + 1.85 * PI, 50, 15.0, n_scans, elev, 7)
                pts += post + [e_last]; marks += [-1] * (len(post) + 1)
                scenes.append((name, s, _raw(pts), np.array(marks)))
                continue
            # first-half comparisons: the returns that keep the first branch, then one that flips halfPassed, then (the
            # flipping return's neighbour) a return that would have kept it, now in the second half
            stay = [(t_i, o, pr) for t_i, o, pr in pairs if not _flips(name, o, s, e)]
            go = [(t_i, o, pr) for t_i, o, pr in pairs if _flips(name, o, s, e)]
            for t_f, o_f, pr_f in go:
                if not pr_f:
                    continue
                pre = _arc(s + 0.05, s + 0.6 * PI, 40, 15.0, n_scans, elev, 1)
                pts, marks = [first] + pre, [-1] * (len(pre) + 1)
                for t_i, o, pr in stay:
                    for j, (x, y) in enumerate(pr):
                        pts.append((x, y, _ring_z(x, y, 5 + j, n_scans, elev))); marks.append(t_i)
                x, y = pr_f[0]
                pts.append((x, y, _ring_z(x, y, 4, n_scans, elev))); marks.append(t_f)
                for t_i, o, pr in stay[:2] + go:
                    if pr:
                        x, y = pr[-1]
                        pts.append((x, y, _ring_z(x, y, 6, n_scans, elev))); marks.append(t_i)
                post = _arc(s + 1.2 * PI, s + 1.85 * PI, 40, 15.0, n_scans, elev, 7)
                pts += post + [e_last]; marks += [-1] * (len(post) + 1)
                scenes.append((name + "#%d" % t_f, s, _raw(pts), np.array(marks)))
    return scenes


def _flips(name, o, s, e):
    """whether a first-half return with raw ori o sets halfPassed"""
    return _f(F32(_pre(o, s)) - F32(s)) > PI


def _raw(pts):
    a = np.zeros((len(pts), 4), F32)
    a[:, :3] = np.array([[float(p[0]), float(p[1]), float(p[2])] for p in pts], np.float64).astype(F32)
    return a


# ------------------------------------------------------------------------------------------------ the walk, fed libm
def walk(raw, n_scans, minimum_range, rings=None):
    """scanRegistration.cpp:141-153,208-236 in numpy on the returns that reach the walk, with the host libm's atan2f:
    (index of every walked return, relTime, branch (0 first half, 1 second), start, end)"""
    p = np.asarray(raw, F32)
    thres = F32(minimum_range)
    ok = np.isfinite(p[:, :3]).all(1) & ~((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]) < thres * thres)
    idx = np.flatnonzero(ok)
    ori = host_ori(p[idx, 0], p[idx, 1])
    s = float(ori[0])
    e = _f(float(ori[-1]) + TWO_PI)
    if _f(F32(e) - F32(s)) > 3 * PI:                      # float subtraction, double compare (:145-153)
        e = _f(e - TWO_PI)
    elif _f(F32(e) - F32(s)) < PI:
        e = _f(e + TWO_PI)
    r = E.ring_ids(p[idx], n_scans) if rings is None else rings[idx]
    half, rel, br, keep = False, [], [], []
    for i, o, ring in zip(idx, ori.tolist(), r):
        if ring < 0:
            continue
        if not half:
            o = _pre(o, s)
            half = _f(F32(o) - F32(s)) > PI
            b = 0
        else:
            o = _f(o + TWO_PI)
            if o < e - PI * 3 / 2:
                o = _f(o + TWO_PI)
            elif o > e + PI / 2:
                o = _f(o - TWO_PI)
            b = 1
        rel.append(F32(F32(o) - F32(s)) / F32(F32(e) - F32(s)))
        br.append(b)
        keep.append(i)
    return np.array(keep), np.array(rel, F32), np.array(br), s, e


def intensity(ring, rel):
    return (np.asarray(ring, np.float64) + 0.1 * np.asarray(rel, F32).astype(np.float64)).astype(F32)
