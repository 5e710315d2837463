"""CPU: the transcendentals of ring assignment and the sweep walk at their rounding edges (tests/libm_edge_cases.py).
Pinned here:
  * the device's atan2f restatement (a-loam_b200/csrc/libm_atan.cuh, built for the host) equals the host libm's atan2f on
    1e8 random pairs and on every threshold return, and its atanf equals libm's on every finite float;
  * its correctly rounded atan (the device's fallback near a float rounding boundary of the angle) equals mpmath's;
  * every elevation triple has its d and its exact angle in the midpoint band, the host libm's atan is correctly rounded
    on every triple (so the oracle and a correctly rounded device agree), and the oracle's ring equals the libm model;
  * every azimuth target float is reached, both branches occur on each threshold, and the libm-fed walk model gives the
    oracle's relTime bit for bit;
  * the reference's own scanRegistration.cpp equals the oracle on the new scans."""
import math

import numpy as np
import pytest

import libm_edge_cases as M
import ring_edge_cases as E
from refsource import ref_registration

SENSORS = [16, 32, 64]
CLOUDS = ("full", "sharp", "less_sharp", "flat", "less_flat")


def test_atan2f_restatement_equals_libm_on_random_pairs():
    first = np.zeros(2, np.float32)
    import ctypes as C
    bad = M.lc().lc_compare_atan2f_random(100_000_000, 12345, first.ctypes.data_as(C.POINTER(C.c_float)))
    assert bad == 0, (bad, first)


def test_atanf_restatement_equals_libm_on_every_float():
    import ctypes as C
    first = np.zeros(1, np.float32)
    bad = M.lc().lc_compare_atanf_range(0, 1 << 32, first.ctypes.data_as(C.POINTER(C.c_float)))
    assert bad == 0, (bad, first)


def test_atan_correct_rounds_correctly():
    """the double-double fallback against mpmath, started from approximations up to 3 ulps off, over the elevation range"""
    rng = np.random.default_rng(7)
    ds = np.concatenate([rng.uniform(-0.6, 0.3, 3000), rng.uniform(-50, 50, 300), [0.0, 1e-300, -1e-20, 1e20]])
    for d in ds.tolist():
        want = M.exact_atan(d)
        for k in (-3, 0, 2):
            a0 = float(np.nextafter(want, np.inf)) if k > 0 else float(np.nextafter(want, -np.inf)) if k < 0 else want
            assert M.lc().lc_atan_correct(d, a0) == want, (d, k)


@pytest.fixture(scope="module")
def triples():
    return {ns: M.midpoint_triples(ns) for ns in SENSORS}


@pytest.mark.parametrize("ns", SENSORS)
def test_midpoint_triples(orc, triples, ns):
    """each triple's d lies in the band of doubles whose correctly rounded angle is within BAND ulps of the midpoint; the
    host's atan equals the correctly rounded one on every d found (none is a residual); the host's float angle is one of
    the two floats of the decision; the oracle's ring is the libm model's"""
    rows, residual, empty = [], [], []
    for name, v in triples[ns].items():
        dlo, dhi = v["d"]
        tb = int(M._dbits(abs(v["mid"])))
        for z, h2 in v["zh2"].tolist() + v["control"].tolist():
            d = float(np.float64(np.float32(z)) / math.sqrt(float(np.float32(h2))))
            assert dlo <= d <= dhi or [z, h2] in v["control"].tolist(), (name, z, h2)
        for z, h2 in v["zh2"].tolist():
            d = float(np.float64(np.float32(z)) / math.sqrt(float(np.float32(h2))))
            t = M.angle_of_atan(M.exact_atan(d))
            assert abs(int(M._dbits(abs(t))) - tb) <= M.BAND, (name, d)
            if math.atan(d) != M.exact_atan(d):
                residual.append((name, d))
            p = M._xy_on(h2, 0.7)
            assert p is not None
            a = E.elevation(np.array([[p[0], p[1], z]], np.float32))[0]
            assert a in (v["below"], v["above"]), (name, a)
            assert np.float32(M.lc().lc_elevation_deg(p[0], p[1], z)) == a, (name, d)
        if len(v["zh2"]) == 0:
            empty.append(name)
        rows.append("%s %d" % (name, len(v["zh2"])))
    assert residual == [], residual
    # every decision is reached or listed: the float returns at 5.7-90 m whose d falls in the band
    reached = len(triples[ns]) - len(empty)
    assert reached >= len(triples[ns]) // 2, (ns, empty)
    print("%d-line midpoint triples per decision (0 = no float return at 5.7-90 m has its d in the band): %s" % (ns, ", ".join(rows)))
    raw, kind = M.midpoint_scan(ns)
    f = orc.Features(raw, ns, E.MIN_RANGE[ns], orc.SORT_CANONICAL)
    rings = E.ring_ids(raw, ns)
    thres = np.float32(E.MIN_RANGE[ns])
    p = raw
    ok = ~((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]) < thres * thres)
    keep = ok & (rings >= 0)
    order = np.argsort(rings[keep], kind="stable")
    assert np.array_equal(f.full[:, :3].view(np.uint32), raw[keep][order, :3].view(np.uint32))
    assert np.array_equal(f.full[:, 3].astype(np.int32), rings[keep][order])
    assert np.count_nonzero(kind == 1) == sum(len(v["zh2"]) for v in triples[ns].values())


@pytest.mark.parametrize("ns", SENSORS)
def test_oracle_equals_the_reference_source_on_midpoint_scans(orc, ns):
    raw, _ = M.midpoint_scan(ns)
    _vs_reference(orc, raw, ns, ("midpoint", ns))


def _vs_reference(orc, raw, ns, tag):
    ref = ref_registration(ns, E.MIN_RANGE[ns])
    got = ref.run(raw, orc.SORT_LITERAL)
    want = orc.Features(raw, ns, E.MIN_RANGE[ns], mode=orc.SORT_LITERAL)
    for name in CLOUDS:
        a, b = got[name], getattr(want, name)
        assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (tag, name)


def elevations(synth, ns):
    return list(synth.nominal_elevations(E.SENSOR_OF[ns]))


@pytest.fixture(scope="module")
def scenes(synth):
    return {ns: M.threshold_scenes(ns, elevations(synth, ns)) for ns in SENSORS}


@pytest.mark.parametrize("ns", SENSORS)
def test_threshold_scenes_reach_every_target(scenes, ns):
    """per comparison: every target float within +-3 ulps of the threshold's image is reached, both outcomes occur, the
    restatement equals libm on every threshold return, and the scenes hold returns the host libm misrounds (counted per
    comparison: near +-pi/2 the libm result is rarely off)"""
    import ctypes as C
    by, report = {}, []
    for name, s, raw, marks in scenes[ns]:
        base = name.split("#")[0]
        value, thr, taken, role = M.COMPARISONS[base]
        pts = raw[marks >= 0]
        ori = M.host_ori(pts[:, 0], pts[:, 1])
        d = by.setdefault(base, {"vals": set(), "taken": set(), "n": 0, "mis": 0})
        for (x, y, _, _), o in zip(pts.tolist(), ori.tolist()):
            d["vals"].add(value(np.float32(o), s, 0.0))    # no comparison's value depends on the end
            d["n"] += 1
            d["mis"] += bool(M.misrounded(x, y))
        y = np.ascontiguousarray(pts[:, 1]); x = np.ascontiguousarray(pts[:, 0])
        assert M.lc().lc_compare_atan2f_pairs(y.ctypes.data_as(C.POINTER(C.c_float)), x.ctypes.data_as(C.POINTER(C.c_float)), len(x)) == 0
    for base, (value, thr, taken, role) in M.COMPARISONS.items():
        d = by[base]
        assert len(d["vals"]) >= 2 * M.ULPS + 1, (base, sorted(d["vals"]))
        report.append("%s: %d returns, %d target values, %d misrounded by libm" % (base, d["n"], len(d["vals"]), d["mis"]))
    assert sum(d["mis"] for d in by.values()) > 0
    print("%d-line threshold scenes: %s" % (ns, "; ".join(report)))


@pytest.mark.parametrize("ns", SENSORS)
def test_walk_model_equals_the_oracle_relTime(orc, scenes, ns):
    """the libm-fed walk model reproduces the oracle's intensity bit for bit on every scene; both branches of every
    threshold occur"""
    branches = set()
    for name, s, raw, marks in scenes[ns]:
        f = orc.Features(raw, ns, E.MIN_RANGE[ns], orc.SORT_CANONICAL)
        idx, rel, br, s_, e_ = M.walk(raw, ns, E.MIN_RANGE[ns])
        rings = E.ring_ids(raw, ns)[idx]
        want = M.intensity(rings, rel)
        order = np.argsort(rings, kind="stable")
        assert np.array_equal(f.full[:, :3].view(np.uint32), raw[idx][order, :3].view(np.uint32)), name
        assert np.array_equal(f.full[:, 3].view(np.uint32), want[order].view(np.uint32)), name
        branches |= {(name.split("#")[0], int(b)) for b in br}
    for base, (_, _, _, role) in M.COMPARISONS.items():
        assert (base, 0) in branches and (base, 1 if role != "last" else 0) in branches, base


@pytest.mark.parametrize("ns", [16, 64])
def test_oracle_equals_the_reference_source_on_threshold_scenes(orc, scenes, ns):
    for name, s, raw, marks in scenes[ns]:
        _vs_reference(orc, raw, ns, (name, ns))
