"""CPU: ring assignment (scanRegistration.cpp:166-205) at every decision of the 16-, 32- and 64-line formulas
(tests/ring_edge_cases.py).  The edge sweeps put returns on every float32 angle within 40 ulps of each decision; the offset
layouts fire lasers off the bin centres and off the sensor origin.  Pinned here:
  * the sweeps straddle every decision, and the layouts put returns near the edges, split lasers across rings and (HDL-64)
    leave rings with two lasers or none;
  * a numpy restatement of the line and the formulas gives the oracle's ring ids, and each plausible mis-transcription of
    them (float libm overloads, an FMA in x*x + y*y, the VLP-16 formula in double, floor for int()) does not;
  * the oracle equals the reference's own scanRegistration.cpp (oracle/_ref) on all of it;
  * synth.scan_beams with the nominal beam table is synth.scan_seam bit for bit."""
import numpy as np
import pytest

import ring_edge_cases as E
from refsource import ref_registration

SENSORS = [16, 32, 64]
CLOUDS = ("full", "sharp", "less_sharp", "flat", "less_flat")


@pytest.fixture(scope="module")
def sweeps():
    out = {}
    for ns in SENSORS:
        raw, target, edge = E.edge_scan(ns)
        out[ns] = (raw, target, edge)
    return out


def _expected_full(raw, ns):
    """the ring-major cloud the restatement predicts: surviving returns stably sorted by ring (xyz only)"""
    p = np.asarray(raw, np.float32)
    thres = np.float32(E.MIN_RANGE[ns])
    ok = np.isfinite(p[:, :3]).all(1) & ~((p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1] + p[:, 2] * p[:, 2]) < thres * thres)
    p = p[ok]
    r = E.ring_ids(p, ns)
    keep = r >= 0
    order = np.argsort(r[keep], kind="stable")
    return p[keep][order, :3], r[keep][order], p[~keep]


def _oracle_rings(orc, raw, ns):
    f = orc.Features(raw, ns, E.MIN_RANGE[ns], mode=orc.SORT_CANONICAL)
    return f, f.full[:, 3].astype(np.int32)


@pytest.mark.parametrize("ns", SENSORS)
def test_edge_sweeps_straddle_every_decision(sweeps, ns):
    raw, target, edge = sweeps[ns]
    summary = E.check_edge_scan(raw, target, edge, ns)
    assert len(summary) == len(E.edges(ns))
    print("%d-line edge sweep: %d returns, %d decisions, each straddled: %s" % (ns, len(raw), len(summary),
          ", ".join("%s %d->%d" % (k, v[1], v[2]) for k, v in summary.items())))


@pytest.mark.parametrize("ns", SENSORS)
def test_restatement_equals_the_oracle_on_edge_sweeps(orc, sweeps, ns):
    """the numpy restatement's ring of every return equals the int() of the oracle's intensity, and the returns it drops
    are exactly the ones missing from the oracle's ring-major cloud"""
    raw = sweeps[ns][0]
    f, rings = _oracle_rings(orc, raw, ns)
    xyz, want, dropped = _expected_full(raw, ns)
    assert f.full.shape[0] == xyz.shape[0]
    assert np.array_equal(f.full[:, :3].view(np.uint32), xyz.view(np.uint32))
    assert np.array_equal(rings, want)
    assert len(dropped) > 0 and min(len(f.sharp), len(f.less_sharp), len(f.flat), len(f.less_flat)) > 0


@pytest.mark.parametrize("ns", SENSORS)
def test_each_mutation_changes_a_ring_on_edge_sweeps(orc, sweeps, ns):
    """every mis-transcription that applies to the formula disagrees with the oracle on at least one return"""
    raw = sweeps[ns][0]
    xyz, want, _ = _expected_full(raw, ns)
    _, rings = _oracle_rings(orc, raw, ns)
    assert np.array_equal(rings, want)
    p = np.asarray(raw, np.float32)
    base = E.ring_ids(p, ns)
    found = {}
    for m in E.MUTATIONS:
        if ns not in E.APPLIES[m]:
            continue
        found[m] = int(np.count_nonzero(E.ring_ids(p, ns, m) != base))
        assert found[m] > 0, (ns, m)
    print("%d-line edge sweep, returns whose ring a mutation changes: %s" % (ns, found))


@pytest.mark.parametrize("name", E.LAYOUTS)
def test_offset_layouts(orc, synth, name):
    """the layouts' properties on scans 0-4, and the restatement equal to the oracle on them"""
    ns = {"VLP-16-offset": 16, "HDL-32-offset": 32, "HDL-64-offset": 64}[name]
    for k in range(5):
        raw, summary = E.check_layout(synth, name, k)
        f, rings = _oracle_rings(orc, raw, ns)
        xyz, want, _ = _expected_full(raw, ns)
        assert np.array_equal(f.full[:, :3].view(np.uint32), xyz.view(np.uint32)) and np.array_equal(rings, want), (name, k)
        print(name, k, summary)


@pytest.mark.parametrize("sensor", ["VLP-16", "HDL-32", "HDL-64"])
def test_scan_beams_with_the_nominal_table_is_scan_seam(synth, sensor):
    """the beam-table generator with the nominal elevations and zero origin offsets writes the same bytes as the default
    calls (which the golden files pin), on the default sweep and on a cut, offset, laser-major, counter-clockwise one"""
    ns = synth.SENSORS[sensor][0]
    el = synth.nominal_elevations(sensor)
    a = synth.scan(sensor, 3)
    b = synth.scan_beams(sensor, 3, el, np.zeros(ns))
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    off = np.linspace(-2.0, 2.0, ns)
    a = synth.scan_seam(sensor, 2, -2.5, 1.0, off, True, True, n_az=901)
    b, beams = synth.scan_beams(sensor, 2, el, np.zeros(ns), -2.5, 1.0, off, True, True, n_az=901, return_beams=True)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    assert np.all(np.diff(beams) >= 0) and beams.max() == ns - 1          # laser-major: beam by beam
    # a laser off the origin moves only its own returns, by its offset along z
    dz = np.zeros(ns); dz[1] = 0.05
    c, cb = synth.scan_beams(sensor, 3, el, dz, return_beams=True)
    d, db = synth.scan_beams(sensor, 3, el, None, return_beams=True)
    same = (cb != 1)
    assert np.array_equal(cb[same], db[db != 1]) and np.array_equal(c[same], d[db != 1])


# ------------------------------------------------------------------------------------------------ the reference's own source
def _vs_reference(orc, raw, ns, tag):
    ref = ref_registration(ns, E.MIN_RANGE[ns])
    got = ref.run(raw, orc.SORT_LITERAL)
    want = orc.Features(raw, ns, E.MIN_RANGE[ns], mode=orc.SORT_LITERAL)
    for name in CLOUDS:
        a, b = got[name], getattr(want, name)
        assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (tag, name, a.shape, b.shape)
    n = want.full.shape[0]
    core = slice(5, n - 5)
    assert np.array_equal(got["curvature"][core].view(np.uint32), want.curvature[core].view(np.uint32)), tag
    assert np.array_equal(got["label"][core], want.label[core]) and np.array_equal(got["picked"][core], want.picked[core]), tag
    return got


@pytest.mark.parametrize("ns", SENSORS)
def test_oracle_equals_the_reference_source_on_edge_sweeps(orc, sweeps, ns):
    """scanRegistration.cpp's own line 166 and ring formulas, compiled unmodified, against the oracle on every decision:
    the ring-major cloud, the four feature clouds, curvature, labels and picks bit for bit"""
    raw = sweeps[ns][0]
    got = _vs_reference(orc, raw, ns, ns)
    xyz, want, _ = _expected_full(raw, ns)
    assert np.array_equal(got["full"][:, 3].astype(np.int32), want)


@pytest.mark.parametrize("name", E.LAYOUTS)
def test_oracle_equals_the_reference_source_on_offset_layouts(orc, synth, name):
    ns = {"VLP-16-offset": 16, "HDL-32-offset": 32, "HDL-64-offset": 64}[name]
    for k in range(2):
        _vs_reference(orc, E.layout_scan(synth, name, k), ns, (name, k))
