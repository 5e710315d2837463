"""CPU: driver rings up to 128 (aloam_create_wide) -- the wide oracle against the 64-ring field oracle and a model of ring
assignment and the sweep walk, the reference's own laserOdometry.cpp on 65..128-ring clouds, the synthetic wide sensors, the
configuration checks that run before any device is used and a 128-ring snapshot header."""
import struct

import numpy as np
import pytest

import ring_field_oracle as RF
import wide_ring_oracle as WR
from test_oracle_ring_field import _model, _same, _header, assert_same_features

F32 = np.float32


# ------------------------------------------------------------------------------------------------ 1. the wide oracle
def test_wide_source_edits_only_the_ring_bound():
    src, field = WR.wide_source(), RF.field_source()
    assert src.count("n_scans > 128") == 1 and "n_scans > 64" not in src
    assert src.replace("n_scans > 128", "n_scans > 64") == field


@pytest.mark.parametrize("sensor", ["OS64", "V32C", "L40"])
def test_wide_oracle_equals_the_field_oracle_up_to_64_rings(synth, sensor):
    ns = WR.n_rings(synth, sensor)
    for k, rev in ((0, False), (3, True)):
        raw = synth.scan_rings(sensor, k, reverse=rev)
        assert_same_features(WR.Features(raw, ns, synth.RING_RANGES[0]), RF.Features(raw, ns, synth.RING_RANGES[0]), (sensor, k))


def test_wide_oracle_refuses_what_the_ring_cannot_bin(synth):
    raw = synth.scan_rings("R2", 0)
    for ns in (0, 129):
        with pytest.raises(RuntimeError):
            WR.Features(raw, ns, 0.3)
    for ns in (65, 96, 128):
        WR.Features(raw, ns, 0.3)


INVALID = (128.0, 127.5, -1.0, np.nan, np.inf, -np.inf, None)   # None: n_scans


@pytest.mark.parametrize("sensor,reverse", [("E65", False), ("L96", True), ("OS128", False), ("OS128", True)])
def test_ring_assignment_and_sweep_walk_on_wide_tables(synth, sensor, reverse):
    """the model of test_oracle_ring_field.py: invalid ring values drop the return before the walk, -0.0 is ring 0"""
    raw = synth.scan_rings(sensor, 1, reverse=reverse)
    ns = WR.n_rings(synth, sensor)
    mr = synth.RING_RANGES[0]
    _, _, _, idx, flip = _model(raw, ns, mr)
    assert flip > 0
    rng = np.random.default_rng(ns)
    bad = rng.choice(idx, size=len(idx) // 20, replace=False)
    at = np.searchsorted(idx, flip)
    bad = np.unique(np.concatenate([bad, [idx[0]], idx[at - 2: at + 6]]))
    vals = np.array([ns if v is None else v for v in INVALID], F32)
    raw[bad, 3] = vals[np.arange(len(bad)) % len(vals)]
    zero = rng.choice(np.setdiff1d(idx, bad), size=50, replace=False)
    raw[zero, 3] = F32(-0.0)
    kept, rings, rel, _, moved = _model(raw, ns, mr)
    assert len(kept) == len(idx) - len(bad) and moved > flip and rings.max() >= 64
    f = WR.Features(raw, ns, mr)
    assert np.array_equal(f.full[:, :3].view(np.uint32), raw[kept, :3].view(np.uint32))
    got_ring = np.floor(f.full[:, 3].astype(np.float64) + 1e-3).astype(int)
    assert np.array_equal(got_ring, rings)
    # intensity = ring + 0.1 relTime in float: above ring 64 the fraction's quantum is 2^-17
    assert np.abs(f.full[:, 3].astype(np.float64) - (rings + 0.1 * rel)).max() < 2e-5
    counts = np.bincount(rings, minlength=ns)
    assert np.array_equal(f.scan_start, np.cumsum(counts) - counts + 5) and np.array_equal(f.scan_end, np.cumsum(counts) - 6)


# ------------------------------------------------------------------------------------------------ 2. the reference's odometry
@pytest.mark.parametrize("sensor,reverse", [("OS128", False), ("V128", False), ("L96", True)])
def test_laser_odometry_source_on_wide_tables(orc, synth, sensor, reverse):
    """the reference's laserOdometry.cpp, compiled unmodified, fed the wide oracle's clouds of four scans, gives the poses and
    correspondence counts of the oracle's odometry bit for bit"""
    from refsource import RefOdometry, private_copy
    ref = RefOdometry(private_copy("libref_odometry.so", "wide_%s_%d" % (sensor, reverse)))
    ns = WR.n_rings(synth, sensor)
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    moved, corr = 0.0, 0
    for k in range(4):
        f = WR.Features(synth.scan_rings(sensor, k, reverse=reverse), ns, synth.RING_RANGES[0], orc.SORT_LITERAL)
        assert int(f.full[:, 3].max()) == ns - 1
        got = ref.process(f, stamp=0.1 * (k + 1))
        if k > 0:
            q, t, info = od.register(f.sharp, f.flat, q, t)
            qw, tw = orc.integrate_pose(qw, tw, q, t)
            assert got["counts"].tolist() == [info["corner_corr"], info["plane_corr"]], (k, got["counts"], info)
            moved = max(moved, float(np.abs(t).max()))
            corr = min(corr or 10 ** 9, info["corner_corr"] + info["plane_corr"])
        od.set_last(f.less_sharp, f.less_flat)
        assert np.array_equal(got["q"], q) and np.array_equal(got["t"], t), (k, got["q"] - q, got["t"] - t)
        assert np.array_equal(got["qw"], qw) and np.array_equal(got["tw"], tw), k
    assert moved > 0.05 and corr > 100


# ------------------------------------------------------------------------------------------------ 3. synthetic wide sensors
def test_wide_ring_sensor_tables(synth):
    assert [len(synth.WIDE_RING_SENSORS[s][0]) for s in ("OS128", "V128", "L96", "E65")] == [128, 128, 96, 65]
    assert not set(synth.WIDE_RING_SENSORS) & set(synth.RING_SENSORS)
    for s, (el, _) in synth.WIDE_RING_SENSORS.items():
        d = np.diff(el)
        assert (d > 0).all() or (d < 0).all(), s   # ring ids in elevation order
    os128 = synth.WIDE_RING_SENSORS["OS128"]
    assert os128[1] == 1024 and os128[0][0] == 22.5 and abs(os128[0][-1] + 22.5) < 1e-12
    v = np.array(synth.WIDE_RING_SENSORS["V128"][0])
    assert v[0] == -25.0 and abs(v[-1] - 15.0) < 1e-12
    step = np.diff(v)
    assert step[np.abs(v[:-1]) < 4].max() < step[np.abs(v[:-1]) > 6].min()   # dense at the horizon


@pytest.mark.parametrize("sensor", ["OS128", "V128", "L96", "E65"])
def test_scan_rings_writes_the_laser_ring_of_wide_tables(synth, sensor):
    el = np.array(synth.WIDE_RING_SENSORS[sensor][0])
    raw = synth.scan_rings(sensor, 0)
    rev = synth.scan_rings(sensor, 0, reverse=True)
    assert np.array_equal(raw[:, :3], rev[:, :3]) and np.array_equal(rev[:, 3], len(el) - 1 - raw[:, 3])
    r = raw[:, 3].astype(int)
    assert np.array_equal(r, raw[:, 3]) and r.min() >= 0 and r.max() < len(el) and len(np.unique(r)) > 0.9 * len(el)
    elev = np.degrees(np.arctan2(raw[:, 2].astype(np.float64), np.hypot(raw[:, 0], raw[:, 1])))
    assert np.abs(elev - el[r]).max() < 0.05


# ------------------------------------------------------------------------------------------------ 4. configuration, snapshots
def _code(aloam, wide=True, **kw):
    kw.setdefault("max_points", 4096)
    try:
        ctx = aloam.Aloam(wide=wide, **kw)
    except aloam.AloamError as e:
        return e.code
    ctx.close()
    return 0


def test_create_wide_is_checked_before_the_device(aloam):
    assert aloam.MAX_RINGS == 128 and "aloam_create_wide" in aloam.EXPORTED_SYMBOLS
    F = aloam.RING_FIELD
    for ns in (1, 40, 64, 65, 96, 128):   # accepted: a context, or no device on a machine without one
        assert _code(aloam, n_scans=ns, ring_source=F) in (0, -6), ns
    for ns in (16, 32, 64):
        assert _code(aloam, n_scans=ns) in (0, -6), ns
    assert _code(aloam, n_scans=0, ring_source=F) == -2 and _code(aloam, n_scans=129, ring_source=F) == -2
    assert _code(aloam, n_scans=40) == -2 and _code(aloam, n_scans=128) == -2   # elevation rings stay 16 / 32 / 64
    assert _code(aloam, n_scans=16, ring_source=2) == -1 and _code(aloam, n_scans=128, ring_source=2) == -1
    # the packed index of a 128-wide association index has 24 bits, and index 2^24 - 1 on ring 127 would pack to INT_MAX (the
    # search's "no candidate"); at 64 rings index 2^25 - 1 on ring 63 would, and from 2^25 on the word turns negative
    for mp in ((1 << 24) + 1, 1 << 24):
        assert _code(aloam, n_scans=128, ring_source=F, max_points=mp) == -1
        assert _code(aloam, n_scans=65, ring_source=F, max_points=mp) == -1
    for mp in (1 << 25, (1 << 25) + 1, 1 << 30):
        for ns, kw in ((64, {}), (16, {}), (64, dict(ring_source=F)), (40, dict(ring_source=F))):
            assert _code(aloam, wide=False, n_scans=ns, max_points=mp, **kw) == -1, (ns, mp)
            assert _code(aloam, n_scans=ns, max_points=mp, **kw) == -1, (ns, mp)
    # aloam_create is unchanged
    assert _code(aloam, wide=False, n_scans=65, ring_source=F) == -2 and _code(aloam, wide=False, n_scans=128, ring_source=F) == -2
    msg = aloam.lib().aloam_strerror(-2).decode()
    assert "1..64" in msg and "aloam_create_wide" in msg


def test_snapshot_check_accepts_a_128_ring_header(aloam):
    h = bytearray(_header(1))
    struct.pack_into("<i", h, 36, 128)
    info = aloam.snapshot_info(bytes(h))
    assert info["n_scans"] == 128 and info["bytes"] == 256


def test_os128_scans_hold_short_rings_that_need_the_pass_through(synth):
    """the OS128 scans of the wide GPU tests are compared whole: their highest beams hold rings of 17..39 returns, on which
    passing on only a segment's own marks gives other picks than the oracle (scan 2 is the one of the feature tests)"""
    import short_ring_cases as SC
    short, miss = [], []
    for index in range(5):
        raw = WR.scan(synth, "OS128", index)
        n = np.bincount(raw[:, 3].astype(np.int64), minlength=128)
        short.append(bool(((n >= 17) & (n < 40)).any()))
        miss.append(bool(SC.adjacent_misses(WR.Features(raw, 128, synth.RING_RANGES[0]), 128)))
    assert short[2] and miss[2] and sum(miss) >= 2, (short, miss)


def test_only_the_os128_table_has_short_rings(synth):
    """of the four wide tables only OS128's highest beams see little within range: V128, L96 and E65 hold over 500 returns on
    every ring of every scan of the wide tests, so their whole scans have no ring of 17..39 returns"""
    for sensor in ("V128", "L96", "E65"):
        for index in range(6):
            n = np.bincount(WR.scan(synth, sensor, index)[:, 3].astype(np.int64), minlength=WR.n_rings(synth, sensor))
            assert n.min() > 500, (sensor, index)


def test_recovery_model_reseats_from_every_corner_on_whole_os128_scans(aloam, synth):
    """the host model of recovery (tests/recovery_cases.py) on the oracle's map of whole OS128 scans: a localising lane armed 1.5 m
    off in x and y adopts a candidate on its START row from each of the four corners, stays within 0.1 m from the next row on and
    ends within 1 cm; the GPU test holds the device to the model's candidate and score from (+1.5, -1.5)"""
    for off in ((1.5, -1.5), (1.5, 1.5), (-1.5, 1.5), (-1.5, -1.5)):
        poses, rows = WR.recovery_model(aloam, synth, off)
        assert rows[0]["triggered"] and rows[0]["adopted"], off
        assert not any(r["triggered"] for r in rows[1:]), off
        err = [float(np.abs(r["pose"][4:] - poses[2 + j][4:]).max()) for j, r in enumerate(rows)]
        assert max(err[1:]) < 0.1 and err[-1] < 0.01, (off, err)
