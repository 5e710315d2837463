"""CPU: rings from the sensor driver (aloam_config.ring_source = ALOAM_RING_FIELD) -- the oracle's field mode against its
elevation mode and a model of ring assignment and the sweep walk, the reference's own laserOdometry.cpp on other beam tables,
the PointCloud2 ring unpacker, the snapshot header field and the configuration checks that run before any device is used."""
import math
import struct

import numpy as np
import pytest

import ring_edge_cases as E
import ring_field_oracle as RF

F32 = np.float32
NAMES = ("full", "sharp", "less_sharp", "flat", "less_flat")


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32) if a.dtype == F32 else a, b.view(np.uint32) if b.dtype == F32 else b)


def assert_same_features(got, want, tag):
    for n in NAMES + ("scan_start", "scan_end", "label"):
        assert _same(getattr(got, n), getattr(want, n)), (tag, n)


# ------------------------------------------------------------------------------------------------ 1. field mode == elevation mode
def test_field_mode_with_the_formula_ring_equals_elevation_mode(orc, synth):
    """w = the formula's ring (-1 where it drops the return): the full cloud, the four feature clouds, scan_start / scan_end
    and the labels are bit-identical, on the three sensors, seam scans and scans on every ring edge; stride 8 too"""
    n = 0
    for tag, raw, ns, mr in RF.elevation_cases(synth):
        want = orc.Features(raw, ns, mr)
        wr = RF.formula_rings(raw, ns)
        assert_same_features(RF.Features(wr, ns, mr), want, tag)
        if n % 3 == 0:
            wide = np.concatenate([wr, np.full((len(wr), 4), np.nan, F32)], axis=1)
            assert_same_features(RF.Features(wide, ns, mr), want, tag + "/stride8")
        n += 1
    assert n == 12


def test_field_mode_with_the_literal_sort_equals_elevation_mode(orc, synth):
    raw = synth.scan("VLP-16", 2, n_az=900)
    assert_same_features(RF.Features(RF.formula_rings(raw, 16), 16, 0.3, orc.SORT_LITERAL), orc.Features(raw, 16, 0.3, orc.SORT_LITERAL), "literal")


def test_field_source_edits_only_the_ring_decision():
    src = RF.field_source()
    assert src.count("ring_field(p.w, n_scans)") == 1 and "ring_of(angle, n_scans)" not in src


def test_field_mode_refuses_what_the_ring_cannot_bin(orc, synth):
    raw = synth.scan_rings("R2", 0)
    for ns in (0, 65):
        with pytest.raises(RuntimeError):
            RF.Features(raw, ns, 0.3)
    with pytest.raises(ValueError):
        RF.Features(raw[:, :3], 2, 0.3)
    for ns in (1, 2, 7, 40, 48, 64):   # any count 1..64
        RF.Features(np.where(np.arange(4)[None, :] == 3, 0, raw).astype(F32), ns, 0.3)


# ------------------------------------------------------------------------------------------------ 2. invalid ring values
INVALID = (np.nan, np.inf, -np.inf, -1.0, None, 2.5, 1e9)   # None: n_scans


def _model(raw, n_scans, min_range):
    """the returns field mode keeps, in ring-major order, with their ring and relTime: NaN / range filter, ring = w when it is
    an integer in 0 .. n_scans - 1, and the sweep walk of scanRegistration.cpp:141-236 over the kept returns only"""
    x, y, z, w = (raw[:, k].astype(F32) for k in range(4))
    thres = F32(min_range)
    with np.errstate(invalid="ignore", over="ignore"):
        ok = np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & ~(x * x + y * y + z * z < thres * thres)
        valid = (w >= 0) & (w < n_scans) & (w == np.trunc(w))
    idx = np.flatnonzero(ok)
    ori_all = -np.arctan2(y, x).astype(F32)
    start = ori_all[idx[0]]
    end = F32(float(ori_all[idx[-1]]) + 2 * math.pi)
    if float(end) - float(start) > 3 * math.pi:
        end = F32(float(end) - 2 * math.pi)
    elif float(end) - float(start) < math.pi:
        end = F32(float(end) + 2 * math.pi)
    half, flip = False, -1
    kept, rings, rel = [], [], []
    for i in idx:
        if not valid[i]:
            continue   # `continue` before the walk: a dropped return does not flip halfPassed
        ori = ori_all[i]
        if not half:
            if float(ori) < float(start) - math.pi / 2:
                ori = F32(float(ori) + 2 * math.pi)
            elif float(ori) > float(start) + math.pi * 3 / 2:
                ori = F32(float(ori) - 2 * math.pi)
            if float(F32(ori - start)) > math.pi:
                half, flip = True, i
        else:
            ori = F32(float(ori) + 2 * math.pi)
            if float(ori) < float(end) - math.pi * 3 / 2:
                ori = F32(float(ori) + 2 * math.pi)
            elif float(ori) > float(end) + math.pi / 2:
                ori = F32(float(ori) - 2 * math.pi)
        kept.append(i); rings.append(int(w[i])); rel.append(float(F32(ori - start) / F32(end - start)))
    kept, rings, rel = np.array(kept), np.array(rings), np.array(rel)
    order = np.lexsort((kept, rings))
    return kept[order], rings[order], rel[order], idx, flip


@pytest.mark.parametrize("sensor,reverse", [("V32C", False), ("OS64", True), ("L40", False)])
def test_invalid_ring_values_drop_the_return_and_skip_the_walk(synth, sensor, reverse):
    raw = synth.scan_rings(sensor, 1, reverse=reverse)
    ns = len(synth.RING_SENSORS[sensor][0])
    mr = synth.RING_RANGES[0]
    _, _, _, idx, flip = _model(raw, ns, mr)
    assert flip > 0
    rng = np.random.default_rng(ns)
    bad = rng.choice(idx, size=len(idx) // 20, replace=False)
    # the first kept return (it still sets start_ori), and a run across the return that flips halfPassed
    at = np.searchsorted(idx, flip)
    run = idx[at - 2: at + 6]
    bad = np.unique(np.concatenate([bad, [idx[0]], run]))
    vals = np.array([ns if v is None else v for v in INVALID], F32)
    raw[bad, 3] = vals[np.arange(len(bad)) % len(vals)]
    zero = rng.choice(np.setdiff1d(idx, bad), size=50, replace=False)
    raw[zero, 3] = F32(-0.0)   # -0.0 is ring 0
    kept, rings, rel, _, moved = _model(raw, ns, mr)
    assert len(kept) == len(idx) - len(bad) and moved > flip
    f = RF.Features(raw, ns, mr)
    assert np.array_equal(f.full[:, :3].view(np.uint32), raw[kept, :3].view(np.uint32))
    got_ring = np.floor(f.full[:, 3].astype(np.float64) + 1e-3).astype(int)   # relTime < 1 everywhere in these sweeps
    assert np.array_equal(got_ring, rings)
    assert np.abs(f.full[:, 3].astype(np.float64) - (rings + 0.1 * rel)).max() < 1e-5
    counts = np.bincount(rings, minlength=ns)
    assert np.array_equal(f.scan_start, np.cumsum(counts) - counts + 5) and np.array_equal(f.scan_end, np.cumsum(counts) - 6)


# ------------------------------------------------------------------------------------------------ 3. the reference's odometry
@pytest.mark.parametrize("sensor,reverse", [("OS64", False), ("V32C", False), ("V32C", True)])
def test_laser_odometry_source_on_other_beam_tables(orc, synth, sensor, reverse):
    """the reference's laserOdometry.cpp, compiled unmodified, fed the field-mode clouds of an OS64 / V32C trajectory, gives
    the poses and correspondence counts of the oracle's odometry bit for bit (the node never reads N_SCANS)"""
    from refsource import RefOdometry, private_copy
    ref = RefOdometry(private_copy("libref_odometry.so", "ring_%s_%d" % (sensor, reverse)))
    ns = len(synth.RING_SENSORS[sensor][0])
    od = orc.Odometry()
    q = np.array([0, 0, 0, 1.0]); t = np.zeros(3); qw = q.copy(); tw = t.copy()
    moved, corr = 0.0, 0
    for k in range(4):
        f = RF.Features(synth.scan_rings(sensor, k, reverse=reverse), ns, synth.RING_RANGES[0], orc.SORT_LITERAL)
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


# ------------------------------------------------------------------------------------------------ synthetic driver-ring sensors
def test_ring_sensor_tables(synth):
    assert [len(synth.RING_SENSORS[s][0]) for s in ("OS64", "V32C", "L40", "R1", "R2")] == [64, 32, 40, 1, 2]
    for s, (el, _) in synth.RING_SENSORS.items():
        d = np.diff(el)
        assert (d > 0).all() or (d < 0).all() or len(el) == 1, s   # ring ids in elevation order
    assert synth.RING_SENSORS["OS64"][0][0] == 16.6 and abs(synth.RING_SENSORS["OS64"][0][-1] + 16.6) < 1e-12


@pytest.mark.parametrize("sensor", ["OS64", "V32C", "R2"])
def test_scan_rings_writes_the_laser_ring(synth, sensor):
    el = np.array(synth.RING_SENSORS[sensor][0])
    raw = synth.scan_rings(sensor, 0)
    rev = synth.scan_rings(sensor, 0, reverse=True)
    assert np.array_equal(raw[:, :3], rev[:, :3]) and np.array_equal(rev[:, 3], len(el) - 1 - raw[:, 3])
    r = raw[:, 3].astype(int)
    assert np.array_equal(r, raw[:, 3]) and r.min() >= 0 and r.max() < len(el)
    elev = np.degrees(np.arctan2(raw[:, 2].astype(np.float64), np.hypot(raw[:, 0], raw[:, 1])))
    assert np.abs(elev - el[r]).max() < 0.05   # each return lies on its laser's cone (noise is along the ray)


def test_formula_bins_these_tables_wrongly(synth):
    """why the driver's ring is needed: the HDL-32 formula merges V32C beams and drops one, the HDL-64 formula drops the OS64
    beams above +2 deg"""
    v = np.array(synth.RING_SENSORS["V32C"][0], F32)
    ids = E.ring_of_angle(v, 32)
    assert len(np.unique(ids[ids >= 0])) < 32 and (ids < 0).sum() == 1
    o = np.array(synth.RING_SENSORS["OS64"][0], F32)
    assert (E.ring_of_angle(o, 64) < 0).sum() >= 28


# ------------------------------------------------------------------------------------------------ 4. PointCloud2 ring field
def _io():
    import importlib
    return importlib.import_module("a-loam_b200.io")


def test_unpack_velodyne_pointxyzir(aloam):
    io = _io()
    rng = np.random.default_rng(3)
    n = 37
    xyz = rng.normal(0, 20, (n, 3)).astype(F32)
    ring = rng.integers(0, 128, n).astype(np.uint16)
    ring[:3] = (0, 63, 65535)
    dt = np.dtype({"names": ["x", "y", "z", "intensity", "ring"], "formats": ["<f4", "<f4", "<f4", "<f4", "<u2"],
                   "offsets": [0, 4, 8, 16, 20], "itemsize": 32})
    rec = np.zeros(n, dt)
    rec["x"], rec["y"], rec["z"], rec["intensity"], rec["ring"] = xyz[:, 0], xyz[:, 1], xyz[:, 2], 7.5, ring
    out = io.unpack_points_ring(rec.view(np.uint8), n, 32, 0, 4, 8, 20, io.RING_UINT16)
    assert np.array_equal(out[:, :3], xyz) and np.array_equal(out[:, 3], ring.astype(F32))


def test_unpack_ouster_style_point(aloam):
    """48-byte point: x y z, intensity@16, t@20, reflectivity@24, ring@26 as uint8 or uint16, ambient@28, range@32"""
    io = _io()
    n = 64
    xyz = np.stack([np.arange(n), -np.arange(n), 0.5 * np.arange(n)], 1).astype(F32)
    buf = bytearray(48 * n)
    for i in range(n):
        struct.pack_into("<3f", buf, 48 * i, *xyz[i])
        struct.pack_into("<fIHHHxxI", buf, 48 * i + 16, 1.0, 123456, 77, 0xFFFF, 9, 5000)
        struct.pack_into("<H", buf, 48 * i + 26, 63 - i)   # ring 0 at the top: 63 .. 0
    d = np.frombuffer(bytes(buf), np.uint8)
    out16 = io.unpack_points_ring(d, n, 48, 0, 4, 8, 26, io.RING_UINT16)
    assert np.array_equal(out16[:, :3], xyz) and np.array_equal(out16[:, 3], (63 - np.arange(n)).astype(F32))
    out8 = io.unpack_points_ring(d, n, 48, 0, 4, 8, 26, io.RING_UINT8)   # the low byte of the same little-endian field
    assert np.array_equal(out8[:, 3], (63 - np.arange(n)).astype(F32))
    assert np.array_equal(io.unpack_points_ring(d, n, 48, 0, 4, 8, 47, io.RING_UINT8)[:, 3], np.zeros(n, F32))   # last byte


def test_unpack_ring_refuses_bad_types_and_offsets(aloam):
    io = _io()
    d = np.zeros(48 * 4, np.uint8)
    for ty in (0, 1, 3, 5, 6, 7, 8, 9):   # INT8, INT16, INT32, UINT32, FLOAT32, FLOAT64, ...
        with pytest.raises(ValueError):
            io.unpack_points_ring(d, 4, 48, 0, 4, 8, 26, ty)
    for args in ((0, 4, 8, 47, io.RING_UINT16), (0, 4, 8, 48, io.RING_UINT8), (0, 4, 8, -1, io.RING_UINT8), (45, 4, 8, 26, io.RING_UINT8),
                 (0, -4, 8, 26, io.RING_UINT8)):
        with pytest.raises(ValueError):
            io.unpack_points_ring(d, 4, 48, *args)
    with pytest.raises(ValueError):
        io.unpack_points_ring(d, 4, 11, 0, 4, 8, 0, io.RING_UINT8)   # point_step below x, y, z
    assert io.unpack_points_ring(d, 0, 48, 0, 4, 8, 26, io.RING_UINT8).shape == (0, 4)


# ------------------------------------------------------------------------------------------------ 5. snapshot header, configuration
def _header(ring_source):
    h = bytearray(256)
    h[0:8] = b"ALOAMLS1"
    struct.pack_into("<iiqiii", h, 8, 1, 0, 256, 1, 0, 0)   # version, mapped, total_bytes, scan_index, n_less_sharp, n_less_flat
    struct.pack_into("<i", h, 36, 40)                        # n_scans
    struct.pack_into("<d", h, 104 + 24, 1.0)                 # warm q_w
    struct.pack_into("<i", h, 216, ring_source)
    return bytes(h)


def test_snapshot_ring_source_field(aloam):
    for rs in (0, 1):
        info = aloam.snapshot_info(_header(rs))
        assert info["n_scans"] == 40 and info["bytes"] == 256
    for rs in (2, -1, 256):
        with pytest.raises(aloam.AloamError) as e:
            aloam.snapshot_info(_header(rs))
        assert e.value.code == aloam.ERR_SNAPSHOT


def test_ring_source_is_checked_before_the_device(aloam):
    def code(**kw):
        try:
            ctx = aloam.Aloam(max_points=4096, **kw)
        except aloam.AloamError as e:
            return e.code
        ctx.close()
        return 0
    assert code(n_scans=16, ring_source=2) == -1 and code(n_scans=16, ring_source=-1) == -1
    assert code(n_scans=0, ring_source=aloam.RING_FIELD) == -2 and code(n_scans=65, ring_source=aloam.RING_FIELD) == -2
    assert code(n_scans=40, ring_source=aloam.RING_ELEVATION) == -2
    for ns in (1, 40, 64):   # accepted: a context, or no device on a machine without one
        assert code(n_scans=ns, ring_source=aloam.RING_FIELD) in (0, -6)
    assert "1..64" in aloam.lib().aloam_strerror(-2).decode()
    cfg = aloam.default_config(40)
    assert (cfg.ring_source, round(cfg.minimum_range, 3), round(cfg.line_res, 3), round(cfg.plane_res, 3)) == (0, 0.3, 0.2, 0.4)
