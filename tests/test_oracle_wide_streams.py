"""CPU: the scenes of tests/wide_stream_cases.py do what tests/test_gpu_wide_streams.py relies on.  On the wide oracle
(tests/wide_ring_oracle.py) every ring a full-cap scene holds yields exactly its caps and every other ring nothing, so the fused
slots are occupied up to sharp slot 1535 and flat slot 3071; the oracle's odometry chains give every query slot a
correspondence; high-ring scenes occupy only the end of the per-ring tables; lanes of the distinct batch differ; and the seam
scans carry ratios s outside [0, 1]."""
import numpy as np
import pytest

import wide_stream_cases as S

FRAMES = 5


@pytest.mark.parametrize("name", sorted(S.SCENES))
def test_every_held_ring_yields_its_caps(name):
    ns, rings, _ = S.SCENES[name]
    empty = [r for r in range(ns) if r not in rings]
    for k in range(FRAMES):
        f = S.features(S.scene_scan(name, k), ns)
        for kind, cap in S.CAPS.items():
            n = S.per_ring(getattr(f, kind), ns)
            assert (n[list(rings)] == cap).all() and not n[empty].any(), (name, k, kind)
        assert S.per_ring(f.less_flat, ns)[list(rings)].min() > 0 and not S.per_ring(f.less_flat, ns)[empty].any()
        # the ring-major staging rows k_compact reads: ring r's sharp points sit in rows r * 12 .. r * 12 + 11
        assert len(f.sharp) == S.CAPS["sharp"] * len(rings) and len(f.flat) == S.CAPS["flat"] * len(rings)
        assert ns > 64 and len(f.sharp) <= S.SHARP_SLOTS and len(f.flat) <= S.FLAT_SLOTS


def test_full_128_ring_scans_fill_every_fused_slot():
    f = S.features(S.scene_scan("full128"), 128)
    assert len(f.sharp) == S.SHARP_SLOTS == 1536 and len(f.flat) == S.FLAT_SLOTS == 3072
    assert len(f.less_sharp) == 128 * 120
    # slots 1535 and 3071 hold ring 127's last picks
    assert int(f.sharp[1535, 3]) == 127 and int(f.flat[3071, 3]) == 127
    for name, ns in (("full96", 96), ("full65", 65)):   # the 128-wide slot table partly empty
        g = S.features(S.scene_scan(name), ns)
        assert len(g.sharp) == 12 * ns < S.SHARP_SLOTS and len(g.flat) == 24 * ns < S.FLAT_SLOTS


@pytest.mark.parametrize("name,distortion,nearby", [("full128", False, 2.5), ("full128", True, np.inf), ("full96", False, np.inf),
                                                    ("full65", True, 2.5), ("high64", False, 2.5), ("ends", True, np.inf)])
def test_oracle_chains_reach_the_last_query_slots(orc, name, distortion, nearby):
    """every sharp and flat query of every frame has a correspondence in the oracle's chain (so the last fused slots, 1535 and 3071
    at 128 rings, take part in the solve); the chain moves"""
    ns, rings, _ = S.SCENES[name]
    raws = [S.scene_scan(name, k) for k in range(FRAMES)]
    poses, counts, feats = S.oracle_chain(orc, raws, ns, distortion, nearby)
    for k in range(1, FRAMES):
        assert counts[k] == (12 * len(rings), 24 * len(rings)), (k, counts[k])
    od = orc.Odometry(distortion=distortion, nearby_scan=nearby)
    od.set_last(feats[0].less_sharp, feats[0].less_flat)
    cc, pc, _ = od.associate(feats[1].sharp, feats[1].flat, np.array([0, 0, 0, 1.0]), np.zeros(3))
    assert int(cc[:, 0].max()) == len(feats[1].sharp) - 1 and int(pc[:, 0].max()) == len(feats[1].flat) - 1
    if name == "full128":
        assert int(cc[:, 0].max()) == 1535 and int(pc[:, 0].max()) == 3071
    assert np.abs(poses[-1, 4:6]).min() > 0.05


@pytest.mark.parametrize("name", ["ring127", "ends"])
def test_scenes_without_neighbour_rings_within_reach_find_nothing(orc, name):
    """ring 127 alone, and rings 0 and 127 at nearby_scan 2.5: no 2nd point on another ring, no correspondence, the identity"""
    ns, _, _ = S.SCENES[name]
    poses, counts, _ = S.oracle_chain(orc, [S.scene_scan(name, k) for k in range(3)], ns)
    assert counts[1:] == [(0, 0), (0, 0)] and np.array_equal(poses[-1], [0, 0, 0, 1, 0, 0, 0])


def test_distinct_lanes_hold_distinct_bands():
    seen = set()
    for j in range(16):
        rings = S.band_rings(j)
        assert len(rings) == 16 and max(rings) <= 127
        f = S.features(S.band_scan(j, 1), 128)
        n = S.per_ring(f.sharp, 128)
        assert np.flatnonzero(n).tolist() == list(rings) and (n[list(rings)] == 12).all()
        key = f.sharp[:, :3].tobytes()
        assert key not in seen
        seen.add(key)
    assert max(S.band_rings(15)) >= 120 and {63, 64} <= set(S.band_rings(9)) and min(S.band_rings(10)) >= 64   # lane 9 straddles 63 / 64


def test_seam_scans_have_ratios_outside_0_1(synth):
    for k in range(2):
        f = S.features(S.seam_scan(synth, k), 128)
        s = S.ratios(f.full)
        assert s.min() < 0.0 and s.max() > 1.0, (k, s.min(), s.max())
        assert int(np.round(f.full[:, 3] - 0.05).max()) >= 120
