"""CPU: mapping_skip_frame.  The reference's three nodes, compiled from their own sources (tests/refsource.py; the sequence
and odometry-only drivers of oracle/ref_skip.mk), chained on their published topics with mapping_skip_frame = 2 and 3, pin the skip-aware oracle chain (tests/skip_refs.py) that the GPU tests
compare against: laserOdometry sends scan j to the mapper exactly when j % k == 0 (one entry of its main() runs the whole
sequence, so its loop-local frameCount counts the scans); a mapped scan's /aft_mapped_to_init is the oracle's CubeMap.step, and
every other scan's /aft_mapped_to_init_high_frec is the oracle's transform_associate_to_map with the T_wmap_wodom of the latest
mapped scan.  Also the config field of the C ABI and its Python mirror."""
import ctypes as C

import numpy as np
import pytest

import skip_refs as S
from refsource import RefMapping, ref_registration

N_SCANS = 12


@pytest.mark.parametrize("skip", [2, 3])
def test_the_three_reference_nodes_with_mapping_skip_frame_equal_the_oracle_chain(orc, synth, skip):
    ns, _, mr = synth.SENSORS["VLP-16"][:3]
    scans = [synth.scan("VLP-16", k, n_az=900) for k in range(N_SCANS)]
    reg = ref_registration(ns, mr)
    odo = S.RefOdometrySequence(S.skip_driver("libref_odometry_seq.so", "skip%d" % skip), skip)
    for j, raw in enumerate(scans):
        odo.queue(reg.run(raw, orc.SORT_LITERAL), stamp=0.1 * (j + 1))
    turns = odo.run()
    # the odometry node published clouds for exactly the scans j % k == 0
    assert [t["clouds"] is not None for t in turns] == [S.mapped(j, skip) for j in range(N_SCANS)]
    mp = RefMapping(S.skip_driver("libref_mapping_skip.so", "skip%d" % skip), 0.2, 0.4, orc.SORT_LITERAL)
    got = []
    n_high = 0
    for j, t in enumerate(turns):
        stamp = 0.1 * (j + 1)
        if t["clouds"] is not None:
            corner, surf, full = t["clouds"]
            m = mp.process(corner, surf, full, t["pose"][:4], t["pose"][4:], stamp)
            got.append(m["pub"])                                   # /aft_mapped_to_init
            n_high += 1                                            # its odometry message also went through the handler
        else:
            pose, n = S.ref_map_odometry_only(mp, t["pose"][:4], t["pose"][4:], stamp)
            n_high += 1
            assert n == n_high, (j, n, n_high)
            got.append(pose)                                       # /aft_mapped_to_init_high_frec
    odom, want = S.oracle_chain(orc, synth, scans, skip, ("VLP-16", "base", 900), sort_mode=orc.SORT_LITERAL, leaves=(0.2, 0.4))
    for j, t in enumerate(turns):
        assert np.array_equal(t["pose"], odom[j]), ("/laser_odom_to_init", j, t["pose"] - odom[j])
        if t["clouds"] is not None:   # the clouds laserMapping receives are the scan's less-sharp / less-flat clouds, unchanged
            f = orc.Features(scans[j], ns, mr, mode=orc.SORT_LITERAL)
            assert np.array_equal(t["clouds"][0], f.less_sharp) and np.array_equal(t["clouds"][1], f.less_flat), j
        assert np.array_equal(got[j], want[j]), ("mapped" if S.mapped(j, skip) else "high-frequency", j, got[j] - want[j])
    # not a comparison of identities: the mapper moved T_wmap_wodom away from the identity before some skipped scan
    skipped = [j for j in range(N_SCANS) if not S.mapped(j, skip)]
    assert max(float(np.abs(want[j] - odom[j]).max()) for j in skipped) > 0


def test_config_field_and_default(aloam):
    names = [f[0] for f in aloam.Config._fields_]
    assert names[-1] == "mapping_skip_frame"
    for n in (16, 32, 64):
        assert aloam.default_config(n).mapping_skip_frame == 1   # launch/aloam_velodyne_*.launch:6


def test_negative_skip_is_refused_before_any_device_work(aloam):
    cfg = aloam.default_config(16)
    cfg.mapping_skip_frame = -1
    h = C.c_void_p()
    assert aloam.lib().aloam_create(C.byref(cfg), C.byref(h)) == -1 and not h.value
