"""CPU: the model of a growth-on lane store (tests/growth_edge_cases.py) against cube_edge_cases.Model and the allocator model of
test_oracle_cube_growth, its scenarios' tight pools and negative controls, the snapshots they restore, and its mutations: every
mis-transcription of the allocator changes the predicted outcome of at least one GPU scenario."""
import numpy as np
import pytest

import cube_edge_cases as E
import growth_edge_cases as G
from test_oracle_cube_growth import MAX_CUBE, POOL, Pool, pack

EMPTY = G.EMPTY


@pytest.mark.parametrize("growth", [0, 1])
def test_growth_off_and_on_reproduce_the_ring_buffer_model(growth):
    """on cube_edge_cases' jump paths (a few points per cube, far from any limit) the model holds E.Model's cubes, point for
    point, with either setting, and every held cube owns a one-slab run"""
    for name, frames in E.jump_paths().items():
        ref, _ = E.run_model(frames)
        m = G.Model((16384, 20000), growth, strict=False)
        for q, t, surf in frames:
            _, flag = m.frame(EMPTY, surf, q, t)
            assert not flag, name
        assert m.held() == ref.held(), name
        for k in ref.held():
            assert np.array_equal(m.cube(*k), ref.cube(*k)), (name, k)
            assert m.runs[k][1] == 0
        assert int(m.pools[1].used.sum()) == len(m.held()), name


@pytest.mark.parametrize("growth", [0, 1])
@pytest.mark.parametrize("jump,fill_k", [(40, (4, 5, 6)), (12, (5,)), (-40, (4, 5, 6)), (-12, (5,))])
def test_slab_pool_after_wraps_with_either_setting(growth, jump, fill_k):
    """test_gpu_cube_edges.test_slab_pool_after_wraps in the model, one point per cube: the wrapped cubes' slabs are back in the
    pool, exactly 1024 cubes are stored and the frame is flagged, with growth off and on alike"""
    rng = np.random.default_rng(abs(jump) + (jump < 0))

    def grid(cen, t, kk):
        ii, jj, ks = np.meshgrid(np.arange(E.CW), np.arange(E.CH), np.asarray(kk), indexing="ij")
        out = np.zeros((ii.size, 4), np.float32)
        for a, idx in enumerate((ii, jj, ks)):
            out[:, a] = (idx.ravel() - cen[a]) * 50.0 + rng.uniform(-10, 10, ii.size) - t[a]
        return out[rng.permutation(ii.size)]

    m = G.Model((3000, 3000), growth, strict=False)
    far = np.array([50.0 * jump, 0.0, 0.0])
    m.frame(EMPTY, grid(E.CEN0, np.zeros(3), fill_k), G.IDENT, np.zeros(3))
    m.frame(EMPTY, EMPTY, G.IDENT, far)
    kept = len(m.held())
    _, flag = m.frame(EMPTY, grid(m.cen, far, (4, 5, 6)), G.IDENT, far)
    assert kept == (0 if abs(jump) == 40 else 16 * E.CH)
    assert flag and len(m.held()) == 1024 and int(m.pools[1].used.sum()) == 1024


def test_the_allocator_agrees_with_pool_and_pack():
    """the model's take is Pool.take on random sequences of takes and frees; random stores restore to pack()'s runs; after random frames every held run is aligned, runs never overlap and the bitmap
    is exactly their union (nothing leaks, nothing is handed out twice), with growth on"""
    rng = np.random.default_rng(0)
    a, b, held = Pool(), G._Pool(), []
    for _ in range(3000):
        if held and rng.random() < 0.4:
            r = held.pop(int(rng.integers(len(held))))
            a.free(*r); b.free(*r)
        else:
            o = int(rng.choice(11, p=[0.4, 0.2, 0.1, 0.1, 0.05, 0.05, 0.04, 0.03, 0.02, 0.005, 0.005]))
            s = a.take(o)
            assert b.take(o) == s
            if s >= 0:
                held.append((s, o))
        assert np.array_equal(a.used, b.used)
    cap = 1024
    for trial in range(6):
        s = G.Store()
        budget = POOL - 200
        for ijk in [G.FILL[k] for k in rng.permutation(len(G.FILL))[:120]]:
            n = int(rng.choice([1, cap, cap + 1, 3 * cap, 8 * cap]))
            if s.slabs(1, cap) + (1 << G.run_order(n, cap)) > budget:
                continue
            s.put(1, ijk, G.at(ijk, rng, n))
        m = G.Model((cap, cap), 1, strict=False)
        m.restore(s.counts, s.pts, 1)
        runs, used = pack(s.counts[1], cap)
        assert {i: r for (ty, i), r in m.runs.items()} == runs and int(m.pools[1].used.sum()) == used
        for f in range(4):
            t = (G.JUMP * (f % 2), 0.0, 0.0)
            cubes = [G.FILL[k] for k in rng.permutation(len(G.FILL))[:40]] + [G.NEW[k] for k in rng.permutation(200)[:40]]
            surf = np.concatenate([G.at(c, rng, int(rng.integers(1, 40))) for c in cubes])
            m.frame(EMPTY, surf[rng.permutation(len(surf))] - np.array([*t, 0.0], np.float32), G.IDENT, np.array(t))
            bitmap = np.zeros(POOL, bool)
            for (ty, i), (s0, o) in m.runs.items():
                assert s0 % (1 << o) == 0 and not bitmap[s0:s0 + (1 << o)].any()
                assert m.count(ty, i) <= cap << o
                bitmap[s0:s0 + (1 << o)] = True
            assert np.array_equal(bitmap, m.pools[1].used), (trial, f)


def test_passes_through_is_the_leaf_too_small_exit():
    """PCL gives up when (extent / leaf + 1) cubed passes INT_MAX: from about 0.129 m per axis at 1e-4 m"""
    p = np.zeros((2, 4), np.float32)
    p[1, :3] = 0.128
    assert not G.passes_through(p)              # 1281^3 cells: the filter sorts
    p[1, :3] = 0.13
    assert G.passes_through(p)                  # 1301^3
    p[1, 2] = 0.0
    assert not G.passes_through(p)              # flat on one axis
    assert G.passes_through(p[:1])
    p[1, :3] = 1000.0
    with pytest.raises(AssertionError):
        G.passes_through(p)                     # 10^7 cells per axis: the 64-bit product wraps


def _flags(sc, mut=None):
    return [o[0] for o in G.outcome(sc, mut)]


def test_scenarios_are_tight_and_their_negative_controls_flag():
    """each scenario's flags as its docstring says, and each negative control (one more one-slab cube) flags a frame where the
    scenario does not"""
    S = G.scenarios()
    want = {"wrap_single_word": [False, False, True], "one_word_low": [False, False], "one_word_high": [False, False],
            "multi_word": [False, False], "whole_pool": [True, True, False, False, False, False, False, False],
            "competing_on": [True, True], "competing_off": [False, False, True, True], "deferred": [True, False],
            "retry": [True, False, False], "unaligned_holes": [False, True, False], "two_orders": [False, False],
            "restart_on": [False, False, True], "restart_off": [False, False, True], "restart_on_fresh": [False, True],
            "restart_off_fresh": [False, True]}
    for name, flags in want.items():
        assert _flags(S[name]) == flags, name
    for name, sc in S.items():
        if name.endswith("_extra"):
            base = _flags(S[name[:-len("_extra")]])
            extra = _flags(sc)
            if name.startswith("competing"):   # B gets no point where it won
                B = (1, E.cube_index(6, 0, 0))
                b, e = dict(G.outcome(S[name[:-len("_extra")]])[-2][1]), dict(G.outcome(sc)[-2][1])
                assert b[B] == (1025 if sc.growth else 1) and e.get(B, 0) == (1024 if sc.growth else 0), name
            else:
                extra = extra[len(extra) - len(base):]   # (a control whose first frame opens the extra cube)
                assert any(e and not b for e, b in zip(extra, base)), name
    # the continuations of both restarts are the fresh contexts' runs
    for g in ("on", "off"):
        a, b = G.outcome(S["restart_" + g]), G.outcome(S["restart_%s_fresh" % g])
        assert a[-2:] == b


def test_whole_pool_growth_stops_at_half_the_pool():
    """max_points = 256: a full 512-slab cube cannot take its 1024-slab run in an insert (its old run is held while the new one is
    taken), so it stops at 131072 points; restored, a cube holds all 2^18"""
    S = G.scenarios()
    counts = [m.count(1, E.cube_index(5, 0, 0)) for step, m, _, _ in G.walk(S["whole_pool"]) if step[0] == "frame"][:1]
    assert counts == [512 * 256]
    assert G.max_order(256) == 10 and (256 << 10) == MAX_CUBE


def test_every_mutation_changes_a_scenario():
    S = G.scenarios()
    base = {name: G.outcome(sc) for name, sc in S.items()}
    for mut in G.MUTATIONS:
        caught = [name for name, sc in S.items() if G.outcome(sc, mut) != base[name]]
        assert caught, mut


def test_scenario_snapshots_pass_the_checks(aloam):
    """every restored store is a well-formed growth-on snapshot of its context's configuration; the whole-pool cube and the
    multi-word runs are refused with growth off in the header"""
    import ctypes as C
    for name, sc in G.scenarios().items():
        cfg = G.config(sc.max_points)
        for step in sc.steps:
            if step[0] != "restore":
                continue
            for growth in (1, 0):
                b = G.snapshot(cfg, step[1], growth)
                code = aloam.lib().aloam_snapshot_check(C.c_void_p(b.ctypes.data), len(b), None)
                one_slab = (step[1].counts[1] <= min(65536, sc.max_points)).all() and (step[1].counts[0] <= min(16384, sc.max_points)).all()
                assert code == (0 if growth or one_slab else aloam.ERR_SNAPSHOT), (name, growth)
