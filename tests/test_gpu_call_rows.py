"""GPU: what the readers of the last mapped stream call (aloam_registered_rows, aloam_map_rows, aloam_recovery_rows,
aloam_debug_recovery_scores) return after every way a call can end.  One two-lane context on the VLP-16 world of
tests/test_gpu_map_rows.py (lane 0 localises against the prior map, armed off its true pose so that recovery triggers; lane 1 maps)
walks through a table of calls; after each one all four readers are read and compared with the rule of that ending:
  * this    -- the call's own rows: the kinds and sink offsets its schedule implies, recovery only on localising rows, and the
               candidate scores readable for exactly the lanes with a triggered row (none when recovery or recording was off);
  * prev    -- what the readers returned before the call;
  * state   -- ALOAM_ERR_STATE.
Only errors the host detects or the device flags are used: bad ops, a schedule error, a small sink, empty and oversized views, a
scan whose less-sharp stack overflows its voxel key, a scan with every point under minimum_range."""
import numpy as np
import pytest

import recovery_cases as RV
import track_cases as TC
import track_edge_cases as TE
from test_gpu_map_rows import _localiser, _world

pytestmark = pytest.mark.gpu

OK, ERR_INVALID_ARG, ERR_EMPTY_CLOUD, ERR_CAPACITY, ERR_STATE = 0, -1, -3, -4, -9
IDLE, SCAN, START = 0, 1, 2
B = 2   # lanes of the context


def _code(aloam, fn):
    """fn() -> (0, its result), or (the error code, None)"""
    try:
        return OK, fn()
    except aloam.AloamError as e:
        return e.code, None


def _readers(aloam, c, rows):
    """all four readers, each as (code, value), the first three for `rows` rows"""
    return {"reg": _code(aloam, lambda: c.registered_rows(rows)), "map": _code(aloam, lambda: c.map_rows(rows)),
            "rec": _code(aloam, lambda: c.recovery_rows(rows)),
            "dbg": [_code(aloam, lambda l=l: c.debug_recovery_scores(l)) for l in range(B)]}


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    return a == b


class Call:
    """one lanes call: steps[k][l] = (tensor or None, op); mapped: a mapped call; kinds: the ROW_* of every row it would run"""
    def __init__(self, steps, mapped=True, localising=(), counts=None):
        self.steps, self.mapped = steps, mapped
        self.rows = len(steps) * B
        self.counts = counts or {}
        self.kinds = [0 if op == IDLE else (2 if l in localising else 1) for st in steps for l, (_, op) in enumerate(st)]

    def arrays(self):
        ptrs, counts, ops = np.zeros((len(self.steps), B), np.uint64), np.zeros((len(self.steps), B), np.int64), np.zeros((len(self.steps), B), np.int32)
        for k, st in enumerate(self.steps):
            for l, (d, op) in enumerate(st):
                ops[k, l] = op
                if d is not None:
                    ptrs[k, l], counts[k, l] = d.data_ptr(), self.counts.get((k, l), d.shape[0])
        return ptrs, counts, ops

    def begins(self):
        """the sink offset of every row: the points of the mapped rows before it"""
        _, counts, ops = self.arrays()
        n = np.where(ops.reshape(-1) != IDLE, counts.reshape(-1), 0)
        return np.concatenate([[0], np.cumsum(n)[:-1]])

    def __call__(self, c):
        ptrs, counts, ops = self.arrays()
        return c.scan_stream_lanes(ptrs, counts, ops, True, mapped=self.mapped)


def _check_registered(aloam, call, got):
    """aloam_registered_rows of the call that just ended: its own rows"""
    code, res = got["reg"]
    assert code == OK, code
    begin, count = res
    assert np.array_equal(begin, call.begins()), (begin, call.begins())
    assert np.array_equal(count > 0, np.array(call.kinds) != aloam.ROW_IDLE), count


def _check_records(aloam, call, got, recovery):
    """the records, recovery rows and candidate scores of the call that just ended: its own rows"""
    code, rows = got["map"]
    assert code == OK and list(rows["kind"]) == call.kinds, (code, rows and rows["kind"], call.kinds)
    code, rec = got["rec"]
    assert code == OK
    loc = np.array(call.kinds) == aloam.ROW_LOCALISED
    assert not rec["triggered"][~loc].any()
    if not recovery:
        assert not rec["triggered"].any() and (rec["best"] == -1).all() and not rec["pose"].any()
    trig = rec["triggered"].reshape(-1, B).any(axis=0)
    for l in range(B):
        assert (got["dbg"][l][0] == OK) == bool(trig[l]), (l, got["dbg"][l][0], trig)


def test_the_readers_after_every_ending(aloam, synth):
    import torch
    W = _world(aloam, synth)
    dev, M = W["dev"], W["M"]
    D = RV.deltas(aloam)
    c = _localiser(aloam, W, B)
    sink = torch.zeros((40 * M, 4), dtype=torch.float32, device="cuda")
    c.set_registered_sink(sink)
    c.set_map_rows(True, TC.ISQ, TC.PTS)
    c.set_recovery(True, RV.TRIGGER, RV.ACCEPT, D)
    true = W["map"][TC.START]
    raw4, _ = TE.overflow_scan(synth)
    over = torch.from_numpy(raw4).cuda()
    far = W["scans"][1].copy(); far[:, :3] *= 1e-3   # every point under minimum_range (scanRegistration.cpp:137)
    near = torch.from_numpy(far).cuda()
    small = torch.zeros((16, 4), dtype=torch.float32, device="cuda")

    def arm(T):
        return lambda c: c.lane_localise(0, T[:4], T[4:])

    def both(n, s0=TC.START, s1=0):   # lane 0 localising from scan s0, lane 1 mapping from scan s1
        return Call([[(dev[s0 + k], START if k == 0 else SCAN), (dev[s1 + k], START if k == 0 else SCAN)] for k in range(n)], localising=(0,))

    def lockstep(n, counts=None):
        def run(c):
            ptrs = np.array([[dev[k].data_ptr(), dev[k + 1].data_ptr()] for k in range(n)], np.uint64)
            cnt = np.array([[dev[k].shape[0], dev[k + 1].shape[0]] for k in range(n)], np.int64) if counts is None else counts
            return c.scan_stream_mapped_batch(ptrs, cnt, True)
        run.rows, run.kinds = n * B, [aloam.ROW_MAPPED] * (n * B)
        run.begins = lambda: np.concatenate([[0], np.cumsum([dev[k + l].shape[0] for k in range(n) for l in range(B)])[:-1]])
        return run

    def set_sink(t):
        return lambda c: c.set_registered_sink(t)

    def rows_off(c):
        c.set_map_rows(False)

    def rows_on(c):
        c.set_map_rows(True, TC.ISQ, TC.PTS)

    def recovery_on(trigger=RV.TRIGGER):
        return lambda c: c.set_recovery(True, trigger, RV.ACCEPT, D)

    odo = Call([[(None, IDLE), (dev[k], START if k == 0 else SCAN)] for k in range(2)], mapped=False)
    bad_op = Call([[(dev[0], 5), (dev[0], START)]])
    not_running = Call([[(dev[0], SCAN), (dev[0], START)]])
    empty = Call([[(dev[0], START), (dev[1], START)]], counts={(0, 1): 0})
    huge = Call([[(dev[0], START), (dev[1], START)]], counts={(0, 1): M + 1})
    odo_empty = Call([[(None, IDLE), (dev[0], START)]], mapped=False, counts={(0, 1): 0})
    overflow = Call([[(over, START), (None, IDLE)]], localising=(0,))
    fails = Call([[(dev[TC.START], START), (near, START)]], localising=(0,))

    # (what, set-up, call, expected return code, registered_rows, map_rows / recovery_rows, debug_recovery_scores, recovery ran)
    table = [
        ("mapped, recording on", arm(TC.mis_armed(true)), both(3), OK, "this", "this", "this", True),
        ("unmapped lanes call", None, odo, OK, "prev", "prev", "prev", None),
        ("bad op", None, bad_op, ERR_INVALID_ARG, "prev", "prev", "prev", None),
        ("SCAN of a lane that is not running", None, not_running, ERR_STATE, "prev", "prev", "prev", None),
        ("registered clouds over the sink", set_sink(small), both(2), ERR_CAPACITY, "prev", "prev", "prev", None),
        ("lockstep call in lane mode", set_sink(sink), lockstep(1), ERR_STATE, "prev", "prev", "prev", None),
        ("unmapped lanes call with an empty scan", None, odo_empty, ERR_EMPTY_CLOUD, "prev", "prev", "prev", None),
        ("mapped call, recording on again", arm(TC.mis_armed(true)), both(2), OK, "this", "this", "this", True),
        ("mapped lanes call with an empty scan", None, empty, ERR_EMPTY_CLOUD, "prev", "state", "prev", None),
        ("mapped lanes call with an oversized scan", None, huge, ERR_CAPACITY, "prev", "state", "prev", None),
        ("reset_odometry", None, lambda c: c.reset_odometry(), OK, "prev", "prev", "prev", None),
        ("scan_to_pose", None, lambda c: c.scan_to_pose(W["scans"][0]), OK, "prev", "prev", "prev", None),
        ("reset_odometry again", None, lambda c: c.reset_odometry(), OK, "prev", "prev", "prev", None),
        ("lockstep call with an empty view", None, lockstep(1, np.array([[dev[0].shape[0], 0]])), ERR_EMPTY_CLOUD,
         "prev", "prev", "prev", None),
        ("lockstep mapped call", None, lockstep(2), OK, "this", "this", "this", True),
        ("mapped call, recording off", rows_off, both(2), OK, "this", "state", "state", None),
        ("mapped call, recording on, recovery off", [rows_on, arm(TC.mis_armed(true))], both(3), OK, "this", "this", "this", False),
        ("mapped call, recovery on", [recovery_on(), arm(TC.mis_armed(true))], both(2), OK, "this", "this", "this", True),
        ("key overflow", [arm(TC.mis_armed(W["map"][4])), recovery_on(1.0)], overflow, ERR_CAPACITY, "this", "this", "this", True),
        ("mapped call fails inside the run", arm(TC.mis_armed(true)), fails, ERR_EMPTY_CLOUD, "state", "state", "state", None),
        ("bad op after the failure", None, bad_op, ERR_INVALID_ARG, "prev", "prev", "prev", None),
    ]
    prev, prev_rows, triggered = None, 0, 0
    for what, setup, call, want, reg, rows, dbg, recovery in table:
        for s in (setup if isinstance(setup, list) else [setup] if setup else []):
            s(c)
        code, _ = _code(aloam, lambda: call(c))
        assert code == want, (what, code, want)
        n = call.rows if "this" in (reg, rows) else prev_rows
        got = _readers(aloam, c, n)
        if reg == "this":
            _check_registered(aloam, call, got)
        if rows == "this":
            assert dbg == "this"
            _check_records(aloam, call, got, recovery)
            triggered += sum(g[0] == OK for g in got["dbg"])
        for key, rule in (("reg", reg), ("map", rows), ("rec", rows), ("dbg", dbg)):
            if rule == "prev":
                assert _same(got[key], prev[key]), (what, key)
            elif rule == "state":
                codes = [g[0] for g in got[key]] if key == "dbg" else [got[key][0]]
                assert all(x == ERR_STATE for x in codes), (what, key, codes)
        prev, prev_rows = got, n
    assert triggered > 0   # some call left candidate scores to read
    c.close()
