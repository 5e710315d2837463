"""Scenes and host computations of the recovery edge-case tests (tests/test_gpu_recovery_edges.py, checked on the CPU by
tests/test_oracle_recovery_edges.py): the float32 fractions that put a row exactly on either side of the trigger and accept tests,
armings that spread a START row's score, the 16-lane schedule whose localising records are not its lanes, candidate sets sized
around one resident wave of k_reloc_score with planted ties, odd deltas, and the settings a context goes through.

Everything builds on the scenario of tests/recovery_cases.py (the VLP-16 world of tests/track_cases.py); the staging and overflow
scans are those of tests/track_edge_cases.py."""
import numpy as np

import recovery_cases as RV
import reloc_cases as RC
import track_cases as TC

# ------------------------------------------------------------------------------------------------- A. float boundaries
ONE32, ZERO32 = np.float32(1), np.float32(0)


def frac_at_most(score, n):
    """the largest float32 f with f * n <= score in float32: a row (score, n) does not trigger at f, and a best score `score`
    holds accept_frac f of n"""
    s, nn = np.float32(score), np.float32(n)
    f = np.float32(s / nn)
    while f > 0 and f * nn > s:
        f = np.nextafter(f, ZERO32)
    while np.nextafter(f, ONE32 + ONE32) * nn <= s:
        f = np.nextafter(f, ONE32 + ONE32)
    return f


def frac_pair(score, n):
    """(f_lo, f_hi = the next float up): the row triggers at f_hi and not at f_lo; a best score `score` is accepted at f_lo and
    not at f_hi"""
    lo = frac_at_most(score, n)
    return lo, np.nextafter(lo, ONE32 + ONE32)


def turned(pose, yaw_deg, off):
    """pose turned by yaw_deg about z (on the left, as TC.mis_armed) and moved by off"""
    yaw = np.radians(yaw_deg)
    out = np.array(pose, np.float64, copy=True)
    out[:4] = TC.qmul(np.array([0, 0, np.sin(yaw / 2), np.cos(yaw / 2)]), out[:4])
    out[4:] = out[4:] + np.asarray(off, np.float64)
    return out


def spread_armings(true):
    """16 armings of one scan whose START rows cover a spread of score / n_score: the true pose, offsets of a few tenths of a
    metre and a few degrees, mis-armed by 20 .. 60 degrees and 1.5 .. 3.5 m, and two off the map (score 0)"""
    out = [np.array(true, np.float64)]
    for k in range(1, 7):
        out.append(turned(true, 1.5 * k * (-1) ** k, (0.15 * k, -0.1 * k, 0.0)))
    for k in range(7):
        out.append(turned(true, 20.0 + 7.0 * k, (1.5 + 0.3 * k, 3.0 - 0.8 * k, 0.0)))
    out.append(TC.off_map(true))
    out.append(TC.off_map(turned(true, 90.0, (0, 0, 0))))
    return out


def lost_armings(true):
    """16 armings whose START rows all lose track (every one triggers at trigger_frac 1 and, on the oracle, scores below
    TC.LOST_RATIO): gross heading and position errors, two off the map"""
    out = [turned(true, 40.0 + 9.0 * k, (2.5 + 0.25 * (k % 4), 3.0 - 1.5 * (k // 4), 0.0)) for k in range(14)]
    return out + [TC.off_map(true), TC.off_map(turned(true, -45.0, (0, 0, 0)))]


# ---------------------------------------------------------------------------------------- B. records that are not lanes
SKIP = 2
STEPS = 6
MAPPING = (0, 5, 10)                       # mapping lanes, interleaved among the localising ones
MIS, OFF, TRUE = (1, 6, 11, 14), (3, 8, 13), (2, 4, 7, 9, 12, 15)


def start_step(lane):
    """the step a lane STARTs at: mapping lanes at 0, localising lanes at 0, 1 or 2 (idle before)"""
    return 0 if lane in MAPPING else lane % 3


def records_schedule(n_scans_world):
    """ops (STEPS, 16) and scan indices of the 16-lane call: mapping lanes run scans 0 .., localising lanes TC.START .. from their
    START step on"""
    ops = np.zeros((STEPS, 16), np.int32)
    idx = np.zeros((STEPS, 16), np.int64)
    for l in range(16):
        s0 = start_step(l)
        first = 0 if l in MAPPING else TC.START
        for k in range(s0, STEPS):
            ops[k, l] = 2 if k == s0 else 1
            idx[k, l] = first + k - s0
    assert idx.max() < n_scans_world
    return ops, idx


def records_armed(true):
    """lane -> arming of the localising lanes: mis-armed, off the map and true"""
    out = {l: TC.mis_armed(true) for l in MIS}
    out.update({l: TC.off_map(true) for l in OFF})
    out.update({l: np.array(true, np.float64) for l in TRUE})
    return out


def localising_records(kinds, localised=2):
    """per step, [(record index, lane)] of the localising rows: records are the localising lanes of the step in lane order"""
    return [[(i, l) for i, l in enumerate(np.flatnonzero(row == localised))] for row in kinds]


# --------------------------------------------------------------------------------------------------- C. candidate sets
CAND_THREADS = 256          # k_recover_cand's CTA
RELOC_WARPS = 8             # warps (hypotheses in flight) per CTA of k_reloc_score
RELOC_CTAS_PER_SM = 4       # k_reloc_score's __launch_bounds__(256, 4): 55 registers, 4 CTAs per SM
MAX_DELTA = 65536


def wave(sms, per_sm=RELOC_CTAS_PER_SM):
    """W: the hypotheses of one resident wave of k_reloc_score"""
    return sms * per_sm * RELOC_WARPS


def sizes(sms):
    """the n_delta of the size cases"""
    W = wave(sms)
    return [1, 255, 256, 257, W - 1, W, W + 1, 2 * W + 3]


def ctas(n, sms):
    """CTAs of a record's k_reloc_score launch (reloc_score_ctas)"""
    return max(1, min(sms * RELOC_CTAS_PER_SM, (n + RELOC_WARPS - 1) // RELOC_WARPS))


def cta_warp(h, n, sms):
    """(CTA, warp) that scores hypothesis h of n: the grid-stride loop hands hypotheses out 8 per CTA, wave after wave"""
    return (h // RELOC_WARPS) % ctas(n, sms), h % RELOC_WARPS


def tie_layout(sms):
    """(n, early, late) of the cross-CTA tie: n = 2W + 3 (the grid-stride loop wraps twice); `late` in the last CTA's warp 5 of the
    first wave, `early` < late in CTA 2's warp 1"""
    W = wave(sms)
    C = sms * RELOC_CTAS_PER_SM
    return 2 * W + 3, 8 * 2 + 1, 8 * (C - 1) + 5


def tail_layout(sms):
    """n of the tail case: the last index n - 1 is scored by the last CTA, and k_recover_cand's last CTA is partial"""
    return wave(sms) - 3


FAR_T = 1.0e3   # a delta's translation that moves every scoring point of a scan of the world off the prior map


def far_deltas(n, seed=0):
    """n deltas that score 0 on the world: headings anywhere, 1 km up and a few metres across"""
    rng = np.random.default_rng(seed)
    yaw = rng.uniform(-np.pi, np.pi, n)
    D = np.zeros((n, 7))
    D[:, 2], D[:, 3] = np.sin(yaw / 2), np.cos(yaw / 2)
    D[:, 4:6] = rng.uniform(-4, 4, (n, 2))
    D[:, 6] = FAR_T
    return D


def random_deltas(n, seed=1, half=4.0):
    """n deltas around the identity: any heading, +-half m across, unnormalised quaternions (scaled by 0.5 .. 2)"""
    rng = np.random.default_rng(seed)
    yaw = rng.uniform(-np.pi, np.pi, n)
    s = rng.uniform(0.5, 2.0, n)
    D = np.zeros((n, 7))
    D[:, 2], D[:, 3] = s * np.sin(yaw / 2), s * np.cos(yaw / 2)
    D[:, 4:6] = rng.uniform(-half, half, (n, 2))
    D[:, 6] = rng.uniform(-0.2, 0.2, n)
    return D


def odd_deltas():
    """(name, delta): quaternions scaled by 1e-3 and 1e3, negated (w < 0), a 180 degree turn (w = 0), turns about x and about
    (1, 1, 1), and translations of +-1e4"""
    a = np.radians(30.0)
    z = np.array([0, 0, np.sin(a / 2), np.cos(a / 2)])
    ax = np.array([np.sin(0.2), 0, 0, np.cos(0.2)])
    u = np.sin(0.15) / np.sqrt(3.0)
    return [("scaled-1e-3", np.r_[z * 1e-3, 0.5, -0.25, 0.0]), ("scaled-1e3", np.r_[z * 1e3, -0.5, 0.25, 0.0]),
            ("negated", np.r_[-z, 0.0, 0.0, 0.0]), ("half-turn", np.r_[0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0]),
            ("x-axis", np.r_[ax, 0.0, 0.0, 0.1]), ("111-axis", np.r_[u, u, u, np.cos(0.15), 1.0, 1.0, 0.0]),
            ("t+1e4", np.r_[0.0, 0.0, 0.0, 1.0, 1e4, 0.0, 0.0]), ("t-1e4", np.r_[z, -1e4, -1e4, -1e4])]


def products(P, Dn):
    """RV.products over many normalised deltas at once: cubemap.cu's qmul term for term, elementwise (the same IEEE double
    operations in the same order, so the same bits)"""
    Dn = np.asarray(Dn, np.float64).reshape(-1, 7)
    ax, ay, az, aw = Dn[:, 0], Dn[:, 1], Dn[:, 2], Dn[:, 3]
    bx, by, bz, bw = (float(v) for v in P[:4])
    out = np.empty_like(Dn)
    out[:, 3] = aw * bw - ax * bx - ay * by - az * bz
    out[:, 0] = aw * bx + ax * bw + ay * bz - az * by
    out[:, 1] = aw * by + ay * bw + az * bx - ax * bz
    out[:, 2] = aw * bz + az * bw + ax * by - ay * bx
    for k in range(3):
        out[:, 4 + k] = float(P[4 + k]) + Dn[:, 4 + k]
    return out


def hypotheses(P, D):
    """the hypotheses whose aloam_prior_relocalise coarse scores the device's candidate scores must equal: products(P,
    normalised(D)), which relocalisation normalises as k_recover_cand does"""
    return products(P, RC.normalised(D))


# ---------------------------------------------------------------------------------------- D. settings over a context's life
def grid_deltas(aloam):
    """20 808 deltas: the recovery lattice at +-8 m, 1 m and 72 headings"""
    return RV.deltas(aloam, half=8.0, step=1.0, n_yaw=72)


def settings(aloam):
    """the n_delta sequence of one context: small, large, smaller, the limit"""
    return [("n3", random_deltas(3, seed=3)), ("n20808", grid_deltas(aloam)), ("n5", random_deltas(5, seed=5)),
            ("n65536", random_deltas(MAX_DELTA, seed=7))]
