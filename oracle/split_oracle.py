"""Per-segment offsets with a split penalty (b2_split_tracks, b2_apply_split) restated in numpy (TEST INFRASTRUCTURE).

The objective (DESIGN.md section 4 "K9s"): a track's mask, rasterised at its ratio, is cut into units (the gap before
each run of 1s and the run; the leading gap in unit 0, the frames after the last run in the last unit).  u_j(o) is
unit j's four-count score against the two-level reference at offset o, and over the aligner's window
    V_0 = u_0,   V_j(o) = u_j(o) + max(V_{j-1}(o), max V_{j-1} - penalty)
in float64 with every operation rounded on its own (Python floats), staying on a tie, the largest offset among equal
maxima.  Counts come from plain frame sums over each unit (``unit_scores``), or from explicit per-frame enumeration
(``unit_score_brute``, tiny cases); the packed-bit prefix arithmetic of the kernels is not used here.
"""
import math

import numpy as np

from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import sync_output_oracle as so


class ThreeLevels(Exception):
    """The reference holds a third level (or a non-finite second one): b2_split_tracks refuses it."""


def ref_levels(ref):
    """(m, beta) of a two-level reference: m = (r == 1.0); beta the other value (0.0 when every frame is 1.0)."""
    r = np.asarray(ref, dtype=np.float64)
    m = r == 1.0
    other = np.flatnonzero(~m)
    beta = float(r[other[0]]) if len(other) else 0.0
    bad = other[~(r[other] == beta)] if len(other) else other
    if len(other) and not math.isfinite(beta):
        raise ThreeLevels(int(other[0]))
    if len(bad):
        raise ThreeLevels(int(bad[0]))
    return m, beta


def levels(ratio, beta):
    level = float(np.float32(min(1.0 / ratio, 1.0)))
    hi = 2.0 * level - 1.0
    alpha = 2.0 * beta - 1.0
    return hi, alpha, hi * alpha


def runs_of(mask):
    x = np.concatenate([[0], np.asarray(mask, np.int8), [0]])
    d = np.flatnonzero(np.diff(x))
    return list(zip(d[0::2].tolist(), d[1::2].tolist()))


def units_of(runs, S):
    """[(start, a, b, end)] per unit."""
    if not runs:
        return [(0, 0, 0, S)]
    out = []
    for j, (a, b) in enumerate(runs):
        out.append((0 if j == 0 else runs[j - 1][1], a, b, S if j == len(runs) - 1 else b))
    return out


def _score(hi, alpha, hia, n_ov, mw, uo, um):
    if n_ov == 0:
        return 0.0
    c11, c01, c10, c00 = float(um), float(mw - um), float(uo - um), float(n_ov - mw - uo + um)
    return (hi * c11 - c01) + (hia * c10 - alpha * c00)


def unit_score_brute(m, mask, unit, o, lv):
    """u_j(o) by enumerating the unit's frames of the overlap."""
    start, _, _, end = unit
    R = len(m)
    c = [[0, 0], [0, 0]]
    n = 0
    for f in range(start, end):
        p = f + o
        if 0 <= p < R:
            c[int(mask[f])][int(m[p])] += 1
            n += 1
    um, mw, uo = c[1][1], c[1][1] + c[0][1], c[1][1] + c[1][0]
    return _score(*lv, n, mw, uo, um)


def unit_scores(m, unit, offsets, lv):
    """u_j(o) for every offset of the window from frame sums (vectorised over offsets)."""
    start, a, b, end = unit
    R = len(m)
    M = np.concatenate([[0], np.cumsum(m.astype(np.int64))])
    o = np.asarray(offsets, np.int64)

    def Mc(p):
        return M[np.clip(p, 0, R)]

    def ov(lo, hi):
        return np.maximum(0, np.minimum(hi, R - o) - np.maximum(lo, -o))

    n_ov = ov(start, end)
    mw = Mc(end + o) - Mc(start + o)
    uo = ov(a, b)
    um = Mc(b + o) - Mc(a + o)
    return [_score(*lv, int(n_ov[i]), int(mw[i]), int(uo[i]), int(um[i])) for i in range(len(o))]


def solve(U, offsets, penalty):
    """The programme over the unit x offset table U (Python floats).  Returns (path offsets per unit, split_score)."""
    W = len(offsets)
    V = list(U[0])
    dec, args = [], []

    def argmax(x):
        best, k = -math.inf, 0
        for i in range(W):
            if x[i] >= best:   # increasing offsets: ties go to the largest
                best, k = x[i], i
        return best, k

    for j in range(1, len(U)):
        mx, k = argmax(V)
        args.append(k)
        c = mx - penalty
        sw = [c > V[i] for i in range(W)]
        dec.append(sw)
        V = [U[j][i] + (c if sw[i] else V[i]) for i in range(W)]
    _, k = argmax(V)
    path = [k]
    for j in range(len(U) - 1, 0, -1):
        if dec[j - 1][k]:
            k = args[j - 1]
        path.append(k)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + U[j][i]
    return [offsets[i] for i in path], score


def split_track(ref, cue_start, cue_end, keep, ratio, sample_rate, start_seconds, max_offset_samples, penalty,
                brute=False):
    """One track: (cue_offset list, n_segments, split_score).  A NaN ratio or an empty window: ([0]*, 0, NaN)."""
    n = len(cue_start)
    if math.isnan(ratio) or len(ref) == 0:
        return [0] * n, 0, math.nan
    m, beta = ref_levels(ref)
    samples = ro.rasterize(cue_start, cue_end, keep, sample_rate, start_seconds, ratio)[0]
    mask = samples > 0
    S, R = len(mask), len(m)
    o_lo, o_hi = ao.offset_range(R, S, max_offset_samples)
    if o_lo > o_hi:
        return [0] * n, 0, math.nan
    offsets = list(range(o_lo, o_hi + 1))
    lv = levels(ratio, beta)
    runs = runs_of(mask)
    units = units_of(runs, S)
    if brute:
        U = [[unit_score_brute(m, mask, u, o, lv) for o in offsets] for u in units]
    else:
        U = [unit_scores(m, u, offsets, lv) for u in units]
    path, score = solve(U, offsets, penalty)
    n_seg = 1 + sum(1 for j in range(1, len(path)) if path[j] != path[j - 1])
    cue_off = []
    for i in range(n):
        st = ro.scale_seconds(float(cue_start[i]), ratio)
        first = int(round((st - start_seconds) * sample_rate))
        f = min(max(slice(first, first).indices(S)[0], 0), S - 1)
        j = next((k for k, (_, b) in enumerate(runs) if b > f), len(units) - 1)
        cue_off.append(path[j])
    return cue_off, n_seg, score


def split_tracks(ref, ref_off, track_video, cue_start, cue_end, cue_keep, cue_off, ratio, sample_rate, start_seconds,
                 max_offset_samples, penalty):
    """b2_split_tracks over T tracks: (cue_offset [cues], n_segments [T], split_score [T]) as numpy arrays."""
    T = len(cue_off) - 1
    co = np.zeros(int(cue_off[-1]), np.int32)
    ns = np.zeros(T, np.int32)
    sc = np.full(T, np.nan)
    for t in range(T):
        v = int(track_video[t])
        c0, c1 = int(cue_off[t]), int(cue_off[t + 1])
        keep = None if cue_keep is None else [bool(k) for k in cue_keep[c0:c1]]
        o, ns[t], sc[t] = split_track(np.asarray(ref[ref_off[v]:ref_off[v + 1]]), cue_start[c0:c1], cue_end[c0:c1],
                                      keep, float(ratio[t]), sample_rate, start_seconds, max_offset_samples, penalty)
        co[c0:c1] = o
    return co, ns, sc


def apply_split(ratio, n_segments, cue_offset, cue_start, cue_end, cue_off, sample_rate, apply_offset_seconds=0.0):
    """b2_apply_split: (synced_start_us, synced_end_us, status) through sync_output_oracle's arithmetic."""
    T = len(cue_off) - 1
    n = int(cue_off[-1])
    su, eu = np.zeros(n, np.int64), np.zeros(n, np.int64)
    st = np.zeros(T, np.int32)
    for t in range(T):
        live = int(n_segments[t]) > 0
        st[t] = (so.WRITTEN | so.APPLIED) if live else so.FAILED
        for i in range(int(cue_off[t]), int(cue_off[t + 1])):
            if live:
                _, scale, off = so.decide(0.0, int(cue_offset[i]), 0, [float(ratio[t])], None, sample_rate,
                                          apply_offset_seconds)
                su[i] = so.td_us(float(cue_start[i]) * scale) + so.td_us(off)
                eu[i] = so.td_us(float(cue_end[i]) * scale) + so.td_us(off)
            else:
                su[i], eu[i] = so.td_us(float(cue_start[i])), so.td_us(float(cue_end[i]))
    return su, eu, st
