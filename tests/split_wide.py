"""oracle/split_oracle.py vectorised over the window, for windows past a few thousand offsets (TEST INFRASTRUCTURE).

The pure-Python ``split_oracle.solve`` takes a Python call per cell, too slow for the 262 144-offset windows of
b2_split_tracks_wide.  Here every unit's scores and every step of the programme are numpy float64 arrays: numpy
rounds each elementwise operation on its own, as Python floats do, so each cell equals the pure-Python oracle's bit
for bit (tests/test_split_wide_cpu.py checks that), and the argmax is np.argmax over the reversed window.
"""
import math

import numpy as np

from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp


def unit_table(m, units, offsets, lv):
    """split_oracle.unit_scores of every unit as one float64 array [units, offsets]: the same counts, the same order
    of operations."""
    R = len(m)
    M = np.concatenate([[0], np.cumsum(np.asarray(m).astype(np.int64))])
    o = np.asarray(offsets, np.int64)
    hi, alpha, hia = lv

    def Mc(p):
        return M[np.clip(p, 0, R)]

    def ov(lo, h):
        return np.maximum(0, np.minimum(h, R - o) - np.maximum(lo, -o))

    U = np.empty((len(units), len(o)))
    for j, (start, a, b, end) in enumerate(units):
        n_ov = ov(start, end)
        mw = Mc(end + o) - Mc(start + o)
        uo = ov(a, b)
        um = Mc(b + o) - Mc(a + o)
        c11, c01, c10, c00 = (x.astype(np.float64) for x in (um, mw - um, uo - um, n_ov - mw - uo + um))
        U[j] = np.where(n_ov == 0, 0.0, (hi * c11 - c01) + (hia * c10 - alpha * c00))
    return U


def solve(U, offsets, penalty):
    """split_oracle.solve over a float64 array U [units, offsets]: (path offsets per unit, split_score)."""
    U = np.asarray(U, np.float64)
    n, W = U.shape

    def argmax(x):   # ties: the largest offset
        k = W - 1 - int(np.argmax(x[::-1]))
        return float(x[k]), k

    V = U[0].copy()
    dec, args = [], []
    for j in range(1, n):
        mx, k = argmax(V)
        args.append(k)
        c = mx - penalty
        sw = c > V
        dec.append(sw)
        V = U[j] + np.where(sw, c, V)
    _, k = argmax(V)
    path = [k]
    for j in range(n - 1, 0, -1):
        if dec[j - 1][k]:
            k = args[j - 1]
        path.append(k)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + float(U[j][i])
    return [offsets[i] for i in path], score


def split_track(ref, cue_start, cue_end, keep, ratio, sample_rate, start_seconds, max_offset_samples, penalty):
    """split_oracle.split_track through unit_table and solve."""
    n = len(cue_start)
    if math.isnan(ratio) or len(ref) == 0:
        return [0] * n, 0, math.nan
    m, beta = sp.ref_levels(ref)
    mask = ro.rasterize(cue_start, cue_end, keep, sample_rate, start_seconds, ratio)[0] > 0
    S, R = len(mask), len(m)
    o_lo, o_hi = ao.offset_range(R, S, max_offset_samples)
    if o_lo > o_hi:
        return [0] * n, 0, math.nan
    offsets = list(range(o_lo, o_hi + 1))
    runs = sp.runs_of(mask)
    units = sp.units_of(runs, S)
    path, score = solve(unit_table(m, units, offsets, sp.levels(ratio, beta)), offsets, penalty)
    n_seg = 1 + sum(1 for j in range(1, len(path)) if path[j] != path[j - 1])
    ends = np.array([b for _, b in runs], np.int64)
    cue_off = []
    for i in range(n):
        st = ro.scale_seconds(float(cue_start[i]), ratio)
        first = int(round((st - start_seconds) * sample_rate))
        f = min(max(slice(first, first).indices(S)[0], 0), S - 1)
        j = int(np.searchsorted(ends, f, side="right")) if len(runs) else 0   # first run ending after f
        cue_off.append(path[min(j, len(units) - 1)])
    return cue_off, n_seg, score


def split_tracks(ref, ref_off, track_video, cue_start, cue_end, cue_keep, cue_off, ratio, sample_rate, start_seconds,
                 max_offset_samples, penalty):
    """split_oracle.split_tracks through split_track above."""
    T = len(cue_off) - 1
    co = np.zeros(int(cue_off[-1]), np.int32)
    ns = np.zeros(T, np.int32)
    sc = np.full(T, np.nan)
    for t in range(T):
        v = int(track_video[t])
        c0, c1 = int(cue_off[t]), int(cue_off[t + 1])
        keep = None if cue_keep is None else [bool(k) for k in cue_keep[c0:c1]]
        o, ns[t], sc[t] = split_track(np.asarray(ref[ref_off[v]:ref_off[v + 1]], np.float64), cue_start[c0:c1],
                                      cue_end[c0:c1], keep, float(ratio[t]), sample_rate, start_seconds,
                                      max_offset_samples, penalty)
        co[c0:c1] = o
    return co, ns, sc
