"""The directed split (b2_split_tracks_directed: segment offsets monotone in one direction) restated beside
oracle/split_oracle.py (TEST INFRASTRUCTURE), in plain Python floats and vectorised over the window.

The programme (DESIGN.md section 4 "K9s"), direction d = +1 (offsets only grow) or -1 (only shrink):
    P_{j-1}(o) = max { V_{j-1}(o') : o' < o }   (d = -1: o' > o; -inf when empty)
    V_0 = u_0,   V_j(o) = u_j(o) + max(V_{j-1}(o), P_{j-1}(o) - penalty)
with split_oracle's rounding (c = P - penalty, then the decision c > V, staying on a tie, then u + (c or V), each
rounded on its own) and its final argmax (the largest offset among equal maxima).  A switch at (j, o) comes from the
argmax of V_{j-1} over the allowed side, ties to the largest offset.

The plain restatement stores every V row and finds each source by that argmax.  The vectorised one keeps only the
record bits the kernel stores (V_{j-1}(o) >= P_{j-1}(o) for d = +1, V_{j-1}(o) > S_{j-1}(o), the exclusive suffix
maximum, for d = -1) and takes the nearest record behind o, so holding the two to each other checks the record
argument.  numpy rounds each elementwise operation on its own as Python floats do, so the two agree bit for bit.
"""
import math

import numpy as np

from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp


def _argmax_range(row, idx):
    """The largest index among the maxima of row over idx (ascending indices); None when idx is empty."""
    best, k = -math.inf, None
    for i in idx:
        if row[i] >= best:
            best, k = row[i], i
    return k


def solve_directed(U, offsets, penalty, d):
    """The directed programme over the unit x offset table U (Python floats), sources by argmax over the stored rows.
    Returns (path offsets per unit, split_score, final maximum)."""
    W, n = len(offsets), len(U)
    V = list(U[0])
    rows, dec = [V], []
    for j in range(1, n):
        P = [-math.inf] * W
        run = -math.inf
        for i in (range(W) if d > 0 else range(W - 1, -1, -1)):
            P[i] = run
            run = V[i] if V[i] > run else run
        sw, Vn = [], []
        for i in range(W):
            c = P[i] - penalty
            s = c > V[i]
            sw.append(s)
            Vn.append(U[j][i] + (c if s else V[i]))
        dec.append(sw)
        V = Vn
        rows.append(V)
    k = _argmax_range(V, range(W))
    top = V[k]
    path = [k]
    for j in range(n - 1, 0, -1):
        if dec[j - 1][k]:
            k = _argmax_range(rows[j - 1], range(0, k) if d > 0 else range(k + 1, W))
        path.append(k)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + U[j][i]
    return [offsets[i] for i in path], score, top


def prefix(V, d):
    """The exclusive prefix (d = +1) or suffix (d = -1) maximum of the float64 row V (-inf where empty)."""
    if d > 0:
        return np.concatenate([[-np.inf], np.maximum.accumulate(V)[:-1]])
    return np.concatenate([np.maximum.accumulate(V[::-1])[::-1][1:], [-np.inf]])


def records(V, d):
    """The record bits of the row V: V >= the prefix maximum (d = +1), V > the suffix maximum (d = -1)."""
    P = prefix(V, d)
    return V >= P if d > 0 else V > P


def programme(U, penalty, d):
    """The directed programme vectorised over a float64 table U [units, offsets]: (M [units] maxima, the last unit's
    argmax index, SW [units, offsets] switch decisions, REC [units, offsets] the records of V_{j-1}; row 0 of SW and
    REC all False)."""
    U = np.asarray(U, np.float64)
    n, W = U.shape
    M = np.empty(n)
    SW = np.zeros((n, W), bool)
    REC = np.zeros((n, W), bool)
    V = U[0].copy()
    M[0] = V.max()
    for j in range(1, n):
        P = prefix(V, d)
        REC[j] = V >= P if d > 0 else V > P
        c = P - penalty
        SW[j] = c > V
        V = U[j] + np.where(SW[j], c, V)
        M[j] = V.max()
    return M, W - 1 - int(np.argmax(V[::-1])), SW, REC


def source(rec, k, d):
    """The nearest record behind k: the largest set index below k (d = +1), the smallest above it (d = -1)."""
    if d > 0:
        return int(np.flatnonzero(rec[:k])[-1])
    return k + 1 + int(np.flatnonzero(rec[k + 1:])[0])


def solve(U, offsets, penalty, d):
    """solve_directed over a float64 table U through programme, sources through the record bits."""
    U = np.asarray(U, np.float64)
    M, k, SW, REC = programme(U, penalty, d)
    n = len(U)
    path = [k]
    for j in range(n - 1, 0, -1):
        if SW[j, k]:
            k = source(REC[j], k, d)
        path.append(k)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + float(U[j][i])
    return [offsets[i] for i in path], score, float(M[-1])


def split_track(ref, cue_start, cue_end, keep, ratio, sample_rate, start_seconds, max_offset_samples, penalty, d,
                vectorised=True):
    """One track split in direction d: (cue_offset list, n_segments, split_score).  A NaN ratio or an empty window:
    ([0]*, 0, NaN).  vectorised: the tables of tests/split_wide.py and solve above; otherwise split_oracle's unit
    scores and solve_directed."""
    import split_wide as sw
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
    lv = sp.levels(ratio, beta)
    runs = sp.runs_of(mask)
    units = sp.units_of(runs, S)
    if vectorised:
        path, score, _ = solve(sw.unit_table(m, units, offsets, lv), offsets, penalty, d)
    else:
        path, score, _ = solve_directed([sp.unit_scores(m, u, offsets, lv) for u in units], offsets, penalty, d)
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
                 max_offset_samples, penalty, d, vectorised=True):
    """b2_split_tracks_directed over T tracks: (cue_offset [cues], n_segments [T], split_score [T]) as numpy arrays."""
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
                                      max_offset_samples, penalty, d, vectorised)
        co[c0:c1] = o
    return co, ns, sc
