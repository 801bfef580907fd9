"""The split along stated breaks (b2_split_tracks_breaks) restated beside oracle/split_oracle.py (TEST
INFRASTRUCTURE), in plain Python floats and vectorised over the window.

The programme (DESIGN.md section 4 "K9s"), breaks = (d_1, .., d_n), each +1 or -1: layer m holds the paths with
exactly m breaks, the i-th break moving the offset strictly up (d_i = +1) or down (-1),
    V_{0,0} = u_0,  V_{0,m} = -inf (m >= 1),  V_{j,0} = u_j + V_{j-1,0},
    c = P^{d_m}_{j-1,m-1}(o) - penalty,   V_{j,m}(o) = u_j(o) + (c if c > V_{j-1,m}(o) else V_{j-1,m}(o))
with P^{+1} the exclusive prefix maximum over o' < o and P^{-1} the exclusive suffix maximum over o' > o (-inf when
empty), each operation rounded on its own as in split_oracle.  profile[m] = max_o V_{last,m}; the path ends at the
largest V_{last,m}(o) over (m, o), ties to the largest offset and then the smallest m.  A break at (j, m, o) comes from
the argmax of V_{j-1,m-1} over the d_m side of o, ties to the largest offset.

The plain restatement stores every row and finds each source by that argmax.  The vectorised one keeps only the
switch and record bits the kernel stores (tests/split_directed.py's record rule, per layer) and takes the nearest
record behind o.  numpy rounds each elementwise operation on its own as Python floats do, so the two agree bit for bit.
"""
import math

import numpy as np

import split_directed as sd
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp


def _end(rows):
    """(m, i) of the largest rows[m][i], ties to the largest i and then the smallest m."""
    best, bm, bi = -math.inf, 0, -1
    for m, row in enumerate(rows):
        for i, x in enumerate(row):
            if x > best or (x == best and i > bi):
                best, bm, bi = x, m, i
    return bm, bi


def solve_breaks(U, offsets, penalty, breaks):
    """The programme over the unit x offset table U (Python floats), sources by argmax over the stored rows.  Returns
    (path offsets per unit, split_score, profile list, the end's layer)."""
    W, n, L = len(offsets), len(U), len(breaks) + 1
    V = [list(map(float, U[0]))] + [[-math.inf] * W for _ in range(L - 1)]
    rows, dec = [V], []
    for j in range(1, n):
        Vn, sw = [[U[j][i] + V[0][i] for i in range(W)]], [[False] * W]
        for m in range(1, L):
            d = breaks[m - 1]
            P = [-math.inf] * W
            run = -math.inf
            for i in (range(W) if d > 0 else range(W - 1, -1, -1)):
                P[i] = run
                run = V[m - 1][i] if V[m - 1][i] > run else run
            row, s = [], []
            for i in range(W):
                c = P[i] - penalty
                x = c > V[m][i]
                s.append(x)
                row.append(U[j][i] + (c if x else V[m][i]))
            Vn.append(row)
            sw.append(s)
        dec.append(sw)
        V = Vn
        rows.append(V)
    profile = [max(r) for r in V]
    m, k = _end(V)
    m_end = m
    path = [k]
    for j in range(n - 1, 0, -1):
        if dec[j - 1][m][k]:
            d = breaks[m - 1]
            k = sd._argmax_range(rows[j - 1][m - 1], range(0, k) if d > 0 else range(k + 1, W))
            m -= 1
        path.append(k)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + U[j][i]
    return [offsets[i] for i in path], score, profile, m_end


def programme(U, penalty, breaks):
    """The programme vectorised over a float64 table U [units, offsets]: (profile [L], the end (m, index), SW [units, L,
    offsets] switch decisions, REC [units, L, offsets] with REC[j, m] the records of V_{j-1,m-1} on the d_m side; unit 0
    and layer 0 all False)."""
    U = np.asarray(U, np.float64)
    n, W = U.shape
    L = len(breaks) + 1
    SW = np.zeros((n, L, W), bool)
    REC = np.zeros((n, L, W), bool)
    V = np.full((L, W), -np.inf)
    V[0] = U[0]
    for j in range(1, n):
        Vn = np.empty_like(V)
        Vn[0] = U[j] + V[0]
        for m in range(1, L):
            d = breaks[m - 1]
            REC[j, m] = sd.records(V[m - 1], d)
            c = sd.prefix(V[m - 1], d) - penalty
            SW[j, m] = c > V[m]
            Vn[m] = U[j] + np.where(SW[j, m], c, V[m])
        V = Vn
    profile = V.max(axis=1)
    args = W - 1 - np.argmax(V[:, ::-1], axis=1)   # each layer's largest argmax
    m = 0
    for x in range(1, L):
        if profile[x] > profile[m] or (profile[x] == profile[m] and args[x] > args[m]):
            m = x
    return profile, (m, int(args[m])), SW, REC


def solve(U, offsets, penalty, breaks):
    """solve_breaks over a float64 table U through programme, sources through the record bits."""
    U = np.asarray(U, np.float64)
    profile, (m, k), SW, REC = programme(U, penalty, breaks)
    m_end = m
    path = [k]
    for j in range(len(U) - 1, 0, -1):
        if SW[j, m, k]:
            k = sd.source(REC[j, m], k, breaks[m - 1])
            m -= 1
        path.append(k)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + float(U[j][i])
    return [offsets[i] for i in path], score, [float(x) for x in profile], m_end


def split_track(ref, cue_start, cue_end, keep, ratio, sample_rate, start_seconds, max_offset_samples, penalty, breaks,
                vectorised=True):
    """One track: (cue_offset list, n_segments, split_score, profile [n + 1]).  A NaN ratio or an empty window: ([0]*,
    0, NaN, NaN row).  vectorised: the tables of tests/split_wide.py and solve above; otherwise split_oracle's unit
    scores and solve_breaks."""
    import split_wide as sw
    n, L = len(cue_start), len(breaks) + 1
    dead = [0] * n, 0, math.nan, [math.nan] * L
    if math.isnan(ratio) or len(ref) == 0:
        return dead
    m, beta = sp.ref_levels(ref)
    mask = ro.rasterize(cue_start, cue_end, keep, sample_rate, start_seconds, ratio)[0] > 0
    S, R = len(mask), len(m)
    o_lo, o_hi = ao.offset_range(R, S, max_offset_samples)
    if o_lo > o_hi:
        return dead
    offsets = list(range(o_lo, o_hi + 1))
    lv = sp.levels(ratio, beta)
    runs = sp.runs_of(mask)
    units = sp.units_of(runs, S)
    if vectorised:
        path, score, profile, _ = solve(sw.unit_table(m, units, offsets, lv), offsets, penalty, breaks)
    else:
        path, score, profile, _ = solve_breaks([sp.unit_scores(m, u, offsets, lv) for u in units], offsets, penalty,
                                               breaks)
    n_seg = 1 + sum(1 for j in range(1, len(path)) if path[j] != path[j - 1])
    ends = np.array([b for _, b in runs], np.int64)
    cue_off = []
    for i in range(n):
        st = ro.scale_seconds(float(cue_start[i]), ratio)
        first = int(round((st - start_seconds) * sample_rate))
        f = min(max(slice(first, first).indices(S)[0], 0), S - 1)
        j = int(np.searchsorted(ends, f, side="right")) if len(runs) else 0   # first run ending after f
        cue_off.append(path[min(j, len(units) - 1)])
    return cue_off, n_seg, score, profile


def split_tracks(ref, ref_off, track_video, cue_start, cue_end, cue_keep, cue_off, ratio, sample_rate, start_seconds,
                 max_offset_samples, penalty, breaks, vectorised=True):
    """b2_split_tracks_breaks over T tracks: (cue_offset [cues], n_segments [T], split_score [T], split_profile
    [T, n + 1]) as numpy arrays."""
    T, L = len(cue_off) - 1, len(breaks) + 1
    co = np.zeros(int(cue_off[-1]), np.int32)
    ns = np.zeros(T, np.int32)
    sc = np.full(T, np.nan)
    pr = np.full((T, L), np.nan)
    for t in range(T):
        v = int(track_video[t])
        c0, c1 = int(cue_off[t]), int(cue_off[t + 1])
        keep = None if cue_keep is None else [bool(k) for k in cue_keep[c0:c1]]
        o, ns[t], sc[t], pr[t] = split_track(np.asarray(ref[ref_off[v]:ref_off[v + 1]], np.float64), cue_start[c0:c1],
                                             cue_end[c0:c1], keep, float(ratio[t]), sample_rate, start_seconds,
                                             max_offset_samples, penalty, breaks, vectorised)
        co[c0:c1] = o
    return co, ns, sc, pr
