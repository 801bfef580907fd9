"""The capped split (b2_split_tracks_capped: at most N segments per track) restated beside oracle/split_oracle.py (TEST
INFRASTRUCTURE), in plain Python floats and vectorised over the window.

The programme (DESIGN.md section 4 "K9s"): layer k = 0 .. N-1 counts the switches allowed so far,
    V_{0,k} = u_0,   V_{j,0} = u_j + V_{j-1,0},   V_{j,k}(o) = u_j(o) + max(V_{j-1,k}(o), M_{j-1,k-1} - penalty),
    M_{j,k} = max_o V_{j,k}(o)
with split_oracle's rounding (c = M - penalty, then the decision c > V, staying on a tie, then u + (c or V), each
rounded on its own), its argmax rule (the largest offset among equal maxima) and its units.  The path is the top
layer's; the profile holds M_{last,k} for every k.  numpy rounds each elementwise operation on its own as Python floats
do, so the two restatements agree bit for bit (tests/test_split_capped_cpu.py checks that).
"""
import math

import numpy as np

from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp


def solve_capped(U, offsets, penalty, N):
    """The capped programme over the unit x offset table U (Python floats).  Returns (path offsets per unit,
    split_score, profile [N])."""
    W = len(offsets)

    def argmax(x):
        best, k = -math.inf, 0
        for i in range(W):
            if x[i] >= best:   # increasing offsets: ties go to the largest
                best, k = x[i], i
        return best, k

    V = [list(U[0]) for _ in range(N)]
    dec, args = [], []   # per unit j >= 1: [layer][offset] switch; per unit j < last: [layer] argmax
    for j in range(1, len(U)):
        mk = [argmax(V[k]) for k in range(N)]
        args.append([i for _, i in mk])
        sw_j, V_next = [], []
        for k in range(N):
            if k == 0:
                sw = [False] * W
                V_next.append([U[j][i] + V[0][i] for i in range(W)])
            else:
                c = mk[k - 1][0] - penalty
                sw = [c > V[k][i] for i in range(W)]
                V_next.append([U[j][i] + (c if sw[i] else V[k][i]) for i in range(W)])
            sw_j.append(sw)
        dec.append(sw_j)
        V = V_next
    last = [argmax(V[k]) for k in range(N)]
    profile = [m for m, _ in last]
    k, i = N - 1, last[N - 1][1]
    path = [i]
    for j in range(len(U) - 1, 0, -1):
        if dec[j - 1][k][i]:
            k -= 1
            i = args[j - 1][k]
        path.append(i)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + U[j][i]
    return [offsets[i] for i in path], score, profile


def programme(U, penalty, N):
    """The capped programme vectorised over a float64 table U [units, offsets]: (M [units, N] maxima, A [units, N]
    argmax indices, SW [units, N, offsets] switch decisions, row 0 all False)."""
    U = np.asarray(U, np.float64)
    n, W = U.shape
    M, A = np.empty((n, N)), np.empty((n, N), np.int64)
    SW = np.zeros((n, N, W), bool)
    V = np.repeat(U[:1], N, axis=0)
    for j in range(n):
        if j:
            Vn = np.empty_like(V)
            Vn[0] = U[j] + V[0]
            for k in range(1, N):
                c = M[j - 1, k - 1] - penalty
                SW[j, k] = c > V[k]
                Vn[k] = U[j] + np.where(SW[j, k], c, V[k])
            V = Vn
        A[j] = W - 1 - np.argmax(V[:, ::-1], axis=1)   # ties: the largest offset
        M[j] = V[np.arange(N), A[j]]
    return M, A, SW


def solve(U, offsets, penalty, N):
    """solve_capped over a float64 table U through programme."""
    U = np.asarray(U, np.float64)
    M, A, SW = programme(U, penalty, N)
    n = len(U)
    k, i = N - 1, int(A[n - 1, N - 1])
    path = [i]
    for j in range(n - 1, 0, -1):
        if SW[j, k, i]:
            k -= 1
            i = int(A[j - 1, k])
        path.append(i)
    path = path[::-1]
    score = 0.0
    for j, i in enumerate(path):
        score = score + float(U[j][i])
    return [offsets[i] for i in path], score, [float(x) for x in M[n - 1]]


def split_track(ref, cue_start, cue_end, keep, ratio, sample_rate, start_seconds, max_offset_samples, penalty,
                max_segments, vectorised=True, brute=False):
    """One track capped at max_segments: (cue_offset list, n_segments, split_score, profile [N]).  A NaN ratio or an
    empty window: ([0]*, 0, NaN, [NaN]*N).  vectorised: the tables of tests/split_wide.py and solve above; otherwise
    split_oracle's unit scores (brute: per-frame enumeration) and solve_capped."""
    import split_wide as sw
    n, N = len(cue_start), max_segments
    dead = ([0] * n, 0, math.nan, [math.nan] * N)
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
        path, score, profile = solve(sw.unit_table(m, units, offsets, lv), offsets, penalty, N)
    else:
        if brute:
            U = [[sp.unit_score_brute(m, mask, u, o, lv) for o in offsets] for u in units]
        else:
            U = [sp.unit_scores(m, u, offsets, lv) for u in units]
        path, score, profile = solve_capped(U, offsets, penalty, N)
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
                 max_offset_samples, penalty, max_segments, vectorised=True):
    """b2_split_tracks_capped over T tracks: (cue_offset [cues], n_segments [T], split_score [T],
    split_profile [T, N]) as numpy arrays."""
    T, N = len(cue_off) - 1, max_segments
    co = np.zeros(int(cue_off[-1]), np.int32)
    ns = np.zeros(T, np.int32)
    sc = np.full(T, np.nan)
    pr = np.full((T, N), np.nan)
    for t in range(T):
        v = int(track_video[t])
        c0, c1 = int(cue_off[t]), int(cue_off[t + 1])
        keep = None if cue_keep is None else [bool(k) for k in cue_keep[c0:c1]]
        o, ns[t], sc[t], pr[t] = split_track(np.asarray(ref[ref_off[v]:ref_off[v + 1]], np.float64), cue_start[c0:c1],
                                             cue_end[c0:c1], keep, float(ratio[t]), sample_rate, start_seconds,
                                             max_offset_samples, penalty, N, vectorised)
        co[c0:c1] = o
    return co, ns, sc, pr
