"""CPU checks of the split along stated breaks (b2_split_tracks_breaks): the restatement (tests/split_breaks.py) against
exhaustive enumeration of the paths that follow the pattern at every exact break count, its record-bit twin against it
bit for bit, penalty +inf against oracle/split_oracle.py, uniform patterns against the directed restatement
(tests/split_directed.py), split.cuh run as the kernel's cluster of C CTAs for every (n, offsets per thread, C) layout
(tests/host_emul/split_breaks_emul.cu) with equal barrier counts in every CTA, the ABI symbol, and the Python
refusals."""
import itertools
import math
import os
import re
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import split_breaks as sb
import split_directed as sd
import split_wide as sw
from oracle import split_oracle as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host_emul", "split_breaks_emul")


def _table(rng, n, W, integer):
    """A unit x offset table with planted ties: repeated values inside and across units."""
    if integer:
        U = rng.randint(-3, 4, (n, W)).astype(np.float64)
    else:
        U = np.round(rng.uniform(-2, 2, (n, W)), 1) * 0.7   # few distinct, inexact values
    for j in range(n):
        k = rng.choice(W, size=min(W, 2), replace=False)
        U[j, k] = U[j].max()
    return U


def _pattern(rng, n):
    return tuple(int(x) for x in rng.choice([1, -1], n))


def _breaks_of(path):
    """The signs of the path's breaks, in track order."""
    return [1 if b > a else -1 for a, b in zip(path, path[1:]) if b != a]


def _follows(path, breaks):
    s = _breaks_of(path)
    return len(s) <= len(breaks) and all(x == d for x, d in zip(s, breaks))


def _pattern_paths(n, W, breaks):
    for a in itertools.product(range(W), repeat=n):
        if _follows(a, breaks):
            yield a


@pytest.mark.parametrize("seed", range(40))
def test_enumeration(seed):
    """Up to 5 units and 9 offsets, patterns of 1 to 3 breaks with mixed signs, integer scores and penalties (every
    sum exact): profile[m] is the best sum - penalty x m over the paths with exactly m breaks following d_1 .. d_m (-inf
    when there is none); the returned path follows the pattern, ends at the best layer, and its split_score is its
    plain sum."""
    rng = np.random.RandomState(2100 + seed)
    n, W = int(rng.randint(1, 6)), int(rng.randint(1, 10))
    breaks = _pattern(rng, int(rng.randint(1, 4)))
    U = _table(rng, n, W, True)
    offsets = list(range(-4, -4 + W))
    pen = float([0, 1, 2, 5][seed % 4])
    best = [-math.inf] * (len(breaks) + 1)
    for a in _pattern_paths(n, W, breaks):
        m = len(_breaks_of(a))
        best[m] = max(best[m], sum(U[j, i] for j, i in enumerate(a)) - pen * m)
    path, score, profile, m_end = sb.solve_breaks([list(map(float, r)) for r in U], offsets, pen, breaks)
    assert profile == best, (seed, breaks, profile, best)
    assert _follows(path, breaks), (path, breaks)
    m = len(_breaks_of(path))
    assert m == m_end and profile[m] == max(profile)
    assert score == sum(U[j, offsets.index(o)] for j, o in enumerate(path))
    assert score - pen * m == profile[m], (seed, path, score, profile)


@pytest.mark.parametrize("seed", range(8))
def test_enumeration_two_levels(seed):
    """The same on whole tracks' unit tables over two-level references (label 0.3, inexact sums): each profile entry
    is the best pattern-following path's value at that break count, computed with the programme's own rounding order,
    and the returned path attains the largest."""
    rng = np.random.RandomState(2300 + seed)
    R, S = int(rng.randint(12, 30)), int(rng.randint(5, 12))
    ref = np.where(rng.rand(R) < 0.5, 1.0, 0.3)
    mask = rng.rand(S) < 0.4
    m, beta = sp.ref_levels(ref)
    units = sp.units_of(sp.runs_of(mask), S)[:5]
    offsets = list(range(-3, 6))
    U = [sp.unit_scores(m, u, offsets, sp.levels(1.0, beta)) for u in units]
    pen = [0.0, 0.3, 1.7][seed % 3]
    breaks = _pattern(rng, 1 + seed % 3)
    path, score, profile, m_end = sb.solve_breaks(U, offsets, pen, breaks)
    assert _follows(path, breaks)
    n, W = len(U), len(offsets)
    best = [-math.inf] * (len(breaks) + 1)
    for a in _pattern_paths(n, W, breaks):
        v = U[0][a[0]]   # the programme's order: V_j = u_j + (V_{j-1} or P - pen)
        for j in range(1, n):
            v = U[j][a[j]] + (v - pen if a[j] != a[j - 1] else v)
        k = len(_breaks_of(a))
        best[k] = max(best[k], v)
    for x, y in zip(profile, best):
        assert (x == y == -math.inf) or math.isclose(x, y, rel_tol=0, abs_tol=1e-9), (profile, best)
    assert math.isclose(score - pen * m_end, max(profile), rel_tol=0, abs_tol=1e-9)


@pytest.mark.parametrize("seed", range(30))
def test_vectorised_equals_plain(seed):
    """The record-bit restatement equals the argmax one bit for bit (path, score, profile, end layer) on tables with
    planted ties, patterns of 1 to 6 mixed breaks, at penalties that split and at +inf; at +inf both equal
    split_oracle.solve, with profile[0] its maximum and every other column -inf."""
    rng = np.random.RandomState(2500 + seed)
    n, W = int(rng.randint(1, 12)), int(rng.randint(1, 60))
    U = _table(rng, n, W, seed % 2 == 0)
    Ul = [list(map(float, r)) for r in U]
    offsets = list(range(-7, -7 + W))
    for breaks in (_pattern(rng, 1), _pattern(rng, 2), _pattern(rng, int(rng.randint(3, 7)))):
        for pen in (0.0, 0.7, 1.0, 2.5, math.inf):
            want = sb.solve_breaks(Ul, offsets, pen, breaks)
            got = sb.solve(U, offsets, pen, breaks)
            assert got == want, (seed, breaks, pen, got, want)
            assert _follows(got[0], breaks)
        inf = sb.solve_breaks(Ul, offsets, math.inf, breaks)
        assert tuple(inf[:2]) == tuple(sp.solve(Ul, offsets, math.inf))
        assert np.isfinite(inf[2][0]) and all(x == -math.inf for x in inf[2][1:]) and inf[3] == 0


def _value(U, a, pen):
    v = U[0][a[0]]
    for j in range(1, len(a)):
        v = U[j][a[j]] + (v - pen if a[j] != a[j - 1] else v)
    return v


@pytest.mark.parametrize("seed", range(30))
def test_uniform_pattern_equals_directed(seed):
    """A uniform pattern (d,) * n on a table of at most n + 1 units: the largest profile entry is the directed
    programme's optimum bit for bit, and where that optimum is attained by one path only the paths and scores are the
    same.  Integer tables (enumerated) and inexact ones (compared)."""
    rng = np.random.RandomState(2700 + seed)
    n_b = int(rng.randint(1, 5))
    d = [1, -1][seed % 2]
    n = int(rng.randint(1, n_b + 2))
    W = int(rng.randint(1, 8))
    U = _table(rng, n, W, seed % 3 != 0)
    Ul = [list(map(float, r)) for r in U]
    offsets = list(range(W))
    for pen in (0.0, 1.0, 3.0, math.inf):
        path, score, profile, _ = sb.solve(U, offsets, pen, (d,) * n_b)
        dpath, dscore, top = sd.solve_directed(Ul, offsets, pen, d)
        assert max(profile) == top, (seed, pen, profile, top)
        attain = [a for a in itertools.product(range(W), repeat=n)
                  if all((b - x) * d >= 0 for x, b in zip(a, a[1:])) and _value(Ul, a, pen) == top]
        if len(attain) == 1:
            assert (path, score) == (dpath, dscore), (seed, pen)


@pytest.mark.parametrize("seed", range(8))
def test_split_tracks_identities(seed):
    """Whole tracks (rasterised cues, two-level references, skipped tracks and empty windows): the plain and the
    vectorised restatements agree bit for bit; at penalty +inf they are split_oracle.split_tracks' results with
    profile[:, 0] finite and the other columns -inf on live tracks, NaN rows on dead ones."""
    rng = np.random.RandomState(2900 + seed)
    label = [0.0, 0.3][seed % 2]
    refs = [np.where(rng.rand(int(rng.randint(200, 700))) < 0.4, 1.0, label) for _ in range(2)]
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])])
    ref = np.concatenate(refs)
    T = 4
    cs, ce, off = [], [], [0]
    for t in range(T):
        k = int(rng.randint(0, 5))
        a = np.sort(np.round(rng.uniform(0, 5, k), 2))
        cs.append(a)
        ce.append(np.round(a + rng.uniform(0.01, 0.8, k), 2))
        off.append(off[-1] + k)
    cs, ce = np.concatenate(cs), np.concatenate(ce)
    ratio = np.array([1.0, 25 / 24.0, np.nan, 24 / 25.0])
    tv = np.array([0, 1, 1, 0])
    mos = [None, 150, 7, 60][seed % 4]
    breaks = [(-1,), (1, 1, 1), (-1, 1), (1, -1, -1, 1)][seed % 4]
    for pen in (0.0, 2.0, math.inf):
        a = sb.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, breaks, vectorised=False)
        b = sb.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, breaks)
        for x, y in zip(a, b):
            assert np.array_equal(x, y, equal_nan=True), (seed, pen)
        assert b[1][2] == 0 and np.isnan(b[2][2]) and np.all(np.isnan(b[3][2]))
    inf = sp.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, math.inf)
    got = sb.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, math.inf, breaks)
    for x, y in zip(inf, got[:3]):
        assert np.array_equal(x, y, equal_nan=True), seed
    live = got[1] > 0
    assert np.all(np.isfinite(got[3][live, 0])) and np.all(got[3][live, 1:] == -np.inf)


def _emulate(m, mask, o_lo, W, breaks, level, beta, pen, C, cta_threads, dead=False):
    nb = len(breaks)
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<5i", len(m), len(mask), o_lo, W, nb))
            f.write(np.asarray(breaks, np.int32).tobytes())
            f.write(struct.pack("<f2d", level, beta, pen))
            f.write(np.asarray(m, np.uint8).tobytes())
            f.write(np.asarray(mask, np.uint8).tobytes())
        subprocess.check_call([EXE, fin, fout, str(C), str(cta_threads)] + (["1"] if dead else []))
        raw = open(fout, "rb").read()
    nu, kM = struct.unpack_from("<2i", raw)
    at = 8
    L = nb + 1
    prof = arg = None
    if nu > 0:
        prof = np.frombuffer(raw[at: at + 8 * L], "<f8")
        arg = np.frombuffer(raw[at + 8 * L: at + 12 * L], "<i4")
        at += 12 * L
    n_b = max(nu - 1, 0) * nb * 2 * W
    bits = np.frombuffer(raw[at: at + n_b], np.uint8).reshape(max(nu - 1, 0), nb, 2, W).astype(bool)
    nc = struct.unpack_from("<i", raw, at + n_b)[0]
    counts = np.frombuffer(raw[at + n_b + 4:], np.int32).reshape(nc, 2)
    return kM, prof, arg, bits[:, :, 0], bits[:, :, 1], counts


@pytest.mark.parametrize("C", list(range(1, 17)))
@pytest.mark.parametrize("nb", list(range(1, 16)))
def test_cluster_emulation_equals_restatement(nb, C):
    """Every layout of the kernel: n = 1 .. 15 breaks (32 / (n + 1) offsets a thread) on C = 1 .. 16 CTAs of 32 or 64
    threads; a window filling the CTAs and one whose last CTA owns a single offset, over a reference with long equal
    stretches (equal prefix maxima in different CTAs) and a mixed pattern.  Every layer's last maximum and argmax, and
    every switch and record bit, equal the vectorised programme's; every CTA runs the same number of CTA and cluster
    barriers."""
    rng = np.random.RandomState(3100 + 17 * nb + C)
    nt = [32, 64][(nb + C) % 2]
    kM = 32 // (nb + 1)
    per_cta = kM * nt
    breaks = _pattern(rng, nb)
    R, S = int(rng.randint(C * per_cta // 2 + 60, C * per_cta + 300)), int(rng.randint(40, 160))
    label = [0.0, 0.3][C % 2]
    ref = np.where(rng.rand(R) < 0.5, 1.0, label)
    ref[: R // 2] = np.where((np.arange(R // 2) // 7) % 2 == 0, 1.0, label)   # ties across CTAs
    mask = rng.rand(S) < 0.3
    level = [1.0, np.float32(1 / (25 / 24.0))][nb % 2]
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(1.0 / float(level), beta)
    units = sp.units_of(sp.runs_of(mask), S)
    for W in sorted({C * per_cta, (C - 1) * per_cta + 1}):
        o_lo = int(rng.randint(-S - 10, max(-S - 9, R - W + 10)))
        offsets = np.arange(o_lo, o_lo + W)
        U = sw.unit_table(m, units, list(offsets), lv)
        for pen in (0.0, 3.0, math.inf):
            k, prof, arg, sws, rec, counts = _emulate(m, mask, o_lo, W, breaks, float(level), beta, pen, C, nt)
            P, _, SW, REC = sb.programme(U, pen, breaks)
            args = W - 1 - np.argmax(np.asarray(_last_rows(U, pen, breaks))[:, ::-1], axis=1)
            assert k == kM
            assert np.all(counts == counts[0]), (nb, C, W, counts)
            assert counts[0][1] == len(units) + 1
            assert np.array_equal(prof, P), (nb, C, W, pen)
            assert np.array_equal(arg, offsets[args]), (nb, C, W, pen)
            assert np.array_equal(sws, SW[1:, 1:]), (nb, C, W, pen)
            assert np.array_equal(rec, REC[1:, 1:]), (nb, C, W, pen)
    *_, counts = _emulate(m, mask, 0, 1, breaks, float(level), beta, 0.0, C, nt, dead=True)
    assert counts.shape == (C, 2) and not counts.any()


def _last_rows(U, pen, breaks):
    """The last unit's rows V_{last,m} of the programme (the vectorised restatement's recurrence)."""
    U = np.asarray(U, np.float64)
    L = len(breaks) + 1
    V = np.full((L, U.shape[1]), -np.inf)
    V[0] = U[0]
    for j in range(1, len(U)):
        Vn = np.empty_like(V)
        Vn[0] = U[j] + V[0]
        for m in range(1, L):
            c = sd.prefix(V[m - 1], breaks[m - 1]) - pen
            Vn[m] = U[j] + np.where(c > V[m], c, V[m])
        V = Vn
    return V


def test_breaks_symbol_and_refusals():
    """The symbol is exported with the header's signature; a handle-less call is refused."""
    from ffsubsync_b200 import _native
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    decl = re.search(r"int b2_split_tracks_breaks\((.*?)\);", header, re.S)
    assert "b2_split_tracks_breaks" in _native.EXPORTS and decl
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl.group(1), flags=re.S).split(",")]
    names = [re.split(r"[\s*]+", p)[-1] for p in params]
    assert names[14:23] == ["max_offset_samples", "split_penalty", "breaks", "n_breaks", "cue_offset", "n_segments",
                            "split_score", "split_profile", "memspace"], names
    assert params[16].startswith("const int32_t*") and params[17].startswith("int ")
    lib = _native.load()
    assert len(lib.b2_split_tracks_breaks.argtypes) == len(params) == 23
    assert lib.b2_split_tracks_breaks(None, None, 1, None, 0, None, 0, None, None, None, None, None, 100, 0.0, 0,
                                      1.0, None, 1, None, None, None, None, 0) == -1


def test_batch_refuses_bad_breaks():
    """BatchSynchronizer.split_tracks / split_tracks_host refuse an empty sequence, bools, entries other than +-1, a
    non-sequence, and split_breaks with max_segments or split_direction, before anything else; good patterns come
    back as tuples of ints."""
    from ffsubsync_b200.batch import BatchSynchronizer
    f = BatchSynchronizer._split_breaks
    assert f(None, None, None) is None
    assert f(None, None, [-1]) == (-1,)
    assert f(None, None, np.array([1, 1, -1])) == (1, 1, -1)
    for bad in ([0], [2], [1, -2], [True], [1, False], [0.5], ["up"], [1.0], np.array([True])):
        with pytest.raises(ValueError, match="entries must be"):
            f(None, None, bad)
    for bad in (1, -1, "+1", b"\x01"):
        with pytest.raises(ValueError, match="must be a sequence"):
            f(None, None, bad)
    for empty in ([], ()):
        with pytest.raises(ValueError, match="at least one break"):
            f(None, None, empty)
    with pytest.raises(ValueError, match="cannot be combined"):
        f(2, None, (1,))
    with pytest.raises(ValueError, match="cannot be combined"):
        f(None, -1, (-1,))
