"""CPU checks of the directed split (b2_split_tracks_directed: segment offsets that only grow or only shrink): the
directed restatement (tests/split_directed.py) against exhaustive enumeration of monotone paths and against
oracle/split_oracle.py at penalty +inf, its record-bit twin against it bit for bit, the record rule against the argmax
on rows full of ties, split.cuh run as the directed kernel's cluster of C CTAs (tests/host_emul/split_directed_emul.cu)
against the restatement with equal barrier counts in every CTA, and the ABI symbol."""
import itertools
import math
import os
import re
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import split_directed as sd
import split_wide as sw
from oracle import split_oracle as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host_emul", "split_directed_emul")


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


def _monotone(path, d):
    return all((b - a) * d >= 0 for a, b in zip(path, path[1:]))


@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("seed", range(24))
def test_enumeration(seed, d):
    """Up to 5 units and 9 offsets, integer scores and penalties (every sum exact): the best sum - penalty x changes
    over every path monotone in direction d is the restatement's final maximum; the returned path is monotone, attains
    it, and its split_score is its plain sum."""
    rng = np.random.RandomState(300 + seed)
    n, W = int(rng.randint(1, 6)), int(rng.randint(1, 10))
    U = _table(rng, n, W, True)
    offsets = list(range(-4, -4 + W))
    pen = float([0, 1, 2, 5][seed % 4])
    best = -math.inf
    for a in itertools.product(range(W), repeat=n):
        if not _monotone(a, d):
            continue
        ch = sum(a[j] != a[j - 1] for j in range(1, n))
        best = max(best, sum(U[j, i] for j, i in enumerate(a)) - pen * ch)
    path, score, top = sd.solve_directed([list(map(float, r)) for r in U], offsets, pen, d)
    assert top == best, (seed, d, top, best)
    assert _monotone(path, d), path
    ch = sum(path[j] != path[j - 1] for j in range(1, n))
    assert score == sum(U[j, offsets.index(o)] for j, o in enumerate(path))
    assert score - pen * ch == top, (seed, d, path, score, top)


@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("seed", range(6))
def test_enumeration_two_levels(seed, d):
    """The same on whole tracks' unit tables over two-level references (label 0.3, inexact sums): the restatement's
    maximum is the best monotone path's value computed with the programme's own rounding order, and its path attains
    it."""
    rng = np.random.RandomState(700 + seed)
    R, S = int(rng.randint(12, 30)), int(rng.randint(5, 12))
    ref = np.where(rng.rand(R) < 0.5, 1.0, 0.3)
    mask = rng.rand(S) < 0.4
    m, beta = sp.ref_levels(ref)
    units = sp.units_of(sp.runs_of(mask), S)[:5]
    offsets = list(range(-3, 6))
    U = [sp.unit_scores(m, u, offsets, sp.levels(1.0, beta)) for u in units]
    pen = [0.0, 0.3, 1.7][seed % 3]
    path, score, top = sd.solve_directed(U, offsets, pen, d)
    assert _monotone(path, d)
    n, W = len(U), len(offsets)
    vals = []
    for a in itertools.product(range(W), repeat=n):
        if not _monotone(a, d):
            continue
        v = U[0][a[0]]   # the programme's order: V_j = u_j + (V_{j-1} or V_{j-1}' - pen)
        for j in range(1, n):
            v = U[j][a[j]] + (v - pen if a[j] != a[j - 1] else v)
        vals.append(v)
    assert math.isclose(top, max(vals), rel_tol=0, abs_tol=1e-9), (top, max(vals))
    ch = sum(path[j] != path[j - 1] for j in range(1, n))
    assert math.isclose(score - pen * ch, top, rel_tol=0, abs_tol=1e-9)


@pytest.mark.parametrize("seed", range(30))
def test_vectorised_equals_plain(seed):
    """The record-bit restatement equals the argmax one bit for bit (path, score, maximum) on tables with planted
    ties, in both directions, at penalties that split and at +inf; at +inf both equal split_oracle.solve."""
    rng = np.random.RandomState(500 + seed)
    n, W = int(rng.randint(1, 12)), int(rng.randint(1, 60))
    U = _table(rng, n, W, seed % 2 == 0)
    Ul = [list(map(float, r)) for r in U]
    offsets = list(range(-7, -7 + W))
    for d in (1, -1):
        for pen in (0.0, 0.7, 1.0, 2.5, math.inf):
            want = sd.solve_directed(Ul, offsets, pen, d)
            got = sd.solve(U, offsets, pen, d)
            assert got == want, (seed, d, pen, got, want)
            assert _monotone(got[0], d)
        assert sd.solve_directed(Ul, offsets, math.inf, d)[:2] == sp.solve(Ul, offsets, math.inf)


@pytest.mark.parametrize("seed", range(40))
def test_record_rule_is_the_argmax(seed):
    """On random rows with many ties, the nearest record behind every offset is the argmax over that side with ties
    to the largest offset."""
    rng = np.random.RandomState(1100 + seed)
    W = int(rng.randint(2, 80))
    V = rng.randint(-2, 3, W).astype(np.float64)
    if seed % 3 == 0:
        V[rng.rand(W) < 0.3] = -np.inf   # never a value of the programme, but the rule holds for it too
        V[int(rng.randint(0, W))] = 0.0
    for d in (1, -1):
        rec = sd.records(V, d)
        for k in range(W):
            idx = range(0, k) if d > 0 else range(k + 1, W)
            want = sd._argmax_range(list(V), idx)
            if want is None or V[want] == -np.inf:
                continue
            assert sd.source(rec, k, d) == want, (seed, d, k)


@pytest.mark.parametrize("seed", range(8))
def test_split_tracks_identities(seed):
    """Whole tracks (rasterised cues, two-level references, skipped tracks and empty windows): the plain and the
    vectorised restatements agree bit for bit in both directions; at penalty +inf they are split_oracle.split_tracks'
    results; every cue offset path is monotone in rasterised-start order."""
    rng = np.random.RandomState(900 + seed)
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
    for d in (1, -1):
        for pen in (0.0, 2.0, math.inf):
            a = sd.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, d, vectorised=False)
            b = sd.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, d)
            for x, y in zip(a, b):
                assert np.array_equal(x, y, equal_nan=True), (seed, d, pen)
            assert b[1][2] == 0 and np.isnan(b[2][2])
            for t in range(T):
                o = b[0][off[t]:off[t + 1]]
                assert _monotone(list(o), d), (t, o)   # cue starts are sorted, so rasterised starts are too
        inf = sp.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, math.inf)
        got = sd.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, math.inf, d)
        for x, y in zip(inf, got):
            assert np.array_equal(x, y, equal_nan=True), (seed, d)


def _emulate(m, mask, o_lo, W, level, beta, pen, d, C, cta_threads, dead=False):
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<4if2d", len(m), len(mask), o_lo, W, level, beta, pen))
            f.write(np.asarray(m, np.uint8).tobytes())
            f.write(np.asarray(mask, np.uint8).tobytes())
        subprocess.check_call([EXE, fin, fout, str(d), str(C), str(cta_threads)] + (["1"] if dead else []))
        raw = open(fout, "rb").read()
    nu = struct.unpack_from("<i", raw)[0]
    mx = np.frombuffer(raw[4: 4 + 8 * nu], "<f8")
    at = 4 + 8 * nu
    arg = struct.unpack_from("<i", raw, at)[0]
    at += 4
    n_b = max(nu - 1, 0) * 2 * W
    bits = np.frombuffer(raw[at: at + n_b], np.uint8).reshape(max(nu - 1, 0), 2, W).astype(bool)
    nc = struct.unpack_from("<i", raw, at + n_b)[0]
    counts = np.frombuffer(raw[at + n_b + 4:], np.int32).reshape(nc, 2)
    return mx, arg, bits[:, 0], bits[:, 1], counts


@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("C", list(range(1, 17)))
def test_cluster_emulation_equals_restatement(C, d):
    """C CTAs of 32 to 128 threads: a window filling the CTAs, one whose last CTA owns one offset, and one whose last
    CTA owns none, over a reference with long equal stretches (equal prefix maxima in different CTAs).  Every unit's
    maximum, the last argmax, and every switch and record bit equal the vectorised programme's; every CTA runs the
    same number of CTA and cluster barriers (C = 1: the plain launch, no cluster barrier)."""
    rng = np.random.RandomState(1300 + 17 * C + (d > 0))
    nt = [32, 64, 128][C % 3]
    per_cta = 32 * nt
    R, S = int(rng.randint(C * per_cta // 2, C * per_cta + 500)), int(rng.randint(50, 300))
    label = [0.0, 0.3][C % 2]
    ref = np.where(rng.rand(R) < 0.5, 1.0, label)
    ref[: R // 2] = np.where((np.arange(R // 2) // 7) % 2 == 0, 1.0, label)   # ties across CTAs
    mask = rng.rand(S) < 0.3
    level = [1.0, np.float32(1 / (25 / 24.0))][C % 2]
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(1.0 / float(level), beta)
    units = sp.units_of(sp.runs_of(mask), S)
    widths = {C * per_cta, (C - 1) * per_cta + 1, max(1, (C - 1) * per_cta - 32 * int(rng.randint(1, nt)))}
    for W in sorted(widths):
        o_lo = int(rng.randint(-S - 10, max(-S - 9, R - W + 10)))
        offsets = np.arange(o_lo, o_lo + W)
        U = sw.unit_table(m, units, list(offsets), lv)
        for pen in (0.0, 3.0, math.inf):
            mx, arg, sws, rec, counts = _emulate(m, mask, o_lo, W, float(level), beta, pen, d, C, nt)
            M, A, SW, REC = sd.programme(U, pen, d)
            assert np.all(counts == counts[0]), (C, W, counts)
            assert counts[0][1] == (len(units) + 1 if C > 1 else 0)
            assert np.array_equal(mx, M), (C, W, pen)
            assert arg == offsets[A], (C, W, pen)
            assert np.array_equal(sws, SW[1:]), (C, W, pen)
            assert np.array_equal(rec, REC[1:]), (C, W, pen)
    _, _, _, _, counts = _emulate(m, mask, 0, 1, float(level), beta, 0.0, d, C, nt, dead=True)
    assert counts.shape == (C, 2) and not counts.any()


def test_directed_symbol_and_refusals():
    """The symbol is exported with the header's signature; a handle-less call is refused."""
    from ffsubsync_b200 import _native
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    decl = re.search(r"int b2_split_tracks_directed\((.*?)\);", header, re.S)
    assert "b2_split_tracks_directed" in _native.EXPORTS and decl
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl.group(1), flags=re.S).split(",")]
    names = [re.split(r"[\s*]+", p)[-1] for p in params]
    assert names[14:21] == ["max_offset_samples", "split_penalty", "direction", "cue_offset", "n_segments",
                            "split_score", "memspace"], names
    assert params[16].startswith("int ")
    lib = _native.load()
    assert len(lib.b2_split_tracks_directed.argtypes) == len(params) == 21
    assert lib.b2_split_tracks_directed(None, None, 1, None, 0, None, 0, None, None, None, None, None, 100, 0.0, 0,
                                        1.0, 1, None, None, None, 0) == -1


def test_batch_refuses_bad_directions():
    """BatchSynchronizer.split_tracks / split_tracks_host refuse a direction other than None, +1 and -1, and one
    combined with max_segments, before anything else."""
    from ffsubsync_b200.batch import BatchSynchronizer
    for bad in (0, 2, -2, True, 0.5, "up"):
        with pytest.raises(ValueError, match="split_direction must be"):
            BatchSynchronizer._split_direction(None, bad)
    with pytest.raises(ValueError, match="cannot be combined"):
        BatchSynchronizer._split_direction(2, 1)
    for ok in (None, 1, -1):
        BatchSynchronizer._split_direction(None, ok)
