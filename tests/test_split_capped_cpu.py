"""CPU checks of the capped split (b2_split_tracks_capped: at most N segments per track): the capped oracle
(tests/split_capped.py) against exhaustive enumeration and against oracle/split_oracle.py, its vectorised twin against
it bit for bit, split.cuh run as the capped kernel's cluster of N x C CTAs (tests/host_emul/split_capped_emul.cu)
against the oracle with equal barrier counts in every CTA, and the ABI symbol."""
import itertools
import math
import os
import re
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import split_capped as sc
import split_wide as sw
from oracle import split_oracle as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host_emul", "split_capped_emul")


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


@pytest.mark.parametrize("seed", range(24))
def test_enumeration(seed):
    """Up to 5 units and 9 offsets, integer scores and penalties (every sum exact): the best sum - penalty x changes
    over every assignment with at most n - 1 changes is profile[n - 1] for every n <= N; the returned path attains
    profile[N - 1] with at most N segments, and its split_score is its plain sum."""
    rng = np.random.RandomState(300 + seed)
    n, W = int(rng.randint(1, 6)), int(rng.randint(1, 10))
    U = _table(rng, n, W, True)
    offsets = list(range(-4, -4 + W))
    pen = float([0, 1, 2, 5][seed % 4])
    best = {}   # changes -> best penalised sum
    for a in itertools.product(range(W), repeat=n):
        ch = sum(a[j] != a[j - 1] for j in range(1, n))
        val = sum(U[j, i] for j, i in enumerate(a)) - pen * ch
        best[ch] = max(best.get(ch, -math.inf), val)
    for N in range(1, 6):
        path, score, profile = sc.solve_capped([list(map(float, r)) for r in U], offsets, pen, N)
        for m in range(1, N + 1):
            assert profile[m - 1] == max(v for ch, v in best.items() if ch <= m - 1), (seed, N, m, profile, best)
        ch = sum(path[j] != path[j - 1] for j in range(1, n))
        assert ch + 1 <= N
        assert score == sum(U[j, offsets.index(o)] for j, o in enumerate(path))
        assert score - pen * ch == profile[N - 1], (seed, N, path, score, profile)


@pytest.mark.parametrize("seed", range(30))
def test_vectorised_equals_plain(seed):
    rng = np.random.RandomState(500 + seed)
    n, W = int(rng.randint(1, 12)), int(rng.randint(1, 60))
    U = _table(rng, n, W, seed % 2 == 0)
    offsets = list(range(-7, -7 + W))
    for N in (1, 2, 3, 7, 16):
        for pen in (0.0, 0.7, 1.0, 2.5, math.inf):
            want = sc.solve_capped([list(map(float, r)) for r in U], offsets, pen, N)
            got = sc.solve(U, offsets, pen, N)
            assert got[0] == want[0] and got[1] == want[1] and got[2] == want[2], (seed, N, pen, got, want)


@pytest.mark.parametrize("seed", range(20))
def test_oracle_identities(seed):
    """On tables: N >= units gives split_oracle.solve's path and score, with profile[N - 1] its maximum; N = 1 gives
    solve at penalty +inf; the profile never decreases; at most N segments."""
    rng = np.random.RandomState(800 + seed)
    n, W = int(rng.randint(1, 10)), int(rng.randint(1, 40))
    U = [list(map(float, r)) for r in _table(rng, n, W, seed % 3 != 0)]
    offsets = list(range(3, 3 + W))
    for pen in (0.0, 1.5, 4.0, math.inf):
        want = sp.solve(U, offsets, pen)
        for N in (n, n + 1, 16):
            if N > 16:
                continue
            path, score, profile = sc.solve_capped(U, offsets, pen, N)
            assert (path, score) == want, (seed, pen, N)
        inf = sp.solve(U, offsets, math.inf)
        path, score, profile = sc.solve_capped(U, offsets, pen, 1)
        assert (path, score) == inf and len(set(path)) == 1
        for N in (2, 3, 5):
            path, _, profile = sc.solve_capped(U, offsets, pen, N)
            assert all(profile[k] <= profile[k + 1] for k in range(N - 1)), profile
            assert 1 + sum(path[j] != path[j - 1] for j in range(1, n)) <= N


@pytest.mark.parametrize("seed", range(8))
def test_split_tracks_identities(seed):
    """Whole tracks (rasterised cues, two-level references, skipped tracks and empty windows): the plain and the
    vectorised capped oracle agree bit for bit; with N at least every track's unit count the results are
    split_oracle.split_tracks'; N = 1 gives its results at penalty +inf; dead tracks get a NaN profile."""
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
    for pen in (0.0, 2.0, math.inf):
        a = sc.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, 3, vectorised=False)
        b = sc.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, 3)
        for x, y in zip(a, b):
            assert np.array_equal(x, y, equal_nan=True), (seed, pen)
        assert np.all(np.isnan(b[3][2])) and b[1][2] == 0
        full = sc.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, 16)
        want = sp.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen)
        for x, y in zip(want, full[:3]):
            assert np.array_equal(x, y, equal_nan=True), (seed, pen)
        one = sc.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, 1)
        inf = sp.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, math.inf)
        for x, y in zip(inf, one[:3]):
            assert np.array_equal(x, y, equal_nan=True), (seed, pen)


def test_brute_units():
    """The plain oracle's brute-force unit scores give the same capped results as the frame sums."""
    rng = np.random.RandomState(4)
    ref = np.where(rng.rand(150) < 0.5, 1.0, 0.3)
    cs = np.array([0.2, 0.5, 0.9])
    ce = cs + 0.15
    for N in (1, 2, 3):
        a = sc.split_track(ref, cs, ce, None, 1.0, 100, 0.0, 20, 0.5, N, vectorised=False)
        b = sc.split_track(ref, cs, ce, None, 1.0, 100, 0.0, 20, 0.5, N, vectorised=False, brute=True)
        assert a == b


def _emulate(m, mask, o_lo, W, level, beta, pen, N, C, cta_threads, dead=False):
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<4if2d", len(m), len(mask), o_lo, W, level, beta, pen))
            f.write(np.asarray(m, np.uint8).tobytes())
            f.write(np.asarray(mask, np.uint8).tobytes())
        subprocess.check_call([EXE, fin, fout, str(N), str(C), str(cta_threads)] + (["1"] if dead else []))
        raw = open(fout, "rb").read()
    nu = struct.unpack_from("<i", raw)[0]
    rec = np.frombuffer(raw[4: 4 + 12 * nu * N], np.dtype([("mx", "<f8"), ("arg", "<i4")]))
    mx, args = rec["mx"].reshape(nu, N), rec["arg"].reshape(nu, N)
    at = 4 + 12 * nu * N
    n_sw = max(nu - 1, 0) * N * W
    switches = np.frombuffer(raw[at: at + n_sw], np.uint8).reshape(max(nu - 1, 0), N, W)
    nc = struct.unpack_from("<i", raw, at + n_sw)[0]
    counts = np.frombuffer(raw[at + n_sw + 4:], np.int32).reshape(nc, 2)
    return mx, args, switches, counts


LAYOUTS = [(1, 1), (2, 1), (3, 1), (16, 1), (1, 2), (2, 2), (8, 2), (3, 3), (4, 4), (5, 3), (2, 8), (1, 16)]


@pytest.mark.parametrize("N,C", LAYOUTS, ids=lambda x: str(x))
def test_cluster_emulation_equals_oracle(N, C):
    """N layers x C parts of 32 to 128 threads: a window filling the parts, one whose last part owns one offset, and
    one whose last part owns none.  Every layer's unit maximum and argmax and every switch bit equal the vectorised
    programme's, and every CTA runs the same number of CTA and cluster barriers."""
    rng = np.random.RandomState(1300 + 17 * N + C)
    nt = [32, 64, 128][(N + C) % 3]
    per_cta = 32 * nt
    R, S = int(rng.randint(C * per_cta // 2, C * per_cta + 500)), int(rng.randint(50, 300))
    label = [0.0, 0.3][C % 2]
    ref = np.where(rng.rand(R) < 0.5, 1.0, label)
    ref[: R // 2] = np.where((np.arange(R // 2) // 7) % 2 == 0, 1.0, label)   # ties across parts
    mask = rng.rand(S) < 0.3
    level = [1.0, np.float32(1 / (25 / 24.0))][(N + C) % 2]
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(1.0 / float(level), beta)
    units = sp.units_of(sp.runs_of(mask), S)
    widths = {C * per_cta, (C - 1) * per_cta + 1, max(1, (C - 1) * per_cta - 32 * int(rng.randint(1, nt)))}
    for W in sorted(widths):
        o_lo = int(rng.randint(-S - 10, max(-S - 9, R - W + 10)))
        offsets = list(range(o_lo, o_lo + W))
        U = sw.unit_table(m, units, offsets, lv)
        for pen in (0.0, 3.0, math.inf):
            mx, args, switches, counts = _emulate(m, mask, o_lo, W, float(level), beta, pen, N, C, nt)
            M, A, SW = sc.programme(U, pen, N)
            assert np.all(counts == counts[0]), (N, C, W, counts)
            assert counts[0][1] == len(units) + 1
            assert np.array_equal(mx, M), (N, C, W, pen)
            assert np.array_equal(args, np.asarray(offsets)[A]), (N, C, W, pen)
            assert np.array_equal(switches.astype(bool), SW[1:]), (N, C, W, pen)
    _, _, _, counts = _emulate(m, mask, 0, 1, float(level), beta, 0.0, N, C, nt, dead=True)
    assert counts.shape == (N * C, 2) and not counts.any()


def test_capped_symbol_and_refusals():
    """The symbol is exported with the header's signature; a handle-less call is refused."""
    from ffsubsync_b200 import _native
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    decl = re.search(r"int b2_split_tracks_capped\((.*?)\);", header, re.S)
    assert "b2_split_tracks_capped" in _native.EXPORTS and decl
    params = [p.strip() for p in re.sub(r"/\*.*?\*/", "", decl.group(1), flags=re.S).split(",")]
    names = [re.split(r"[\s*]+", p)[-1] for p in params]
    assert names[14:22] == ["max_offset_samples", "split_penalty", "max_segments", "cue_offset", "n_segments",
                            "split_score", "split_profile", "memspace"], names
    assert params[16].startswith("int ") and params[20].startswith("double*")
    lib = _native.load()
    assert len(lib.b2_split_tracks_capped.argtypes) == len(params) == 22
    assert lib.b2_split_tracks_capped(None, None, 1, None, 0, None, 0, None, None, None, None, None, 100, 0.0, 0, 1.0,
                                      2, None, None, None, None, 0) == -1
