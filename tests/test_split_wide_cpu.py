"""CPU checks of the wide per-segment split (b2_split_tracks_wide): the vectorised oracle (tests/split_wide.py) against
oracle/split_oracle.py bit for bit, split.cuh run as a cluster of 1 to 16 CTAs (tests/host_emul/split_cluster_emul.cu)
against the oracle with equal barrier counts in every CTA, and the ABI symbol."""
import math
import os
import re
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import split_wide as sw
from oracle import split_oracle as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host_emul", "split_cluster_emul")


def _tie_table(rng, n, W, integer):
    """A unit x offset table with planted ties: repeated values inside and across units."""
    if integer:
        U = rng.randint(-3, 4, (n, W)).astype(np.float64)
    else:
        U = np.round(rng.uniform(-2, 2, (n, W)), 1) * 0.7   # few distinct, inexact values
    for j in range(n):   # the row maximum at several offsets
        k = rng.choice(W, size=min(W, 3), replace=False)
        U[j, k] = U[j].max()
    return U


@pytest.mark.parametrize("seed", range(30))
def test_vectorised_solve_equals_solve(seed):
    rng = np.random.RandomState(500 + seed)
    n, W = int(rng.randint(1, 12)), int(rng.randint(1, 60))
    U = _tie_table(rng, n, W, seed % 2 == 0)
    offsets = list(range(-int(rng.randint(0, 30)), 0))
    offsets = list(range(offsets[0] if offsets else 0, (offsets[0] if offsets else 0) + W))
    for pen in (0.0, 0.7, 1.0, 2.5, math.inf):
        want = sp.solve([list(map(float, r)) for r in U], offsets, pen)
        got = sw.solve(U, offsets, pen)
        assert got[0] == want[0] and got[1] == want[1], (seed, pen, got, want)


@pytest.mark.parametrize("seed", range(12))
def test_unit_table_equals_unit_scores(seed):
    rng = np.random.RandomState(700 + seed)
    R, S = int(rng.randint(1, 300)), int(rng.randint(2, 300))
    label = [0.0, 0.3, -0.5][seed % 3]
    ratio = [1.0, 25 / 24.0][seed % 2]
    ref = np.where(rng.rand(R) < 0.5, 1.0, label)
    mask = rng.rand(S) < [0.1, 0.5, 0.9][seed % 3]
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(ratio, beta)
    units = sp.units_of(sp.runs_of(mask), S)
    offsets = list(range(-S - 5, R + 5))
    U = sw.unit_table(m, units, offsets, lv)
    for j, u in enumerate(units):
        want = sp.unit_scores(m, u, offsets, lv)
        assert [float(x) for x in U[j]] == want, (seed, j)


@pytest.mark.parametrize("seed", range(8))
def test_vectorised_split_tracks_equals_oracle(seed):
    rng = np.random.RandomState(900 + seed)
    label = [0.0, 0.3][seed % 2]
    refs = [np.where(rng.rand(int(rng.randint(200, 900))) < 0.4, 1.0, label) for _ in range(2)]
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])])
    ref = np.concatenate(refs)
    T = 4
    cs, ce, off = [], [], [0]
    for t in range(T):
        k = int(rng.randint(0, 9))
        a = np.sort(np.round(rng.uniform(0, 6, k), 2))
        cs.append(a)
        ce.append(np.round(a + rng.uniform(0.01, 0.8, k), 2))
        off.append(off[-1] + k)
    cs, ce = np.concatenate(cs), np.concatenate(ce)
    keep = (rng.rand(len(cs)) > 0.2).astype(np.uint8)
    ratio = np.array([1.0, 25 / 24.0, np.nan, 24 / 25.0])
    tv = np.array([0, 1, 1, 0])
    mos = [None, 150, 7, 400][seed % 4]
    for pen in (0.0, 2.0, math.inf):
        want = sp.split_tracks(ref, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen)
        got = sw.split_tracks(ref, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen)
        for w, g in zip(want, got):
            assert np.array_equal(w, g, equal_nan=True), (seed, pen, w, g)


def _emulate_cluster(m, mask, o_lo, W, level, beta, pen, C, cta_threads, dead=False):
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<4if2d", len(m), len(mask), o_lo, W, level, beta, pen))
            f.write(np.asarray(m, np.uint8).tobytes())
            f.write(np.asarray(mask, np.uint8).tobytes())
        subprocess.check_call([EXE, fin, fout, str(C), str(cta_threads)] + (["1"] if dead else []))
        raw = open(fout, "rb").read()
    nu = struct.unpack_from("<i", raw)[0]
    mx, args = [], []
    for j in range(nu):
        a, b = struct.unpack_from("<di", raw, 4 + 12 * j)
        mx.append(a)
        args.append(b)
    at = 4 + 12 * nu
    n_sw = max(nu - 1, 0) * W
    switches = np.frombuffer(raw[at: at + n_sw], np.uint8).reshape(max(nu - 1, 0), W)
    c = struct.unpack_from("<i", raw, at + n_sw)[0]
    counts = np.frombuffer(raw[at + n_sw + 4:], np.int32).reshape(c, 2)
    return mx, args, switches, counts


@pytest.mark.parametrize("C", range(1, 17))
def test_cluster_emulation_equals_oracle(C):
    """C CTAs of 32 to 128 threads: a window filling the cluster, one whose last CTA owns one offset, and one whose
    last CTA owns none.  Every unit's maximum and argmax and every switch bit equal the vectorised oracle's programme,
    and every CTA runs the same number of CTA and cluster barriers."""
    rng = np.random.RandomState(1100 + C)
    nt = [32, 64, 128][C % 3]
    per_cta = 32 * nt
    R, S = int(rng.randint(C * per_cta // 2, C * per_cta + 500)), int(rng.randint(50, 400))
    label = [0.0, 0.3][C % 2]
    ref = np.where(rng.rand(R) < 0.5, 1.0, label)
    # a periodic stretch: exact ties between offsets that sit in different CTAs
    ref[: R // 2] = np.where((np.arange(R // 2) // 7) % 2 == 0, 1.0, label)
    mask = rng.rand(S) < 0.3
    level = [1.0, np.float32(1 / (25 / 24.0))][C % 2]
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(1.0 / float(level), beta)
    units = sp.units_of(sp.runs_of(mask), S)
    widths = {C * per_cta, (C - 1) * per_cta + 1, max(1, (C - 1) * per_cta - 32 * int(rng.randint(1, nt)))}
    for W in sorted(widths):
        o_lo = int(rng.randint(-S - 10, max(-S - 9, R - W + 10)))
        offsets = list(range(o_lo, o_lo + W))
        U = sw.unit_table(m, units, offsets, lv)
        for pen in (0.0, 3.0, math.inf):
            mx, args, switches, counts = _emulate_cluster(m, mask, o_lo, W, float(level), beta, pen, C, nt)
            assert len(mx) == len(units)
            assert np.all(counts == counts[0]), (C, W, counts)
            assert counts[0][1] == len(units) + 1
            V = U[0].copy()
            for j in range(len(units)):
                if j:
                    c = pmx - pen
                    want_sw = c > V
                    assert np.array_equal(switches[j - 1].astype(bool), want_sw), (C, W, pen, j)
                    V = U[j] + np.where(want_sw, c, V)
                k = W - 1 - int(np.argmax(V[::-1]))
                pmx = float(V[k])
                assert mx[j] == pmx and args[j] == offsets[k], (C, W, pen, j, mx[j], pmx, args[j], offsets[k])
    # the skipped track: every CTA leaves before its first barrier
    _, _, _, counts = _emulate_cluster(m, mask, 0, 1, float(level), beta, 0.0, C, nt, dead=True)
    assert counts.shape == (C, 2) and not counts.any()


def test_wide_symbol_and_handleless_refusal():
    from ffsubsync_b200 import _native
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    assert "b2_split_tracks_wide" in _native.EXPORTS and re.search(r"\bb2_split_tracks_wide\s*\(", header)
    lib = _native.load()
    assert lib.b2_split_tracks_wide(None, None, 1, None, 0, None, 0, None, None, None, None, None, 100, 0.0, 0, 1.0,
                                    None, None, None, 0) == -1
