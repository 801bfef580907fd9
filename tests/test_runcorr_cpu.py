"""The run path's arithmetic (csrc/runcorr.cuh) run thread by thread on the CPU
(tests/host_emul/runcorr_emul.cu) against the exact correlation at every offset of the window.

The exact score is built from integer counts with rational arithmetic, so the check is the bound
itself: |run score - exact| must stay within eps / 2 (eps is the nomination margin of
runcorr.cuh, which also covers the re-score's own float64 error), and for +-1 signals (level 1,
label 0) the run score must equal the exact integer."""
import os
import struct
import subprocess
import tempfile
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host_emul", "runcorr_emul")


def _emulate(ref_bits, sub_bits, o_lo, W, level, label):
    R, S = len(ref_bits), len(sub_bits)
    ref = np.where(ref_bits, np.float32(1.0), np.float32(label)).astype(np.float32)
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("4i2f", R, S, o_lo, W, level, label))
            f.write(ref.tobytes())
            f.write(np.asarray(sub_bits, np.uint8).tobytes())
        subprocess.check_call([EXE, fin, fout])
        raw = open(fout, "rb").read()
    score = np.frombuffer(raw[: 8 * W], np.float64)
    eps = np.frombuffer(raw[8 * W: 8 * W + 8], np.float64)[0]
    um = np.frombuffer(raw[8 * W + 8:], np.int32)
    return score, eps, um


def _xcorr_int(u, m, o_lo, W):
    """c[o] = sum_j u[j] m[j + o] for o in o_lo .. o_lo + W - 1 (exact, integer)."""
    S, R = len(u), len(m)
    n = 1
    while n < R + S + W:
        n *= 2
    fu = np.fft.rfft(u.astype(np.float64)[::-1], n)
    fm = np.fft.rfft(m.astype(np.float64), n)
    full = np.rint(np.fft.irfft(fu * fm, n)).astype(np.int64)  # full[k] = sum_j u[j] m[k - (S-1) + j]
    o = np.arange(o_lo, o_lo + W)
    idx = o + S - 1
    ok = (idx >= 0) & (idx < n) & (o < R) & (o > -S)
    out = np.zeros(W, np.int64)
    out[ok] = full[idx[ok]]
    return out


def _exact(ref_bits, sub_bits, o_lo, W, level, label):
    """Counts c11, c01, c10, c00 per offset and the exact score of the products rescore_kernel sums."""
    u = np.asarray(sub_bits, np.int64)
    m = np.asarray(ref_bits, np.int64)
    S, R = len(u), len(m)
    o = np.arange(o_lo, o_lo + W, dtype=np.int64)
    j_lo = np.maximum(0, -o)
    j_hi = np.minimum(S, R - o)
    n_ov = np.maximum(0, j_hi - j_lo)
    U = np.concatenate([[0], np.cumsum(u)])
    M = np.concatenate([[0], np.cumsum(m)])
    live = n_ov > 0
    uo = np.where(live, U[np.clip(j_hi, 0, S)] - U[np.clip(j_lo, 0, S)], 0)
    mw = np.where(live, M[np.clip(j_hi + o, 0, R)] - M[np.clip(j_lo + o, 0, R)], 0)
    um = _xcorr_int(u, m, o_lo, W)
    hi = Fraction(2.0 * float(np.float32(level)) - 1.0)
    alpha = Fraction(2.0 * float(np.float32(label)) - 1.0)
    exact = []
    for i in range(W):
        c11 = int(um[i])
        c01 = int(mw[i]) - c11
        c10 = int(uo[i]) - c11
        c00 = int(n_ov[i]) - int(mw[i]) - int(uo[i]) + c11
        exact.append(hi * c11 - c01 + hi * alpha * c10 - alpha * c00)
    return exact, um


def _check(ref_bits, sub_bits, o_lo, W, level, label):
    score, eps, um_got = _emulate(ref_bits, sub_bits, o_lo, W, level, label)
    exact, um = _exact(ref_bits, sub_bits, o_lo, W, level, label)
    assert np.array_equal(um_got, um), "UM counts differ"
    worst = max(abs(Fraction(float(s)) - e) for s, e in zip(score, exact)) if W else 0
    assert worst <= Fraction(eps) / 2, (float(worst), eps)
    if level == 1.0 and label == 0.0:
        assert all(Fraction(float(s)) == e for s, e in zip(score, exact))
    # eps is the documented bound for a 2 h pair's size class, not a loose constant
    n = min(len(ref_bits), len(sub_bits))
    assert eps < 1e-9 * max(n, 1) ** 2 + 1e-12
    return score, eps


def _runs(S, starts_lens):
    u = np.zeros(S, np.uint8)
    for a, n in starts_lens:
        u[a:a + n] = 1
    return u


def _random_mask(rng, n, p_on=0.02, mean_len=30):
    u = np.zeros(n, np.uint8)
    j = 0
    while j < n:
        if rng.rand() < p_on:
            L = max(1, int(rng.exponential(mean_len)))
            u[j:j + L] = 1
            j += L + 1
        else:
            j += int(rng.exponential(20)) + 1
    return u


LEVELS = [1.0, 0.96, 0.999]
LABELS = [0.0, 0.3]


@pytest.mark.parametrize("level", LEVELS)
@pytest.mark.parametrize("label", LABELS)
def test_random_runs_every_offset(level, label):
    rng = np.random.RandomState(int(level * 1000) + int(label * 10))
    R, S = 5000, 4200
    m = (rng.rand(R) < 0.45).astype(np.uint8)
    u = _random_mask(rng, S)
    # window covering every offset with an overlap and beyond on both sides
    _check(m, u, -S - 40, R + S + 80, level, label)


@pytest.mark.parametrize("label", LABELS)
def test_runs_touching_the_edges(label):
    rng = np.random.RandomState(7)
    R, S = 900, 700
    m = (rng.rand(R) < 0.5).astype(np.uint8)
    m[0] = m[-1] = 1
    u = _runs(S, [(0, 5), (40, 1), (42, 1), (44, 1), (300, 64), (S - 3, 3)])
    _check(m, u, -S - 33, R + S + 66, 0.96, label)
    _check(m, u, -S - 33, R + S + 66, 1.0, label)


@pytest.mark.parametrize("level,label", [(1.0, 0.0), (0.999, 0.3)])
def test_adjacent_one_frame_runs(level, label):
    rng = np.random.RandomState(3)
    R, S = 1200, 1000
    m = (rng.rand(R) < 0.5).astype(np.uint8)
    u = np.zeros(S, np.uint8)
    u[::2] = 1  # every run one frame long, one frame apart: 500 runs, 1000 endpoints
    _check(m, u, -S - 5, R + S + 10, level, label)


@pytest.mark.parametrize("case", ["no_cues", "one_cue", "all_cue"])
def test_degenerate_masks(case):
    rng = np.random.RandomState(11)
    R, S = 700, 650
    m = (rng.rand(R) < 0.3).astype(np.uint8)
    u = {"no_cues": np.zeros(S, np.uint8), "one_cue": _runs(S, [(100, 37)]),
         "all_cue": np.ones(S, np.uint8)}[case]
    for level, label in [(1.0, 0.0), (0.96, 0.3)]:
        _check(m, u, -S - 10, R + S + 20, level, label)


@pytest.mark.parametrize("R,S", [(300, 20000), (20000, 300)])
def test_lopsided_lengths(R, S):
    rng = np.random.RandomState(R)
    m = (rng.rand(R) < 0.5).astype(np.uint8)
    u = _random_mask(rng, S, p_on=0.05)
    _check(m, u, -S - 17, R + S + 34, 0.96, 0.3)
    _check(m, u, -S - 17, R + S + 34, 1.0, 0.0)


def test_reference_all_speech_and_all_silence():
    rng = np.random.RandomState(5)
    S = 800
    u = _random_mask(rng, S, p_on=0.05)
    for m in (np.ones(1000, np.uint8), np.zeros(1000, np.uint8)):
        _check(m, u, -S - 3, 1000 + S + 6, 0.96, 0.3)


def test_window_of_one_offset():
    rng = np.random.RandomState(2)
    m = (rng.rand(3000) < 0.5).astype(np.uint8)
    u = _random_mask(rng, 2500)
    for o in (-2600, -2499, -17, 0, 31, 2999, 3000):
        _check(m, u, o, 1, 0.96, 0.3)
        _check(m, u, o, 1, 1.0, 0.0)


def test_widest_window():
    """32 x 1024 offsets: every thread of the widest CTA, windows running off both ends of the reference."""
    rng = np.random.RandomState(9)
    R, S = 40000, 36000
    m = (rng.rand(R) < 0.4).astype(np.uint8)
    u = _random_mask(rng, S, p_on=0.01, mean_len=200)
    _check(m, u, -16384, 32 * 1024, 1.0, 0.0)
    _check(m, u, R - 16000, 32 * 1024, 0.96, 0.3)


@pytest.mark.parametrize("n_runs", [7, 8, 14, 15])
def test_anticorrelated_reference_fills_the_counters(n_runs):
    """A reference that is the complement of the mask at a planted offset: speech just after every run end,
    silence at every run start, so every run adds 2 to the same 4-bit counter (7 runs fill it to 14; the
    flush every kRunsPerFlush runs must come before it wraps).  Run counts on both sides of the flushes."""
    rng = np.random.RandomState(n_runs)
    S, R, o_star = 600, 2000, 777
    u = _runs(S, [(20 + 40 * i, 1 + i % 5) for i in range(n_runs)])
    m = (rng.rand(R) < 0.5).astype(np.uint8)
    m[o_star:o_star + S] = 1 - u
    for level, label in [(1.0, 0.0), (0.96, 0.3)]:
        score, _ = _check(m, u, o_star - 100, 224, level, label)
    assert score[100] == score.min()   # every frame disagrees at the planted offset (last call: level 0.96)


def test_two_hour_bound_size():
    """eps for a 2 h pair (720 000 frames each side) is about 1e-4 - the figure DESIGN.md quotes."""
    rng = np.random.RandomState(4)
    R = S = 720000
    m = (rng.rand(R) < 0.5).astype(np.uint8)
    u = _random_mask(rng, S, p_on=0.004, mean_len=250)
    score, eps = _check(m, u, -6000, 64, 0.96, 0.0)
    assert 5e-5 < eps < 2e-4, eps
