"""The rasterisers' cue arithmetic (csrc/raster_math.cuh, the functions raster_cues_kernel and
raster_bits_kernel call) run on the CPU (tests/host_emul/raster_emul.cu) against the reference
evaluated in Python, record by record:
    scaled = timedelta(seconds=t * ratio).total_seconds()
    first  = int(round((scaled_start - start_seconds) * sample_rate))
    last   = first + int(round((scaled_end - scaled_start) * sample_rate))
    (first, last) = slice(first, last).indices(n)[:2]
on about 10^6 records from the edge catalogue below, where a subtly wrong formula goes wrong:
  * products that are exact half-microsecond ties (both parities of the microsecond, negative times),
    at ratio 1, the bench ratios, 2.0, 0.9 and 1.1;
  * half-frame starts and durations (both parities) with start_seconds in {0, 0.005, 0.3, 12.345};
  * every slice case: first below -n (clamps to 0), in [-n, -1] (wraps), at and past n, last at n and
    n + 1, last < first, zero and negative durations;
  * cue times near 2 h and 10 h, and random times of every magnitude up to the 2^53 us limit.
Also b2_rasterize_lengths on the same adversarial ends and its rejection of inputs the arithmetic does
not reproduce (non-finite times and ratios, |t| * ratio at or beyond 2^53 us).

The generators are shared with tests/test_gpu_raster_exact.py, which feeds the same catalogue to both
kernels."""
import math
import os
import subprocess
import sys
import tempfile
from datetime import timedelta

import numpy as np
import pytest

import cases
from conftest import ROOT
from oracle import raster_oracle as ro

EXE = os.path.join(ROOT, "tests", "host_emul", "raster_emul")

BENCH = [1.0, 24.0 / 23.976, 25.0 / 24.0, 23.976 / 24.0, 24.0 / 25.0]
RATIOS = BENCH + [2.0, 0.9, 1.1]
START_SECONDS = [0.0, 0.005, 0.3, 12.345]
MAX_CUE_SECONDS = 2.0 ** 53 / 1e6          # raster_math.cuh B2_MAX_CUE_SECONDS

IN_DT = np.dtype([("st", "<f8"), ("en", "<f8"), ("r", "<f8"), ("ss", "<f8"), ("sr", "<i8"), ("n", "<i8")])
OUT_DT = np.dtype([("sst", "<f8"), ("sen", "<f8"), ("first", "<i8"), ("last", "<i8")])


# ------------------------------------------------------------------------------------ generators

def _ulps(x, j):
    """x moved by j ulps (j may be negative), elementwise."""
    x = np.array(x, np.float64)
    d = np.inf if j > 0 else -np.inf
    for _ in range(abs(j)):
        x = np.nextafter(x, d)
    return x


def half_us_products(rng, W_lo, W_hi, n_try, half_frame=False):
    """Products y = W + (k + 1/2) 1e-6 (W integer in [W_lo, W_hi)) with modf(y)[0] * 1e6 == k + 1/2 exactly:
    ties of timedelta's microsecond rounding.  half_frame: k a multiple of 5 000, so that the two
    roundings of the tie fall on either side of a half frame at 100 Hz for any start_seconds that is a
    multiple of 5 ms (a wrong microsecond rounding then moves a frame).  Returns (y, k)."""
    W = rng.randint(W_lo, W_hi, n_try).astype(np.float64)
    if half_frame:
        k = 5000.0 * rng.randint(0, 200, n_try)
    else:
        k = rng.randint(0, 1000000, n_try).astype(np.float64)
    y0 = W + (k + 0.5) * 1e-6
    ys, ks = [], []
    for j in range(-3, 4):
        y = _ulps(y0, j)
        hit = np.modf(y)[0] * 1e6 == k + 0.5
        ys.append(y[hit])
        ks.append(k[hit])
    y, k = np.concatenate(ys), np.concatenate(ks)
    y, idx = np.unique(y, return_index=True)
    return y, k[idx]


def times_with_product(y, r):
    """For each y, a time t with fl(t * r) == y if one lies within 4 ulps of y / r (else dropped)."""
    t0 = y / r
    got = np.full(len(y), np.nan)
    for j in (0, -1, 1, -2, 2, -3, 3, -4, 4):
        t = _ulps(t0, j)
        ok = np.isnan(got) & (t * r == y)
        got[ok] = t[ok]
    keep = ~np.isnan(got)
    return got[keep], y[keep]


def half_us_times(rng, r, W_lo, W_hi, n_try, half_frame=False):
    """Times whose product with r is a half-microsecond tie, both signs (modf and rint are odd)."""
    y, _ = half_us_products(rng, W_lo, W_hi, n_try, half_frame)
    t, y = times_with_product(y, r)
    sign = np.where(rng.rand(len(t)) < 0.3, -1.0, 1.0)
    return t * sign


def half_frame_cues(rng, r, ss, n_cues, lo_frame=0, hi_frame=720000, sr=100):
    """(start, end) times whose scaled start sits half a frame after a frame of start_seconds ss, and whose
    scaled duration is a whole number of frames plus a half (both parities of each)."""
    m = rng.randint(lo_frame, hi_frame, n_cues)
    d = rng.randint(0, 600, n_cues)
    us_per_frame = 1000000 // sr
    st_us = np.rint(ss * 1e6).astype(np.int64) + m * us_per_frame + us_per_frame // 2
    en_us = st_us + d * us_per_frame + us_per_frame // 2
    st, en = st_us / 1e6, en_us / 1e6
    return st / r, en / r


def slice_case_cues(rng, r, ss, n, n_cues, sr=100):
    """(start, end) times whose frames cover every slice case of a length-n signal: first in [-3n, 2n]
    (below -n clamps to 0, [-n, -1] wraps, n and beyond clamp to n), durations in [-n, 2n] (zero,
    negative, last at n and n + 1, last < first).  Frames land up to 0.45 frame off the grid."""
    first = rng.randint(-3 * n, 2 * n + 1, n_cues)
    dur = rng.randint(-n, 2 * n + 1, n_cues)
    jit = rng.uniform(-0.45, 0.45, (2, n_cues))
    st = ss + (first + jit[0]) / sr
    en = st + (dur + jit[1]) / sr
    return st / r, en / r


def long_time_cues(rng, r, centre, n_cues):
    """Times within 10 s of `centre` seconds of scaled time (2 h, 10 h): ulp(t) ~ 1e-12, frames tight."""
    st = centre + rng.uniform(-10.0, 0.0, n_cues)
    en = st + rng.uniform(0.0, 5.0, n_cues)
    return st / r, en / r


def random_magnitude_times(rng, r, n):
    """Times of every magnitude from 1 us to just below the 2^53 us limit, both signs."""
    mag = 10.0 ** rng.uniform(-6, math.log10(MAX_CUE_SECONDS) - 1e-9, n)
    t = mag * np.where(rng.rand(n) < 0.5, -1.0, 1.0) / r
    return t[np.abs(t) * r < MAX_CUE_SECONDS]


# ------------------------------------------------------------------------------------ reference

def reference(rec):
    """The reference's arithmetic in Python, for every record: (scaled start, scaled end, first, last)."""
    out = np.empty(len(rec), OUT_DT)
    rows = []
    for st, en, r, ss, sr, n in rec.tolist():
        a = timedelta(seconds=st * r).total_seconds()
        b = timedelta(seconds=en * r).total_seconds()
        first = int(round((a - ss) * sr))
        last = first + int(round((b - a) * sr))
        lo, hi, _ = slice(first, last).indices(n)
        rows.append((a, b, lo, hi))
    out[:] = rows
    return out


def emulate(rec):
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        np.ascontiguousarray(rec, IN_DT).tofile(fin)
        subprocess.check_call([EXE, fin, fout])
        return np.fromfile(fout, OUT_DT)


def records(st, en, r, ss, n, sr=100):
    rec = np.empty(len(st), IN_DT)
    rec["st"], rec["en"], rec["r"], rec["ss"], rec["sr"], rec["n"] = st, en, r, ss, sr, n
    return rec


def catalogue(seed=0):
    """About 10^6 records of the edge catalogue; also returns the number of records of each family."""
    rng = np.random.RandomState(seed)
    parts, fam = [], {}

    def add(name, rec):
        parts.append(rec)
        fam[name] = fam.get(name, 0) + len(rec)

    for r in RATIOS:
        for W_lo, W_hi, n_try, hf in ((0, 1, 3000, False), (1, 100, 200000, False), (100, 7300, 400000, False),
                                      (35900, 36100, 400000, False), (0, 600, 100000, True)):
            t = half_us_times(rng, r, W_lo, W_hi, n_try, hf)
            # tie at the start, at the end, or both; random other end
            other = t + np.where(t >= 0, 1.0, -1.0) * rng.uniform(0, 5, len(t))
            both = np.roll(t, 1)
            ss = rng.choice(START_SECONDS, len(t))
            n = np.maximum(2, (np.abs(t) * r * 100).astype(np.int64) + rng.randint(-200, 200, len(t)))
            add("half_us", records(t, other, r, ss, n))
            add("half_us", records(other, t, r, ss, n))
            add("half_us", records(t, both, r, ss, n))
        for ss in START_SECONDS:
            st, en = half_frame_cues(rng, r, ss, 6000)
            n = rng.randint(2, 730000, len(st))
            add("half_frame", records(st, en, r, ss, n))
            st, en = half_frame_cues(rng, r, ss, 2000, 3590000, 3600000)
            add("half_frame", records(st, en, r, ss, rng.randint(3590000, 3610000, len(st))))
            for n in (1, 2, 31, 32, 33, 1000, 720002):
                st, en = slice_case_cues(rng, r, ss, n, 1200)
                add("slice", records(st, en, r, ss, n))
        for centre in (7200.0, 36000.0):
            st, en = long_time_cues(rng, r, centre, 10000)
            ss = rng.choice(START_SECONDS, len(st))
            add("long", records(st, en, r, ss, int(centre * 100) + 2))
        t = random_magnitude_times(rng, r, 25000)
        e = t + rng.uniform(-1, 5, len(t))
        ss = rng.choice(START_SECONDS, len(t))
        add("magnitude", records(t, e, r, ss, rng.randint(1, 1 << 40, len(t))))
    return np.concatenate(parts), fam


# ------------------------------------------------------------------------------------ tests

@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


def test_closed_form_equals_timedelta_on_the_ties():
    """The ties the catalogue is built from really are ties, and the oracle's closed form agrees."""
    rng = np.random.RandomState(1)
    y, k = half_us_products(rng, 1, 7300, 400000)
    assert len(y) > 30 and {0, 1} <= set((k % 2).astype(int).tolist())
    for x in np.concatenate([y, -y]).tolist():
        assert timedelta(seconds=x).total_seconds() == ro.seconds_via_timedelta_closed_form(x), x


def test_cue_arithmetic_matches_reference(built):
    rec, fam = catalogue()
    assert 800000 <= len(rec) <= 1500000, len(rec)
    got = emulate(rec)
    want = reference(rec)
    assert len(got) == len(rec)
    for f in OUT_DT.names:
        bad = np.flatnonzero(got[f] != want[f])
        assert len(bad) == 0, (f, len(bad), [(rec[i].tolist(), got[i].tolist(), want[i].tolist()) for i in bad[:5]])

    # the catalogue reaches what it is meant to reach (judged from the reference's own values)
    r, ss, sr = rec["r"], rec["ss"], rec["sr"]
    prod = rec["st"] * r
    frac_us = np.modf(prod)[0] * 1e6
    tie = np.modf(np.abs(frac_us))[0] == 0.5
    k = np.floor(np.abs(frac_us)).astype(np.int64)
    for ratio in RATIOS:
        sel = tie & (r == ratio)
        assert np.sum(sel & (k % 2 == 0)) >= 100 and np.sum(sel & (k % 2 == 1)) >= 100, ratio
        assert np.sum(sel & (prod < 0)) >= 50, ratio
    x0 = (want["sst"] - ss) * sr
    dur = (want["sen"] - want["sst"]) * sr
    for s in START_SECONDS:
        for x in (x0, dur):
            half = (ss == s) & (np.modf(np.abs(x))[0] == 0.5)
            par = np.floor(np.abs(x)).astype(np.int64) % 2
            assert np.sum(half & (par == 0)) >= 100 and np.sum(half & (par == 1)) >= 100, s
    raw_first = np.array([int(round(v)) for v in x0.tolist()], dtype=object)
    n = rec["n"]
    first_i = np.array([int(v) for v in raw_first], np.int64)
    assert np.sum(first_i < -n) >= 1000         # clamps to 0
    assert np.sum((first_i >= -n) & (first_i < 0)) >= 1000      # wraps
    assert np.sum(first_i == n) >= 10 and np.sum(first_i > n) >= 1000
    assert np.sum(want["last"] == n) >= 1000 and np.sum(want["last"] < want["first"]) >= 1000
    assert np.sum(np.rint(dur) == 0) >= 100 and np.sum(dur < -0.5) >= 1000
    assert fam["long"] >= 100000 and fam["magnitude"] >= 100000


def test_lengths_on_adversarial_ends(built):
    """b2_rasterize_lengths == int(max(0, max scaled end) * sr) + 2 of the reference, per (track, ratio),
    for ends at half-microsecond ties, whole and half frames, negative ends, long times and tracks whose
    longest cue is a metadata cue (lengths ignore keep)."""
    from ffsubsync_b200 import _native
    lib = _native.load()
    rng = np.random.RandomState(7)
    ratios = np.array(RATIOS)
    tracks = []
    for r in RATIOS:
        tracks.append(half_us_times(rng, r, 1, 7300, 200000)[:40])
        st, en = half_frame_cues(rng, r, 0.0, 40)
        tracks.append(en)
        tracks.append(np.rint(en * r * 100) / 100 / r)      # whole frames of scaled time
        tracks.append(-np.abs(en))                          # every end negative: length 2
        tracks.append(long_time_cues(rng, r, 36000.0, 30)[1])
    tracks.append(np.zeros(0))
    tracks.append(np.array([-0.0, 0.0]))
    for sr in (100, 1000, 48000):
        for per_pair in (0, 1):
            rr = np.tile(ratios, len(tracks)) if per_pair else ratios
            if per_pair:
                rr = rr * np.where(rng.rand(len(rr)) < 0.5, 1.0, 1.0 + 1e-9)
            K = len(ratios)
            ends = np.concatenate(tracks).astype(np.float64)
            off = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int64)
            lengths = np.empty(len(tracks) * K, np.int64)
            rr = np.ascontiguousarray(rr, np.float64)
            st = lib.b2_rasterize_lengths(ends.ctypes.data, off.ctypes.data, len(tracks), rr.ctypes.data, K,
                                          per_pair, sr, lengths.ctypes.data)
            assert st == 0
            for b, t in enumerate(tracks):
                for k in range(K):
                    r = float(rr[b * K + k] if per_pair else rr[k])
                    max_time = 0
                    for e in t.tolist():
                        max_time = max(max_time, timedelta(seconds=e * r).total_seconds())
                    assert lengths[b * K + k] == int(max_time * sr) + 2, (sr, per_pair, b, k)


def _lengths_status(ends, ratios, per_pair=0, off=None):
    from ffsubsync_b200 import _native
    lib = _native.load()
    ends = np.ascontiguousarray(ends, np.float64)
    ratios = np.ascontiguousarray(ratios, np.float64)
    off = np.array([0, len(ends)] if off is None else off, np.int64)
    B = len(off) - 1
    K = len(ratios) // B if per_pair else len(ratios)
    lengths = np.empty(max(1, B * K), np.int64)
    return lib.b2_rasterize_lengths(ends.ctypes.data, off.ctypes.data, B, ratios.ctypes.data, K, per_pair, 100,
                                    lengths.ctypes.data), lengths


def test_lengths_reject_what_the_arithmetic_does_not_reproduce(built):
    """Non-finite ends (also on a cue that is not the longest, and on metadata cues: lengths see every end),
    ends whose product with the largest ratio reaches 2^53 us, and ratios that are not finite and positive."""
    L = MAX_CUE_SECONDS
    below = np.nextafter(L, 0)
    ok = [1.0, 2.0, 3.5]
    assert _lengths_status(ok, [1.0, 0.5])[0] == 0
    for bad_end in (np.nan, np.inf, -np.inf, L, -L, 1e13, -1e13, 1e300):
        st, _ = _lengths_status([1.0, bad_end, 3.0], [1.0])
        assert st == -1, bad_end
    # the limit is on |t| * ratio as the arithmetic computes it: at ratio 2 half the time reaches it
    assert _lengths_status([below], [1.0])[0] == 0
    assert _lengths_status([-below], [1.0])[0] == 0
    assert _lengths_status([L / 2], [2.0])[0] == -1
    assert _lengths_status([below / 2], [2.0])[0] == 0
    assert _lengths_status([L / 1.4], [1.0, 1.3])[0] == 0
    assert _lengths_status([L / 1.4], [1.0, 1.5, 1.3])[0] == -1           # the largest ratio decides
    # a time just below the limit is exact, and the length is the reference's
    st, n = _lengths_status([below], [1.0])
    assert n[0] == int(timedelta(seconds=below).total_seconds() * 100) + 2
    for bad_r in (0.0, -1.0, np.nan, np.inf, -np.inf):
        assert _lengths_status(ok, [1.0, bad_r])[0] == -1, bad_r
        assert _lengths_status(ok + ok, [1.0, 1.0, 1.0, bad_r], per_pair=1, off=[0, 3, 6])[0] == -1, bad_r
    # a bad end in the second track only
    assert _lengths_status(ok + [1.0, np.nan], [1.0], off=[0, 3, 5])[0] == -1
    # the reference raises for the same inputs
    for bad in (np.nan, np.inf):
        with pytest.raises((ValueError, OverflowError)):
            timedelta(seconds=bad)


def test_bench_ratio_grid_lengths_unchanged(built):
    """The bench's synthetic cue lists: lengths as before at every ratio of the grid."""
    from ffsubsync_b200 import _native
    lib = _native.load()
    starts, ends = cases.synthetic_cues(16, 7200.0)
    ratios = np.array(cases.ratio_grid())
    lengths = np.empty(len(ratios), dtype=np.int64)
    off = np.array([0, len(ends)], dtype=np.int64)
    assert lib.b2_rasterize_lengths(ends.ctypes.data, off.ctypes.data, 1, ratios.ctypes.data, len(ratios), 0,
                                    100, lengths.ctypes.data) == 0
    for r, n in zip(ratios, lengths):
        assert n == len(ro.rasterize(starts, ends, None, 100, 0, r)[0])
