"""Deterministic input generators shared by make_golden.py (which runs the real reference in
the build container) and the tests (which replay the same inputs through the oracle and the
CUDA path).  Pure numpy; every case is a function of small integer parameters so fixtures
only need to store parameters + expected outputs."""
import numpy as np

FRAMERATE_RATIOS = [24.0 / 23.976, 25.0 / 23.976, 25.0 / 24.0]  # constants.py:9


def ratio_grid():
    """[1.0] + ratios + inverses, in the order try_sync builds it (ffsubsync.py:131-142,196-199)."""
    r = np.array(FRAMERATE_RATIOS)
    return [1.0] + list(np.concatenate([r, 1.0 / r]))


def small_align_case(seed: int):
    """Small random (ref, sub, max_offset_samples) with a mix of value kinds and mask regimes."""
    rng = np.random.RandomState(1000 + seed)
    n_ref = int(rng.randint(1, 200))
    n_sub = int(rng.randint(1, 200))
    kind = seed % 5
    if kind == 0:      # binary
        ref = (rng.rand(n_ref) > 0.5).astype(float)
        sub = (rng.rand(n_sub) > 0.5).astype(float)
    elif kind == 1:    # two-level subtitle side, like a non-unit framerate ratio
        ref = (rng.rand(n_ref) > 0.4).astype(float)
        sub = (rng.rand(n_sub) > 0.6).astype(float) * 0.96
    elif kind == 2:    # "not sure" non-speech label 0.5 on the reference side
        ref = np.where(rng.rand(n_ref) > 0.5, 1.0, 0.5)
        sub = (rng.rand(n_sub) > 0.5).astype(float)
    elif kind == 3:    # arbitrary floats in [0, 1]
        ref = rng.rand(n_ref)
        sub = rng.rand(n_sub)
    else:              # correlated pair: sub is a shifted copy of ref
        shift = int(rng.randint(-20, 21))
        base = (rng.rand(n_ref + 64) > 0.5).astype(float)
        ref = base[32 : 32 + n_ref]
        idx = np.clip(np.arange(n_sub) + 32 + shift, 0, len(base) - 1)
        sub = base[idx]
    mode = (seed // 5) % 4
    if mode == 0:
        mos = None
    elif mode == 1:
        mos = int(rng.randint(0, 12))
    elif mode == 2:
        mos = int(rng.randint(12, 120))
    else:
        mos = int(rng.randint(120, 1200))  # exercises the negative-slice wrap corner
    return ref, sub, mos


def shifted_pair(n: int, shift: int = 1234, seed: int = 0):
    """SURVEY.md section 8c golden: ref = rand > 0.6, sub = ref delayed by ``shift`` frames."""
    rng = np.random.RandomState(seed)
    ref = (rng.rand(n) > 0.6).astype(float)
    sub = np.concatenate([np.zeros(shift), ref])[:n]
    return ref, sub


# Wide-window alignments (large FFT path): lengths, shift, subtitle level, masks to run.
WIDE_CASES = [
    dict(seed=1, R=70000, S=60000, shift=4321, level=1.0, mos_list=[None, 40000]),
    dict(seed=2, R=200000, S=9000, shift=-150000, level=1.0, mos_list=[None]),       # R >> S, negative offset... (sub late in ref)
    dict(seed=3, R=9000, S=200000, shift=120000, level=0.96, mos_list=[None, 150000]),   # S >> R, float level
    dict(seed=4, R=131000, S=131100, shift=77, level=1.0, mos_list=[None]),            # R + S just above 2^18
    dict(seed=5, R=131072, S=131072, shift=-5, level=0.5, mos_list=[None, 70000]),      # R + S == 2^18 exactly
    dict(seed=6, R=300000, S=280000, shift=None, level=1.0, mos_list=[None]),           # unrelated signals
]


def wide_pair(seed, R, S, shift, level, mos_list=None):
    """ref = rand > 0.55; sub[j] = level * ref[j + offset] with offset = -shift ... i.e. the subtitles are the
    reference delayed by ``shift`` frames (negative: advanced), or independent noise when shift is None."""
    rng = np.random.RandomState(seed)
    ref = (rng.rand(R) > 0.55).astype(float)
    if shift is None:
        sub = (rng.rand(S) > 0.5).astype(float) * level
    else:
        idx = np.arange(S) - shift
        ok = (idx >= 0) & (idx < R)
        sub = np.where(ok, ref[np.clip(idx, 0, R - 1)], (rng.rand(S) > 0.5).astype(float)) * level
    return ref, sub


def scaled_signal(sub: np.ndarray, sf: float) -> np.ndarray:
    """Nearest-neighbour resampling of a 100 Hz signal by a framerate ratio (the construction
    the reference's own multi-segment test uses to emulate SubtitleScaler on a raw signal)."""
    out = np.zeros(int(len(sub) * sf) + 2)
    k = np.arange(len(out))
    src = np.round(k / sf).astype(int)
    ok = src < len(sub)
    out[k[ok]] = sub[src[ok]]
    return out


def multi_segment_case(true_scale: float, true_shift: float, sr: int = 100):
    """Inputs of tests/test_multi_segment.py:135-167: a 24 000-frame subtitle signal that is a
    (scale, shift) warp of a random reference, and the sparse reference (8 x 60 s segments at
    evenly spaced starts, zeros elsewhere) that MultiSegmentVideoSpeechTransformer builds."""
    rng = np.random.RandomState(13)
    n_sub = 24000
    n_ref = int(true_scale * n_sub + abs(true_shift) * sr) + 2000
    ref_full = (rng.rand(n_ref) > 0.6).astype(float)
    m = np.arange(n_sub)
    idx = np.round(true_scale * m + true_shift * sr).astype(int)
    sub = np.zeros(n_sub)
    ok = (idx >= 0) & (idx < n_ref)
    sub[m[ok]] = ref_full[idx[ok]]
    return ref_full, sub


# Signal families that stress the round-off bound tau of the nomination stage: large means (the
# ||c||_2 term of tau dominates), flat or periodic correlation landscapes, exact ties, wide dynamic range.
SIGNAL_FAMILIES = ["random", "ones", "zeros", "period2", "period_block", "sparse", "wide", "ramp"]
# Families aimed at the large-window path's four-step layout: its [M1][1024] work array holds
# z[n] = x[2n] + i x[2n+1] row by row, so one row is 2048 real samples.  A period of 2048 makes every column
# constant (all energy in column bin 0); the impulse train is the extreme broad, flat correlation.
LAYOUT_FAMILIES = ["square_2048", "impulse_2048"]
# (reference, subtitle) family pairings run at the largest transform sizes (2^22, 2^23 and their CPU emulation),
# where every pairing would cost too much: the large-mean and block-periodic references against random subtitles,
# and the layout families on either side.
BIG_TRANSFORM_PAIRS = [(f, "random") for f in ("random", "period_block", "ones", "sparse", "ramp", "wide")] + \
    [(f, g) for f in LAYOUT_FAMILIES for g in ("random", f)] + [("random", f) for f in LAYOUT_FAMILIES]


def signal_family(name, n, rng, level=1.0):
    """float32 signal of family ``name`` and length ``n``; two-level families take the value ``level``."""
    if name == "random":
        return (rng.rand(n) > rng.uniform(0.2, 0.8)).astype(np.float32) * np.float32(level)
    if name == "ones":
        return np.full(n, level, np.float32)
    if name == "zeros":
        return np.zeros(n, np.float32)
    if name == "period2":
        return (np.arange(n) % 2).astype(np.float32) * np.float32(level)
    if name == "period_block":   # period = the block length of the +-60 s window (L = 20 736)
        return ((np.arange(n) // 10368) % 2).astype(np.float32) * np.float32(level)
    if name == "sparse":         # multi-segment reference: a few 60 s windows of speech, zero elsewhere
        x = np.zeros(n, np.float32)
        for s in rng.randint(0, max(1, n - 6000), 6):
            x[s:s + 6000] = (rng.rand(len(x[s:s + 6000])) > 0.5) * np.float32(level)
        return x
    if name == "wide":           # float levels spanning 1e-3 ... 1e3
        return (10.0 ** rng.uniform(-3, 3, n) * rng.choice([0.0, 1.0], n)).astype(np.float32)
    if name == "ramp":
        return np.linspace(0.0, level, n).astype(np.float32)
    if name == "square_2048":
        return ((np.arange(n) // 1024) % 2).astype(np.float32) * np.float32(level)
    if name == "impulse_2048":
        return (np.arange(n) % 2048 == 0).astype(np.float32) * np.float32(level)
    raise ValueError(name)


def synthetic_cues(seed: int, duration_s: float):
    rng = np.random.RandomState(seed)
    t = 5.0
    starts, ends = [], []
    while t < duration_s - 10.0:
        d = rng.uniform(1.0, 5.0)
        starts.append(round(t, 3))
        ends.append(round(t + d, 3))
        t += d + rng.exponential(3.0)
    return np.array(starts), np.array(ends)


def run_lengths(x: np.ndarray):
    """Encode a two-level signal as (level, [start, stop) runs of non-zero samples)."""
    nz = np.asarray(x) != 0
    d = np.diff(np.concatenate([[0], nz.astype(np.int8), [0]]))
    starts = np.flatnonzero(d == 1)
    stops = np.flatnonzero(d == -1)
    levels = np.unique(np.asarray(x)[nz])
    return [float(v) for v in levels], [int(v) for v in starts], [int(v) for v in stops]
