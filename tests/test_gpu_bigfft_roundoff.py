"""The large-window aligner's round-off bound tau (csrc/bigfft.cu, bigfft.cuh) on every signal family at every
transform size N = 2^17 .. 2^23, float and bit-mask subtitle signals.

The four-step FFT path is the one max_offset_samples=None takes for every real movie.  Its fp32 scores only
nominate: every offset within tau of the fp32 maximum is re-scored exactly, which is correct only if
|fp32 score - exact score| <= tau at every offset.  The twiddle and column errors of the four-step chain grow with
M1 = N / 2048 while tau's constants do not, so the margin is measured here where it is thinnest: large N, signals
with a large mean (ones, sparse, ramp), block-periodic signals, and two families aimed at the [M1][1024] layout
(cases.LAYOUT_FAMILIES: a period of 2048 samples is one row, so every column is constant).

Every captured job (b2_capture_nominations) goes through nomination_check.check_jobs: the oracle's window,
max |fp32 - exact| <= tau with the kernels' own tau, the candidate count and B2_ALIGN_CAND_OVERFLOW, the returned
offset as the exact argmax over the 32 largest-offset candidates with the exact score, the tie rule on binary
inputs.  On top of that the captured tau must not fall below the float64 value of the same bound, u (512
sqrt(Es Er) + 192 ||c||_2), computed from the signals the kernels saw and the exact correlation over the whole
N-length output: the fp32 sums behind Es, Er (F1) and ||c||_2 (F3) run over up to 8 M samples, and a sum that
loses mass would shrink tau unnoticed.

At the end the module prints the worst error / tau per (N, encoding) with the family pair that attains it, then per
(N, encoding, family pair)."""
import numpy as np
import pytest

import cases
from nomination_check import Exact, check_jobs
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import sig_oracle as so

pytestmark = pytest.mark.gpu

FAMILIES = cases.SIGNAL_FAMILIES + cases.LAYOUT_FAMILIES
CAPTURE_BYTES = 1 << 29     # captured fp32 scores per call (one N-wide row per job)
TAU_SLACK = 1e-3            # relative: captured tau >= (1 - TAU_SLACK) x the float64 tau
SHAPES = [(0.45, 0.40), (0.15, 0.70), (0.60, 0.30)]   # (R, S) / N: balanced, S >> R, R >> S
MARGIN = {}                 # (N, encoding, family pair) -> worst max |fp32 - exact| / tau


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module", autouse=True)
def report_margins():
    yield
    worst = {}
    for (n, enc, pair), r in MARGIN.items():
        worst[n, enc] = max(worst.get((n, enc), (0.0, "")), (r, pair))
    for (n, enc), (r, pair) in sorted(worst.items()):
        print("large-window error / tau, worst [N=2^%d, %s]: %.3g = tau/%.0f (%s)"
              % (n.bit_length() - 1, enc, r, 1.0 / max(r, 1e-30), pair))
    for (n, enc, pair), r in sorted(MARGIN.items()):
        print("  N=2^%d %s %s: tau/%.0f" % (n.bit_length() - 1, enc, pair, 1.0 / max(r, 1e-30)))


def _check(cap, sigs, labels, mos, enc, out):
    """check_jobs on one call, then tau against its float64 value per job; records the margins."""
    exact = Exact()
    stats = check_jobs(cap, sigs, mos, exact, ("large-window", enc), out=out)
    for (ref, sub), pair, (mx, tau, w, err) in zip(sigs, labels, stats):
        assert w is not None, pair
        want = exact.tau(ref, sub)
        assert float(tau) >= (1.0 - TAU_SLACK) * want, (enc, pair, len(ref), len(sub), float(tau), want)
        assert float(tau) <= 1.01 * want, (enc, pair, len(ref), len(sub), float(tau), want)
        key = (ao.padded_length(len(ref), len(sub)), enc, pair)
        MARGIN[key] = max(MARGIN.get(key, 0.0), err / float(tau))


def _chunks(items, jobs_of, n):
    """Consecutive runs of items whose jobs' captured rows (4 n bytes each) stay within CAPTURE_BYTES."""
    cap_jobs = max(1, CAPTURE_BYTES // (4 * n))
    run, used = [], 0
    for it in items:
        if run and used + jobs_of(it) > cap_jobs:
            yield run
            run, used = [], 0
        run.append(it)
        used += jobs_of(it)
    if run:
        yield run


# ------------------------------------------------------------------- float signals (b2_align_batch)

LEVELS = (1.0, 0.96)
COPY_PAIRS = [(f, "copy") for f in ("balanced", "random", "sparse", "period_block", "square_2048", "impulse_2048")]


def _float_pair(lg, i, fam_r, fam_s):
    """Reference of family fam_r and the subtitle signal of family fam_s at both LEVELS (the same draw).  Random
    and sparse subtitles carry a delayed copy of the reference on their even frames (a real peak); the other
    families stay pure, so that their own landscape is what the transforms see.  fam_s "copy": the subtitles are
    the reference, delayed."""
    n = 1 << lg
    R, S = (int(f * n) for f in SHAPES[i % len(SHAPES)])
    rng = np.random.RandomState(lg * 1000 + i)
    if fam_r == "balanced":        # white, zero-mean +-1 signal: the flat spectrum and sharpest peak of a copy
        ref = (rng.rand(R) > 0.5).astype(np.float32)
    else:
        ref = cases.signal_family(fam_r, R, rng)
    seed, shift = int(rng.randint(1 << 30)), int(rng.randint(-n // 8, n // 8))
    subs = []
    for level in LEVELS:
        if fam_s == "copy":        # the reference itself, delayed by shift: one peak of the full overlap
            src = np.arange(S) - shift
            ok = (src >= 0) & (src < R)
            sub = np.zeros(S, np.float32)
            sub[ok] = ref[src[ok]] * np.float32(level)
            subs.append(sub)
            continue
        sub = cases.signal_family(fam_s, S, np.random.RandomState(seed), level)
        if fam_s in ("random", "sparse"):
            src = np.arange(S) - shift
            ok = (src >= 0) & (src < R) & (np.arange(S) % 2 == 0)
            sub[ok] = (ref[src[ok]] != 0) * np.float32(level)
        subs.append(sub)
    assert ao.padded_length(R, S) == n
    return ref, subs


def _align_checked(handle, pairs, labels, mos=None):
    """b2_align_batch over pairs [(ref, [sub per level])] under the capture, every job checked."""
    K = len(LEVELS)
    refs = [p[0] for p in pairs]
    subs = [s for p in pairs for s in p[1]]
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.int64)
    sub_off = np.concatenate([[0], np.cumsum([len(s) for s in subs])]).astype(np.int64)
    stride = max(max(1, o_hi - o_lo + 1) for o_lo, o_hi in
                 (ao.offset_range(len(pairs[j // K][0]), len(s), mos) for j, s in enumerate(subs)))
    with handle.capture_nominations(len(subs), stride) as cap:
        out = handle.align_batch(np.concatenate(refs), ref_off, np.concatenate(subs), sub_off, len(pairs), K, mos)
    sigs = [(pairs[j // K][0].astype(np.float64), s.astype(np.float64)) for j, s in enumerate(subs)]
    _check(cap, sigs, ["%s x %s@%g" % (labels[j // K] + (LEVELS[j % K],)) for j in range(len(subs))], mos, "float",
           out)


def _float_run(handle, lg, family_pairs, mos=None):
    items = list(enumerate(family_pairs))
    for run in _chunks(items, lambda it: len(LEVELS), 1 << lg):
        pairs = [_float_pair(lg, i, fr, fs) for i, (fr, fs) in run]
        _align_checked(handle, pairs, [p for _, p in run], mos)


@pytest.mark.parametrize("fam_r", FAMILIES)
@pytest.mark.parametrize("lg", [17, 18, 19, 20, 21])
def test_float_every_family_pairing(handle, lg, fam_r):
    """N = 2^17 .. 2^21: reference family fam_r against every subtitle family, levels 1 and 0.96, unmasked."""
    _float_run(handle, lg, [(fam_r, fs) for fs in FAMILIES])


@pytest.mark.parametrize("lg", [22, 23])
def test_float_largest_transforms(handle, lg):
    """N = 2^22 and 2^23 (M1 = 2048, 4096): the pairings of cases.BIG_TRANSFORM_PAIRS, levels 1 and 0.96."""
    _float_run(handle, lg, cases.BIG_TRANSFORM_PAIRS)


@pytest.mark.parametrize("lg", [17, 18, 19, 20, 21, 22, 23])
def test_float_subtitles_copy_the_reference(handle, lg):
    """Subtitles that are the reference delayed (the sharpest, tallest peak the correlation can have), levels 1 and
    0.96, at every N: balanced +-1 (duty cycle 1/2), random, sparse, block-periodic and layout references."""
    _float_run(handle, lg, COPY_PAIRS)


def test_float_clipped_mask(handle, monkeypatch):
    """A mask that clips the window inside N = 2^21 (+-N/5 offsets), on the large-window path."""
    monkeypatch.setenv("B2_ALIGN_PATH", "big")
    _float_run(handle, 21, cases.BIG_TRANSFORM_PAIRS[:8], mos=(1 << 21) // 5)


# ------------------------------------------------ bit-mask subtitles (b2_sync_tracks_sig, unmasked)

RATIOS = [1.0, 25.0 / 24.0]          # subtitle levels 1 and (float)(24/25) = 0.96
CUE_FAMILIES = ["synthetic", "square_2048", "impulse_2048", "one_cue", "blocks"]
# two-level reference families; "mask" is the video's first track rasterised at ratio 1, delayed, with 10 % of its
# frames flipped (a real peak, like a movie's speech against its own subtitles); "mask_exact" the same without flips
REF_FAMILIES = ["mask", "mask_exact", "random", "ones", "zeros", "period2", "period_block", "sparse", "square_2048",
                "impulse_2048"]
BIG_VIDEOS = [("mask", CUE_FAMILIES), ("mask_exact", ["synthetic", "blocks"]), ("period_block", ["synthetic"]), ("ones", ["synthetic"]),
              ("sparse", ["synthetic"]), ("square_2048", ["synthetic", "square_2048"]),
              ("impulse_2048", ["synthetic", "impulse_2048"])]


def _cues(fam, dur, seed):
    """Cue list (start, end seconds) of family fam over dur seconds.  At ratio 1 and 100 Hz, square_2048 is a
    square wave with a period of 2048 frames and impulse_2048 one frame every 2048."""
    if fam == "synthetic":
        return cases.synthetic_cues(seed, dur)
    k = np.arange(int(dur / 20.48))
    if fam == "square_2048":
        return k * 20.48, k * 20.48 + 10.24
    if fam == "impulse_2048":
        return k * 20.48, k * 20.48 + 0.01
    if fam == "one_cue":
        return np.array([0.0]), np.array([round(dur, 2)])
    if fam == "blocks":      # six 60 s stretches of speech, silence elsewhere
        st = np.sort(np.random.RandomState(seed).uniform(0.0, dur - 60.0, 6)).round(3)
        return st, st + 60.0
    raise ValueError(fam)


def _video(lg, v, fam_r, cue_fams):
    """One signal video: its serialized values (1.0 / 0.0) and the cue lists of its tracks."""
    n = 1 << lg
    fr, fs = SHAPES[v % len(SHAPES)]
    R, dur = int(fr * n), fs * n / 100.0
    rng = np.random.RandomState(lg * 100 + v)
    cues = [_cues(f, dur, lg * 100 + 10 * v + t) for t, f in enumerate(cue_fams)]
    if fam_r in ("mask", "mask_exact"):
        mask = ro.rasterize(*cues[0], None, 100, 0, 1.0)[0] != 0
        src = np.arange(R) - int(rng.randint(-n // 16, n // 16))
        ok = (src >= 0) & (src < len(mask))
        x = np.zeros(R, dtype=bool)
        x[ok] = mask[src[ok]]
        if fam_r == "mask":
            x ^= rng.rand(R) < 0.10
    else:
        x = cases.signal_family(fam_r, R, rng) != 0
    return x.astype(np.float64), cues


def _sync_checked(handle, lg, videos, label):
    """b2_sync_tracks_sig, unmasked, want_all, over videos [(ref family, cue families)] under the capture."""
    K = len(RATIOS)
    xs, cs, ce, track_video, sigs, labels = [], [], [], [], [], []
    for v, (fam_r, cue_fams) in videos:
        x, cues = _video(lg, v, fam_r, cue_fams)
        xs.append(x)
        ref = so.frames(x, label).astype(np.float64)
        for f, (st, en) in zip(cue_fams, cues):
            cs.append(st)
            ce.append(en)
            track_video.append(len(xs) - 1)
            for r in RATIOS:
                sub = (ro.rasterize(st, en, None, 100, 0, r)[0] != 0) * float(np.float32(min(1.0 / r, 1.0)))
                assert ao.padded_length(len(ref), len(sub)) == 1 << lg
                sigs.append((ref, sub))
                labels.append("%s@%g x %s@%g" % (fam_r, label, f, float(np.float32(min(1.0 / r, 1.0)))))
    V, T = len(xs), len(track_video)
    sig_off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
    cue_off = np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64)
    with handle.capture_nominations(T * K, 1 << lg) as cap:
        r = handle.sync_tracks_sig(None, np.zeros(V + 1, np.int64), np.array(track_video, np.int32), 16000, 100,
                                   label, np.ones(V, np.uint8), np.concatenate(xs), sig_off, np.concatenate(cs),
                                   np.concatenate(ce), None, cue_off, RATIOS, 0.0, None, want_all=True)
    _check(cap, sigs, labels, None, "bits", (r[3], r[4], None))


def _sync_run(handle, lg, videos, label):
    items = list(enumerate(videos))
    for run in _chunks(items, lambda it: len(it[1][1]) * len(RATIOS), 1 << lg):
        _sync_checked(handle, lg, run, label)


@pytest.mark.parametrize("label", [0.0, 0.3])
@pytest.mark.parametrize("lg", [17, 18, 19, 20, 21])
def test_bits_every_family(handle, lg, label):
    """N = 2^17 .. 2^21: every two-level reference family (label 0: +-1; 0.3: the reference is 1 / -0.4)
    against every cue family, ratios 1 and 25/24 (subtitle levels 1 and 0.96)."""
    _sync_run(handle, lg, [(f, CUE_FAMILIES) for f in REF_FAMILIES], label)


@pytest.mark.parametrize("label", [0.0, 0.3])
@pytest.mark.parametrize("lg", [22, 23])
def test_bits_largest_transforms(handle, lg, label):
    """N = 2^22 and 2^23: the block-periodic, large-mean and layout references of BIG_VIDEOS."""
    _sync_run(handle, lg, BIG_VIDEOS, label)


def test_bits_tracks_sliced(handle, monkeypatch):
    """Several tracks per video under a 64 MB workspace budget: at N = 2^21 one track's two ratio jobs take 32 MB
    beside the 8 MB reference transform, so every video is cut into slices of one track, each with its own
    reference transform."""
    monkeypatch.setenv("B2_BIG_WS_MB", "64")
    _sync_checked(handle, 21, list(enumerate([("mask", ["synthetic", "square_2048", "blocks"]),
                                              ("square_2048", ["impulse_2048", "synthetic", "one_cue"])])), 0.3)
