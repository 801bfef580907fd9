"""Both subtitle rasterisers checked frame for frame against the reference's cue arithmetic
(oracle/raster_oracle.py: timedelta scaling, Python round(), slice clamping) on the edge catalogue of
tests/test_raster_cpu.py: half-microsecond ties, half-frame starts and durations, every slice case,
bit-packing edges and cue times near 2 h and 10 h.

  * K2 (raster_cues_kernel, b2_rasterize) directly: every element equals np.float32 of the oracle's signal
    (shared and per-pair ratios, explicit levels, cue_keep, empty tracks); the lengths equal the oracle's
    and b2_first_last_nonzero equals its frame boundaries.
  * K2b (raster_bits_kernel) through the run path of the aligner: with a reference at least as long as the
    mask (R >= S) and offset 0 inside the window, every mask frame lies in the overlap at offset 0, so one
    wrong frame moves that offset's score by 2 (+-1 jobs) or by at least 2 * level * |2 label - 1| - far
    outside the run path's eps.  The capture of every offset is checked against exact integer counts of
    the oracle raster (tests/test_gpu_runcorr_exact.py), which makes it a frame-for-frame check of the mask.
  * The float-signal path (B2_FUSED_RASTER=0) returns the default's per-ratio outputs bit for bit wherever
    neither nominates more candidates than the re-score takes.
  * Inputs the arithmetic does not reproduce are rejected, and frame boundaries of a float64 level just
    above 0.5 are the reference's."""
import collections
import time
from datetime import timedelta

import numpy as np
import pytest

import test_gpu_runcorr_exact as rx
import test_raster_cpu as rc
from oracle import raster_oracle as ro

pytestmark = pytest.mark.gpu

RATIOS = rc.RATIOS
K_CAND = 32


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module", autouse=True)
def report_time():
    t0 = time.time()
    yield
    print("test_gpu_raster_exact: %.1f s" % (time.time() - t0))


# ------------------------------------------------------------------------------------------ cue lists

def _track(st, en, keep=None, video=0):
    st, en = np.asarray(st, np.float64), np.asarray(en, np.float64)
    keep = np.ones(len(st), np.uint8) if keep is None else np.asarray(keep, np.uint8)
    return dict(st=st, en=en, keep=keep, video=video)


def _cat(*tracks, video=0):
    return _track(np.concatenate([t["st"] for t in tracks]), np.concatenate([t["en"] for t in tracks]),
                  np.concatenate([t["keep"] for t in tracks]), video)


def _frames(spans, r, ss=0.0):
    """Cues whose frames at ratio r are exactly the spans [a, b) (times 0.3 frame early)."""
    a = np.array([s[0] for s in spans], np.float64)
    b = np.array([s[1] for s in spans], np.float64)
    return _track(((a - 0.3) / 100.0 + ss) / r, ((b - 0.3) / 100.0 + ss) / r)


def _packing_spans(base, long_words=3000):
    """Bit-packing edges from frame `base` on: one-frame cues at both ends of words, a cue of exactly one
    word, cues from the last bit of a word to the first of the next, a cue spanning `long_words` words and
    29 overlapping cues OR-ed into one word."""
    w = base // 32 + 2
    spans = []
    for i in range(4):
        a = 32 * (w + 3 * i)
        spans += [(a, a + 1), (a + 31, a + 32), (a + 64, a + 96), (a + 95, a + 97)]
    w += 20
    spans.append((32 * w + 5, 32 * (w + long_words) + 17))
    w += long_words + 10
    spans += [(32 * w + i, 32 * w + i + 1 + i % 3) for i in range(29)]
    spans += [(32 * w + 2, 32 * w + 30), (32 * (w + 2), 32 * (w + 2) + 32)]
    return spans, 32 * (w + 4)


def _ties(rng, r, W_lo, W_hi, n_try, cap, keep_frac=0.9):
    """Cues with a half-microsecond tie at the start, at the end, or both; half of the ties at a half frame."""
    t = np.concatenate([rc.half_us_times(rng, r, W_lo, W_hi, n_try)[:cap // 2],
                        rc.half_us_times(rng, r, W_lo, W_hi, n_try, half_frame=True)[:cap - cap // 2]])
    # short cues, so that few frames are covered twice and a moved edge shows in the raster
    d = rng.uniform(0.01, 0.3, len(t))
    s = np.sort(t)
    pair = np.flatnonzero(np.diff(s)[::2] < 0.5) * 2          # both ends ties: neighbouring ties
    st = np.concatenate([t, t - d, s[pair]])
    en = np.concatenate([t + d, t, s[pair + 1]])
    return _track(st, en, (rng.rand(len(st)) < keep_frac).astype(np.uint8))


def _k2_tracks(rng, ss):
    """The catalogue as cue lists for b2_rasterize at start_seconds ss."""
    tracks = []
    for r in RATIOS:
        tracks.append(_cat(_ties(rng, r, 0, 600, 100000, 300), _track(*rc.half_frame_cues(rng, r, ss, 300, 0, 60000))))
        spans, _ = _packing_spans(1000)
        tracks.append(_frames(spans, r, ss))
    # slice cases (frames below -n, in [-n, -1], at and past n, last past n, negative durations)
    for n in (2, 50, 1000):
        st, en = rc.slice_case_cues(rng, 1.0, ss, n, 300)
        tracks.append(_track(st, en, (rng.rand(len(st)) < 0.9).astype(np.uint8)))
    # 10 h
    st, en = rc.long_time_cues(rng, 1.0, 36000.0, 300)
    tracks.append(_track(st, en))
    # a start far before start_seconds (clamps to 0), one just before it (wraps), one past the end of the
    # signal (clamps to n) with a negative duration
    tracks.append(_track([-20.0, ss - 0.5, ss + 0.2, ss + 30.0], [ss + 1.0, ss - 0.2, ss + 1.0, ss + 0.1]))
    # empty, all dropped, and a dropped cue that sets the length
    tracks.append(_track([], []))
    tracks.append(_track([1.0, 2.0], [1.5, 3.0], [0, 0]))
    tracks.append(_track([1.0, 2.0, 9.0], [1.5, 3.0, 9.5], [1, 1, 0]))
    return tracks


def _flatten(tracks):
    cs = np.concatenate([t["st"] for t in tracks])
    ce = np.concatenate([t["en"] for t in tracks])
    keep = np.concatenate([t["keep"] for t in tracks])
    off = np.concatenate([[0], np.cumsum([len(t["st"]) for t in tracks])]).astype(np.int64)
    return cs, ce, keep, off


def _oracle(t, r, ss):
    return ro.rasterize(t["st"], t["en"], t["keep"].astype(bool), 100, ss, r)[0]


def _raw_first(t, r, ss):
    return np.array([int(round((ro.scale_seconds(s, r) - ss) * 100)) for s in t["st"].tolist()], np.int64)


# ------------------------------------------------------------------------------------------ K2

def _check_k2(handle, tracks, ratios, K, per_pair, ss, levels=None, where=""):
    cs, ce, keep, cue_off = _flatten(tracks)
    out, off = handle.rasterize(cs, ce, keep, cue_off, ratios, K, per_pair, 100, ss, levels=levels)
    first, last = handle.first_last_nonzero(out, off)
    for b, t in enumerate(tracks):
        for k in range(K):
            j = b * K + k
            r = float(ratios[j] if per_pair else ratios[k])
            want = _oracle(t, r, ss)
            got = out[off[j]:off[j + 1]]
            at = (where, ss, b, k, r)
            assert len(got) == len(want), (at, len(got), len(want))
            lv = None if levels is None else levels[j if per_pair else k]
            exp = want.astype(np.float32) if lv is None else np.where(want != 0, np.float32(lv), np.float32(0))
            bad = np.flatnonzero(got != exp)
            assert len(bad) == 0, (at, len(bad), bad[:8].tolist(), got[bad[:8]].tolist(), exp[bad[:8]].tolist())
            f0, f1 = ro.frame_boundaries(want if levels is None else exp.astype(np.float64))
            assert (int(first[j]), int(last[j])) == ((-1, -1) if f0 is None else (f0, f1)), at


@pytest.mark.parametrize("ss", rc.START_SECONDS)
def test_k2_element_for_element(handle, ss):
    rng = np.random.RandomState(int(ss * 1000) + 1)
    tracks = _k2_tracks(rng, ss)
    # shared ratios
    _check_k2(handle, tracks, np.array(RATIOS), len(RATIOS), False, ss, where="shared")
    # per-pair ratios (the golden-section search's shape): each pair its own 3 ratios, two of them off-grid
    K = 3
    pr = np.array([[r, r * (1 + 1e-7 * (b + 1)), rng.uniform(0.9, 1.1)] for b, r in
                   zip(range(len(tracks)), np.resize(RATIOS, len(tracks)))]).ravel()
    _check_k2(handle, tracks, pr, K, True, ss, where="per-pair")
    # explicit levels (SubtitleSpeechTransformer alone: ratio 1, the level of the scaled ratio), shared and
    # per pair
    _check_k2(handle, tracks, np.array([1.0, 1.1]), 2, False, ss, levels=np.array([0.75, 0.501]), where="levels")
    lv = rng.uniform(0.05, 1.0, len(tracks) * K)
    _check_k2(handle, tracks, pr, K, True, ss, levels=lv, where="per-pair levels")

    # the catalogue reaches the slice cases and both parities of the rounding ties
    firsts = []
    for t in tracks:
        n = len(_oracle(t, 1.0, ss))
        f = _raw_first(t, 1.0, ss)
        firsts.append((f, n))
    assert any(np.any(f < -n) for f, n in firsts) and any(np.any((f >= -n) & (f < 0)) for f, n in firsts)
    assert any(np.any(f > n) for f, n in firsts)


def test_k2_rejects_inputs_the_arithmetic_does_not_reproduce(handle):
    from ffsubsync_b200 import _native
    st, en, keep, off = np.array([1.0, 2.0]), np.array([1.5, 3.0]), np.array([1, 0], np.uint8), [0, 2]
    out_off = np.array([0, 400], np.int64)
    L = rc.MAX_CUE_SECONDS

    def call(st=st, en=en, ratios=(1.0,), ss=0.0):
        return handle.rasterize(np.asarray(st), np.asarray(en), keep, off, np.asarray(ratios), len(ratios), False, 100,
                                ss, out_off=out_off)

    call()
    bad = [dict(st=[1.0, np.nan]), dict(st=[np.inf, 2.0]), dict(en=[1.5, -np.inf]), dict(st=[1.0, L]),
           dict(st=[L / 2, 2.0], ratios=(1.0, 2.0)), dict(ratios=(0.0,)), dict(ratios=(-1.0,)),
           dict(ratios=(np.nan,)), dict(ratios=(np.inf,)), dict(ss=np.nan), dict(ss=L), dict(ss=-np.inf)]
    for kw in bad:
        with pytest.raises(_native.NativeError) as e:
            call(**kw)
        assert e.value.status == -1 and "rasterize:" in str(e.value), kw
    # the reference raises for the same cue times
    with pytest.raises((ValueError, OverflowError)):
        ro.scale_seconds(float("nan"), 1.0)


def test_sync_rejects_bad_cue_times(handle):
    """b2_sync_tracks and b2_sync_batch reject a non-finite start of a dropped cue (the reference's scaler
    raises for every cue) and a start_seconds beyond the limit, before any work is queued."""
    from ffsubsync_b200 import _native
    pcm = handle.synth_pcm(np.ones(300, np.uint8), 300, 160, 1)
    off = np.array([0, len(pcm)], np.int64)
    st, en, keep = np.array([0.5, np.nan]), np.array([1.0, 2.0]), np.array([1, 0], np.uint8)
    cue_off = np.array([0, 2], np.int64)
    for kw in (dict(st=st, ss=0.0), dict(st=np.array([0.5, 1.0]), ss=np.inf)):
        with pytest.raises(_native.NativeError) as e:
            handle.sync_tracks(pcm, off, [0], 16000, 100, 0.0, 100000, -1, -1, kw["st"], en, keep, cue_off, [1.0],
                               kw["ss"], 100)
        assert e.value.status == -1 and "sync_tracks:" in str(e.value)
        with pytest.raises(_native.NativeError) as e:
            handle.sync_batch(pcm, off, 16000, 100, 0.0, 100000, -1, -1, kw["st"], en, keep, cue_off, [1.0],
                              kw["ss"], 100)
        assert e.value.status == -1 and "sync_batch:" in str(e.value)
    with pytest.raises(_native.NativeError):
        handle.sync_batch(pcm, off, 16000, 100, 0.0, 100000, -1, -1, st[:1], en[:1], keep[:1], [0, 1], [1.0, np.inf],
                          0.0, 100)


_Sub = collections.namedtuple("_Sub", "start end content")


@pytest.mark.parametrize("ratio", [1.99999998, 2.0])
def test_frame_boundaries_of_a_level_just_above_one_half(handle, ratio):
    """Level min(1/r, 1) = 0.500000005 at r = 1.99999998: above 0.5 in float64 (speech frames), 0.5f in
    float32.  At r = 2 the level is 0.5: no speech frame."""
    from ffsubsync_b200.speech_transformers import SubtitleSpeechTransformer
    subs = [_Sub(timedelta(seconds=1.0), timedelta(seconds=2.5), "hello"),
            _Sub(timedelta(seconds=4.0), timedelta(seconds=4.2), "again")]
    tr = SubtitleSpeechTransformer(100, 0, ratio).fit(subs)
    want, _, f0, f1 = ro.rasterize([1.0, 4.0], [2.5, 4.2], None, 100, 0, ratio, scale=False)
    assert np.array_equal(tr.transform(), want)
    assert (tr.start_frame_, tr.end_frame_) == (f0, f1)
    assert (f0 is None) == (ratio == 2.0)


# ------------------------------------------------------------------------------------------ K2b

MOS = 2000


def _check_premise(call, label):
    assert label != 0.5
    for jb in call.jobs:
        assert jb.live and jb.R >= jb.S and jb.o_lo <= 0 <= jb.o_hi, (jb.R, jb.S, jb.o_lo, jb.o_hi)
        assert len(jb.u) == jb.S


def _check_runs(call, label, where, batch=False):
    """The run path's capture at every offset against the exact counts of the oracle raster, and the proof
    that the run path ran: every job's eps is rc_eps."""
    _check_premise(call, label)
    assert max(len(t["st"]) for t in call.tracks) <= 16384
    assert max(jb.o_hi - jb.o_lo + 1 for jb in call.jobs) <= 32768
    with rx._env(B2_ALIGN_PATH="runs"):
        cap, out, _ = call.capture(True, batch)
    for j, jb in enumerate(call.jobs):
        assert cap["stat"][j][1] == np.float32(jb.eps), (where, j, cap["stat"][j][1], jb.eps)
    rx._check_capture(cap, call.jobs, call.K, call.mos, False, where)
    return cap, out


def _short_tracks(rng, v, ss, R):
    """The catalogue on a reference of R frames: per ratio r, ties and half frames and bit packing at r (their
    positions scaled by r / max ratio, so that every ratio's mask fits the reference), slice cases."""
    tracks = []
    top = (R - 400) / 100.0
    for i, r in enumerate(RATIOS):
        f = r / max(RATIOS)
        a = _ties(rng, r, 1, int(top * 0.9 * f), 60000, 200)
        b = _track(*rc.half_frame_cues(rng, r, ss, 200, 0, int((top - ss) * 90 * f)))
        spans, end = _packing_spans(1000 + 200 * i, 150)
        assert end < (R - 400) * f
        c = _frames(spans, r, ss)
        t = _cat(a, b, c, video=v)
        tracks.append(t)
    st, en = rc.slice_case_cues(rng, 1.0, ss, 300, 200)
    tracks.append(_track(st, en, (rng.rand(len(st)) < 0.9).astype(np.uint8), video=v))
    # a track whose longest cue is dropped, and one of one frame at frame 0
    tracks.append(_track([0.5, 1.0, 20.0], [0.9, 1.3, 25.0], [1, 1, 0], video=v))
    tracks.append(_track([0.0], [0.007], video=v))
    return tracks


def _short_call(handle, label, ss, seed, n_videos=3, R=26000):
    rng = np.random.RandomState(seed)
    pcms, tracks = [], []
    for v in range(n_videos):
        pcms.append(rx._pcm(handle, rx._mask_cls(rng.rand(R) < 0.5, rng), seed * 10 + v))
        tracks += _short_tracks(rng, v, ss, R)
    return rx._Call(handle, pcms, tracks, RATIOS, label, MOS, start_seconds=ss)


def test_k2b_frame_for_frame_through_the_run_path(handle):
    call = _short_call(handle, 0.0, 0.0, 5)
    assert sum(jb.pm1 for jb in call.jobs) >= len(call.jobs) // 2
    _check_runs(call, 0.0, ("short", 0.0))
    # the same inputs through b2_sync_batch (one video per track)
    _check_runs(call, 0.0, ("short", "sync_batch"), batch=True)


def test_k2b_sub_batches_and_start_seconds(handle):
    """Sliced cue_off / sig_off tables (three sub-batches), cues before start_seconds (wrapped to the end of
    the mask) and a label that makes no job +-1 for ratios above 1."""
    call = _short_call(handle, 0.3, 12.345, 6)
    assert any(((_raw_first(t, 1.0, 12.345) < 0) & (t["keep"] != 0)).any() for t in call.tracks)
    with rx._env(B2_SUBBATCHES=3, B2_VAD_SMS=60):
        _check_runs(call, 0.3, ("sub-batches", 12.345))


def test_k2b_two_hour_video_several_tracks(handle):
    """One 2 h video (7 205 s of PCM), one track per ratio with cue times up to 7 204 s: ties near 7 200 s, half
    frames and bit packing near the end, a cue of 3 000 words."""
    rng = np.random.RandomState(7200)
    R = 720500
    ratios = [1.0, 24.0 / 25.0, 23.976 / 24.0]
    pcms = [rx._pcm(handle, rx._mask_cls(rng.rand(R) < 0.45, rng), 7201)]
    tracks = []
    for r in ratios:
        f = r / max(ratios)          # at the largest ratio every track's cues reach 7 199 s
        a = _ties(rng, r, int(7000 * f), int(7190 * f), 400000, 300)
        b = _track(*rc.long_time_cues(rng, r, 7199.0 * f, 300))
        c = _track(*rc.half_frame_cues(rng, r, 0.0, 300, int(700000 * f), int(719000 * f)))
        spans, _ = _packing_spans(int(600000 * f))
        d = _frames(spans, r)
        tracks.append(_cat(a, b, c, d))
    call = rx._Call(handle, pcms, tracks, ratios, 0.0, MOS)
    assert max(float(np.max(t["en"] * r)) for t, r in zip(tracks, ratios)) > 7199.0
    _check_runs(call, 0.0, ("2 h",))


# ------------------------------------------------------------------------------------------ cross-check

def test_float_signal_path_matches_the_bit_masks(handle):
    """Per-ratio outputs of B2_FUSED_RASTER=0 (K2 floats, generic aligner) equal the default (K2b bit masks)
    bit for bit wherever neither run nominates more offsets than the re-score takes."""
    call = _short_call(handle, 0.0, 0.3, 8, n_videos=2)
    cap_d, out_d, _ = call.capture(True)
    with rx._env(B2_FUSED_RASTER=0):
        cap_f, out_f, _ = call.capture(True)
    ok = (cap_d["cand"] <= K_CAND) & (cap_d["cand"] >= 0) & (cap_f["cand"] <= K_CAND) & (cap_f["cand"] >= 0)
    assert ok.sum() >= len(call.jobs) // 2, ok.sum()
    for j in np.flatnonzero(ok):
        assert out_d[3][j] == out_f[3][j] and out_d[4][j] == out_f[4][j], (j, out_d[3][j], out_f[3][j])
