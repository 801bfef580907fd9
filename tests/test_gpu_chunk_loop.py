"""GPU tests of the reference's chunk loop in every batched reference (run on an H100).

The reference reads (2 fr // sr) * 10000 bytes at a time and calls the detector once per read; every call has its own
window grid and its own partial last window (oracle/chunk_oracle.py).  Every reference a batched call builds -
b2_sync_tracks, _gss, _auditok under B2_HOST, B2_DEVICE and resident calls, the run path, a sampled segment longer than
one call, the ingest session and its segments under 100 s reads, window- and call-straddling pushes and 1-byte pushes
across the call boundaries - is compared frame for frame, bit-exact, with chunk_oracle.chunk_loop rounded once to
float32, read through b2_capture_reference or b2_speech_output.  So are VideoSpeechTransformer("energy_zcr") and
b2_vad_stream_*.

Rates: 8 and 16 kHz on the lane kernel (video lengths rounded to 8 samples, so every video stays eligible), 16 kHz on
the lane-group kernel, 11.025, 22.05, 32, 44.1 and 48 kHz.  Only at 22.05 kHz does a call (2 205 000 samples) not
divide into windows (221 samples).  Video lengths: 0, under one window, one call and one call +- 1 sample, two
calls, a call plus a partial window, 2.5 calls.  Around every call boundary the PCM is engineered so that a wrong grid
fails deterministically: windows that are speech on the per-call grid and not on the one-call grid, and the reverse.
At 22.05 kHz the sync results must also equal the oracle pipeline (fft_align per ratio, MaxScoreAligner's rule),
offsets exactly or tied under exact_score."""
import numpy as np
import pytest

import test_gpu_ingest as gi
import test_gpu_reference_exact as rx
from oracle import aligner_oracle as ao
from oracle import chunk_oracle as co
from oracle import raster_oracle as ro
from oracle import segment_oracle as so
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

THR = rx.THR
RATES = {"8k": (8000, None), "16k": (16000, None), "16k-group": (16000, "group"), "11.025k": (11025, None),
         "22.05k": (22050, None), "32k": (32000, None), "44.1k": (44100, None), "48k": (48000, None)}
DETECTORS = [("energy", 0.0), ("energy", 0.3), ("auditok", 0.0), ("auditok", 0.3)]
LOUD = 360   # a square wave of this amplitude: mean square 129 600, speech over a whole window only (threshold 10^5)


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _lengths(fr, aligned):
    fpw, C = vo.frames_per_window(fr, 100), co.read_samples(fr)
    d = 8 if aligned else 1
    return [0, fpw - d, C - d, C, C + d, 2 * C, C + (fpw // 2) // d * d, 5 * C // 2]


def _pattern(pcm, a, fpw, n_windows):
    """Windows [a + i fpw, a + (i+1) fpw) for i < n_windows: even ones a loud square wave, odd ones silent."""
    for i in range(n_windows):
        lo, hi = a + i * fpw, min(a + (i + 1) * fpw, len(pcm))
        if lo >= hi:
            return
        pos = np.arange(hi - lo)
        pcm[lo:hi] = np.where(i % 2 == 0, np.where((pos // 40) % 2 == 0, LOUD, -LOUD), 0).astype(np.int16)


def _engineer(pcm, fr):
    """After every call boundary kC: 8 windows on the per-call grid (speech there; straddled, so not speech, on the
    one-call grid where the grids differ), then 8 windows on the one-call grid (the reverse)."""
    fpw, C = vo.frames_per_window(fr, 100), co.read_samples(fr)
    for b in range(C, len(pcm), C):
        _pattern(pcm, b, fpw, 8)
        _pattern(pcm, -(-(b + 9 * fpw) // fpw) * fpw, fpw, 8)
    return pcm


_CORPORA = {}


def _corpus(cfg):
    if cfg not in _CORPORA:
        fr, layout = RATES[cfg]
        aligned = cfg in ("8k", "16k")
        c = rx._corpus([dict(kind="audio", n=n, tracks=1) for n in _lengths(fr, aligned)], fr, 700 + fr % 113)
        c["pcms"] = [_engineer(p.copy(), fr) for p in c["pcms"]]
        c["pcm"] = np.concatenate(c["pcms"]).astype(np.int16)
        _CORPORA[cfg] = c
    return _CORPORA[cfg]


def _want(c, detector, label):
    det = "auditok" if detector == "auditok" else "energy_zcr"
    kw = {} if detector == "auditok" else dict(energy_threshold=THR)
    return [co.chunk_loop(det, p, c["fr"], 100, label, **kw).astype(np.float32) for p in c["pcms"]]


def _knobs(cfg, **kw):
    if RATES[cfg][1]:
        kw["B2_VAD_LAYOUT"] = RATES[cfg][1]
    return kw


def test_premise_engineered_boundaries():
    """At 22.05 kHz the engineered windows make the one-call grid and the per-call grid disagree right after every call
    boundary; at 16 kHz they agree."""
    for cfg, differs in (("22.05k", True), ("16k", False)):
        c = _corpus(cfg)
        fr, C = c["fr"], co.read_samples(c["fr"])
        for p in c["pcms"]:
            if len(p) <= C:
                continue
            loop = co.chunk_loop("energy_zcr", p, fr, 100, 0.0)
            one = vo.energy_zcr_detect(p, 100, fr, 0.0)
            k = -(-C // vo.frames_per_window(fr, 100))   # the first frame of the second call
            assert (not np.array_equal(loop[k: k + 8], one[k: k + 8])) == differs, cfg
            assert (len(loop) != len(one)) == differs or len(p) % C == 0


# ------------------------------------------------------------------------- whole calls, every rate

@pytest.mark.parametrize("detector,label", DETECTORS)
@pytest.mark.parametrize("cfg", list(RATES))
def test_references_follow_the_chunk_loop(handle, cfg, detector, label):
    c = _corpus(cfg)
    want = _want(c, detector, label)
    entry = "auditok" if detector == "auditok" else "tracks"
    with rx._env(**_knobs(cfg)):
        cap = rx._captured(handle, c, want, lambda keep: rx._call(handle, c, entry, label, detector=detector))
    rx._check(cap, want, where=(cfg, detector, label))


@pytest.mark.parametrize("memspace", ["host", "device", "resident"])
@pytest.mark.parametrize("entry", ["tracks", "gss", "auditok"])
@pytest.mark.parametrize("cfg", ["22.05k", "16k"])
def test_entry_points_and_memory(handle, cfg, entry, memspace):
    from ffsubsync_b200 import _native as N
    ms = {"host": N.B2_HOST, "device": N.B2_DEVICE, "resident": N.B2_DEVICE_RESIDENT}[memspace]
    c = _corpus(cfg)
    detector = "auditok" if entry == "auditok" else "energy"
    want = _want(c, detector, 0.0)
    cap = rx._captured(handle, c, want, lambda keep: rx._call(handle, c, entry, 0.0, ms, detector=detector, keep=keep))
    rx._check(cap, want, where=(cfg, entry, memspace))


def _check_sync(c, res, want, label):
    """best_* and all_* of a sync_tracks-like result against fft_align on the chunk-loop references and
    MaxScoreAligner's rule: offsets equal or tied under exact_score, scores within 1e-5.  With the search (all_* rows
    of K + 1) its column and a winning search are left to the search's own suites."""
    bs, bo, bk, a_s, a_o = res[:5]
    K, W = len(rx.GRID), len(a_s) // len(c["tv"])
    for t, v in enumerate(c["tv"]):
        ref = want[v].astype(np.float64)
        cs, ce = (c[k][c["cue_off"][t]: c["cue_off"][t + 1]] for k in ("cs", "ce"))
        subs = [ro.rasterize(cs, ce, None, 100, 0.0, r)[0] for r in rx.GRID]
        if len(ref) == 0:   # the reference raises on an empty signal
            continue
        cands = [ao.fft_align(ref, s, rx.MOS) for s in subs]
        for k, (s, o) in enumerate(cands):
            got_o = int(a_o[t * W + k])
            tie = got_o == o or ao.exact_score(ref, subs[k], got_o) == ao.exact_score(ref, subs[k], o)
            assert tie, (t, k, got_o, o)
            got_s = a_s[t * W + k]
            assert got_s == s or abs(got_s - s) <= 1e-5 * max(1.0, abs(s)), (t, k, got_s, s)   # -inf: all masked
        k_or = ao.max_score_select(cands, rx.MOS)
        if bk[t] < K and (int(bk[t]), int(bo[t])) != (k_or, cands[k_or][1]):
            assert ao.exact_score(ref, subs[bk[t]], int(bo[t])) == ao.exact_score(ref, subs[k_or], cands[k_or][1]), t


@pytest.mark.parametrize("path", ["default", "runs"])
@pytest.mark.parametrize("detector,label", [("energy", 0.0), ("energy", 0.3), ("auditok", 0.0)])
def test_sync_results_at_22050(handle, detector, label, path):
    """Whole calls at 22.05 kHz against the oracle pipeline over the chunk loop; B2_ALIGN_PATH=runs takes the packed
    run path where it is eligible (the references stay floats: they are not whole videos of windows)."""
    c = _corpus("22.05k")
    want = _want(c, detector, label)
    entry = "auditok" if detector == "auditok" else "tracks"
    knobs = dict(B2_ALIGN_PATH="runs") if path == "runs" else {}
    with rx._env(**knobs):
        cap = rx._captured(handle, c, want, lambda keep: rx._call(handle, c, entry, label, detector=detector))
        res = rx._call(handle, c, entry, label, detector=detector)
    rx._check(cap, want, packed=False, where=(detector, label, path))
    _check_sync(c, res, want, label)


# ------------------------------------------------------------------------- sampled segments, ingest

def _speech(handle, V, run):
    """The references a call writes through b2_speech_output (videos 0 .. V-1)."""
    from ffsubsync_b200 import _native as N
    cap = 4 * 10 ** 6
    buf = np.full(cap, np.nan)
    off = np.full(V + 1, -1, np.int64)
    handle.speech_output(buf, cap, np.arange(V), off, N.B2_HOST)
    try:
        res = run()
    finally:
        handle.speech_output(None, 0, None, None)
    return buf, off, res


def _seg_case(fr):
    """One video of 260 s with a 230 s segment from 10 s (longer than a call), a short one, and an overlapping one."""
    n = 260 * fr
    pcm = _engineer(rx._audio(n, fr, 91), fr)
    starts, lo, hi = [10, 245, 250], [10 * fr + 3, 245 * fr, 250 * fr], [240 * fr, 246 * fr, 260 * fr]
    return pcm, 260.0, np.array(starts), np.array(lo), np.array(hi)


@pytest.mark.parametrize("detector,label", [("energy", 0.0), ("energy", 0.3), ("auditok", 0.0)])
@pytest.mark.parametrize("fr", [22050, 16000])
def test_segment_longer_than_a_call(handle, fr, detector, label):
    from ffsubsync_b200 import _native as N
    pcm, total, starts, lo, hi = _seg_case(fr)
    chunk = co.read_samples(fr)
    det = dict(detector="auditok", chunk_samples=chunk) if detector == "auditok" else dict(energy_threshold=THR)
    want = so.segment_reference(pcm, total, starts, lo, hi, 100, frame_rate=fr, non_speech_label=label, **det)
    want = want.astype(np.float32).astype(np.float64)
    cs, ce = rx._track_cues(5)
    args = dict(detector=N.B2_DETECTOR_AUDITOK if detector == "auditok" else N.B2_DETECTOR_ENERGY_ZCR,
                energy_threshold=THR, chunk_samples=chunk)
    buf, off, _ = _speech(handle, 1, lambda: handle.sync_tracks_seg(
        pcm, [0, len(pcm)], [0], fr, 100, label, [0], [total], [0, 3], starts, lo, hi, cs, ce, None, [0, len(cs)],
        rx.GRID, 0.0, rx.MOS, **args))
    assert off.tolist() == [0, len(want)]
    assert np.array_equal(buf[: len(want)], want), np.flatnonzero(buf[: len(want)] != want)[:8]


def _ingest_refs(handle, videos, fr, detector, label, kind, seed):
    chunk = co.read_samples(fr)
    gi._begin(handle, detector == "auditok", label, chunk if detector == "auditok" else 0, len(videos), fr=fr)
    if kind == "boundary-bytes":   # large pushes up to 300 samples before each call boundary, then 1-byte pushes
        for v, p in enumerate(videos):
            raw, at = p.tobytes(), 0
            for b in list(range(2 * chunk, 2 * len(p), 2 * chunk)) + [len(raw)]:
                handle.ingest_push([v], [raw[at: max(at, b - 600)]])
                at = max(at, b - 600)
                for i in range(at, min(b + 600, len(raw))):
                    handle.ingest_push([v], [raw[i: i + 1]])
                at = min(b + 600, len(raw))
    else:
        gi._push_all(lambda v, c: handle.ingest_push([v], [c]), handle.ingest_push, videos, kind, seed, 2 * chunk,
                     vo.frames_per_window(fr, 100))
    return gi._speech_only(handle, len(videos))


@pytest.mark.parametrize("kind", ["100s", "straddle", "boundary-bytes"])
@pytest.mark.parametrize("detector,label", DETECTORS)
@pytest.mark.parametrize("cfg", ["22.05k", "16k", "44.1k"])
def test_ingest_session(handle, cfg, detector, label, kind):
    """The session's references under every push pattern against the chunk loop, and at 22.05 kHz its sync results
    (label 0) against the whole call's."""
    c = _corpus(cfg)
    fr = c["fr"]
    want = _want(c, detector, label)
    buf, off = _ingest_refs(handle, c["pcms"], fr, detector, label, kind, 3)
    assert off.tolist() == np.concatenate([[0], np.cumsum([len(w) for w in want])]).tolist(), kind
    assert np.array_equal(buf[: off[-1]], np.concatenate(want).astype(np.float64)), kind


@pytest.mark.parametrize("detector,gss", [("energy", False), ("energy", True), ("auditok", False)])
def test_ingest_sync_at_22050(handle, detector, gss):
    """The session's sync results at 22.05 kHz equal the whole call's (gi._check_sync), which equal the oracle
    pipeline (test_sync_results_at_22050)."""
    c = _corpus("22.05k")
    chunk = co.read_samples(22050)
    gi._check_sync(handle, c["pcms"], detector == "auditok", chunk if detector == "auditok" else 0, 0.0, gss,
                   fr=22050, kinds=("straddle", "100s"))


@pytest.mark.parametrize("detector", ["energy", "auditok"])
@pytest.mark.parametrize("fr", [22050, 16000])
def test_ingest_segment_longer_than_a_call(handle, fr, detector):
    from ffsubsync_b200 import _native as N
    pcm, total, starts, lo, hi = _seg_case(fr)
    chunk = co.read_samples(fr)
    det = dict(detector="auditok", chunk_samples=chunk) if detector == "auditok" else dict(energy_threshold=THR)
    want = so.segment_reference(pcm, total, starts, lo, hi, 100, frame_rate=fr, non_speech_label=0.0, **det)
    want = want.astype(np.float32).astype(np.float64)
    gi._begin(handle, detector == "auditok", 0.0, chunk if detector == "auditok" else 0, 1, fr=fr)
    handle.ingest_segments([0], [total], [0, 3], starts)
    rng = np.random.RandomState(fr)
    for j in range(3):
        raw, at = pcm[lo[j]: hi[j]].tobytes(), 0
        while at < len(raw):   # window- and call-straddling pushes
            m = int(rng.choice([2 * 221 * 3 + 7, 2 * chunk - 3, 2 * chunk + 443, 2 * 221 * 1000 - 1]))
            handle.ingest_push([0], [raw[at: at + m]], segments=[j])
            at += m
    buf, off = gi._speech_only(handle, 1)
    assert off.tolist() == [0, len(want)]
    assert np.array_equal(buf[: len(want)], want), np.flatnonzero(buf[: len(want)] != want)[:8]


# ------------------------------------------------------------------------- the Python layer's own chunk loop

@pytest.mark.parametrize("cfg", ["22.05k", "16k"])
def test_video_speech_transformer_and_stream(handle, cfg):
    from ffsubsync_b200.speech_transformers import VideoSpeechTransformer
    c = _corpus(cfg)
    fr = c["fr"]
    p = max(c["pcms"], key=len)
    want = co.chunk_loop("energy_zcr", p, fr, 100, 0.0, energy_threshold=THR)
    t = VideoSpeechTransformer("energy_zcr", 100, fr, 0.0)
    t.fit(p.tobytes())
    assert np.array_equal(np.asarray(t.transform(), np.float64), want)
    handle.vad_stream_begin(fr, 100, 0.0, THR)
    raw, step = p.tobytes(), 2 * co.read_samples(fr)
    for i in range(0, len(raw), step):
        handle.vad_stream_push(raw[i: i + step])
    assert np.array_equal(handle.vad_stream_end().astype(np.float64), want)


# kernel launches of one B2_HOST call over the 16 / 48 kHz corpora, as the one-call tables launch them (H100)
LAUNCHES = {"tracks": 8, "gss": 112, "auditok": 9}


@pytest.mark.parametrize("entry", ["tracks", "gss", "auditok"])
@pytest.mark.parametrize("cfg", ["16k", "48k"])
def test_launches_and_results_unchanged_where_calls_divide(handle, cfg, entry):
    """Where the calls divide into windows the batched calls keep one detector entry per video: the same launches as
    before, and results equal to the oracle pipeline over the one-call detector."""
    c = _corpus(cfg)
    detector = "auditok" if entry == "auditok" else "energy"
    rx._call(handle, c, entry, 0.0, detector=detector)
    n0 = handle.launch_count
    res = rx._call(handle, c, entry, 0.0, detector=detector)
    handle.synchronize()
    assert handle.launch_count - n0 == LAUNCHES[entry], (cfg, entry, handle.launch_count - n0)
    if detector == "energy":
        want = [vo.energy_zcr_detect(p, 100, c["fr"], 0.0, THR).astype(np.float32) for p in c["pcms"]]
    else:
        want = _want(c, detector, 0.0)
    _check_sync(c, res, want, 0.0)
