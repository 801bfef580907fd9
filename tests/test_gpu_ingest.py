"""GPU suite of the batched ingest session (b2_ingest_*, ``BatchSynchronizer.ingest``, ``batch.sync_media``).

Seeded videos of varied lengths - empty, under one window, ragged, two and more auditok detector calls - are pushed
under several cut patterns: 1-byte and odd pushes, window- and call-straddling pushes, the reference's 100 s reads, and
many videos per push call, interleaved.  Everything is compared bit for bit: the references (read through
b2_speech_output) with the one-shot detector over each video's bytes (energy / ZCR; auditok at 100 s calls and at a
call length that is not a multiple of the window), and the sync results (grid, several tracks per video, --gss,
label 0 and a non-zero label) with the non-streamed b2_sync_tracks* call over the same PCM back to back.  Further:
more pushes than staging slots with the caller overwriting its buffer at once, every refused call followed by a
session that works on the same handle, and the ffmpeg driver end to end with a stand-in ffmpeg."""
import ctypes
import stat

import numpy as np
import pytest

from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

FR, SR = 16000, 100
FPW = FR // SR
CHUNK_100S = 100 * FR
THR = 100000
GRID = np.array([0.96, 1.0, 1.04])
MAX_OFF = 6000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _videos(seed, lengths, fr=FR):
    rng = np.random.RandomState(seed)
    fpw = fr // SR
    out = []
    for i, n in enumerate(lengths):
        nw = -(-n // fpw)
        cls = np.repeat(rng.choice([0, 1, 2], size=-(-nw // 37) + 1, p=[0.45, 0.45, 0.1]), 37)[:nw].astype(np.uint8)
        out.append(vo.synth_pcm(cls, fpw, seed=seed * 31 + i)[:n])
    return out


# empty, under one window, ragged, more than two 100 s detector calls
LENGTHS = [0, 97, 7 * FR + 77, 2 * CHUNK_100S + 3 * FR + 5]


def _cuts(kind, nbytes, rng, chunk_bytes, FPW=FPW):
    """Push sizes (bytes) of one video's stream under a cut pattern (FPW: samples per window)."""
    sizes = []
    left = nbytes
    if kind == "bytes":      # 1-byte pushes, then odd pushes shorter than a window and longer ones
        first = min(left, 3001)
        sizes += [1] * first
        left -= first
        while left > 0:
            m = int(rng.choice([1, 3, 2 * FPW - 1, 2 * FPW * 40 + 1, 2 * FPW * 700 + 3]))
            sizes.append(min(m, left))
            left -= sizes[-1]
    elif kind == "straddle":   # every push splits a window and, now and then, a detector call
        while left > 0:
            m = int(rng.choice([2 * FPW * 3 + 7, chunk_bytes - 3, chunk_bytes + 2 * FPW + 1, 2 * FPW * 1000 - 1]))
            sizes.append(min(m, left))
            left -= sizes[-1]
    else:                      # the reference's 100 s reads
        while left > 0:
            sizes.append(min(2 * CHUNK_100S, left))
            left -= sizes[-1]
    return sizes


def _push_all(session_push, session_push_many, videos, kind, seed, chunk_bytes, fpw=FPW):
    """Pushes every video's bytes under a cut pattern, videos interleaved at random; "many": several videos (one of
    them twice) per push call."""
    rng = np.random.RandomState(seed)
    raw = [v.tobytes() for v in videos]
    pattern = "bytes" if kind == "many" else kind
    queues = [list(_cuts(pattern, len(b), rng, chunk_bytes, fpw)) for b in raw]
    at = [0] * len(raw)
    pending = [i for i in range(len(raw)) for _ in queues[i]]
    rng.shuffle(pending)

    def take(v):
        m = queues[v].pop(0)
        c = raw[v][at[v]: at[v] + m]
        at[v] += m
        return c

    if kind != "many":
        for v in pending:
            session_push(v, take(v))
    else:
        while pending:
            k = min(len(pending), int(rng.randint(1, 6)))
            group, pending = pending[:k], pending[k:]
            session_push_many(group, [take(v) for v in group])
    assert all(not q for q in queues) and at == [len(b) for b in raw]


def _begin(handle, auditok, label, chunk, V, expect=None, fr=FR):
    from ffsubsync_b200 import _native as N
    handle.ingest_begin(V, fr, SR, label, detector=N.B2_DETECTOR_AUDITOK if auditok else N.B2_DETECTOR_ENERGY_ZCR,
                        energy_threshold=THR, chunk_samples=chunk, expect_samples=expect)


def _one_shot(handle, videos, auditok, label, chunk, fr=FR):
    """The one-shot detector over each video's bytes, widened to float64 (auditok: rounded once to float32)."""
    pcm = np.concatenate(videos + [np.zeros(0, np.int16)])
    off = np.concatenate([[0], np.cumsum([len(v) for v in videos])]).astype(np.int64)
    if auditok:
        out, o = handle.vad_auditok(pcm, off, fr, SR, label, chunk_samples=chunk)
        return out.astype(np.float32).astype(np.float64), o
    out, o = handle.vad_energy_zcr(pcm, off, fr, SR, label, THR)
    return out.astype(np.float64), o


def _speech_only(handle, V):
    """The session's references through b2_speech_output on a call without tracks."""
    from ffsubsync_b200 import _native as N
    cap = 4 * 10 ** 6
    buf = np.full(cap, np.nan)
    off = np.full(V + 1, -1, np.int64)
    handle.speech_output(buf, cap, np.arange(V), off, N.B2_HOST)
    try:
        handle.ingest_sync_tracks(np.zeros(0, np.int32), np.zeros(0), np.zeros(0), None, [0], GRID, 0.0, MAX_OFF)
    finally:
        handle.speech_output(None, 0, None, None)
    return buf, off


DETECTORS = [(False, 0), (True, CHUNK_100S), (True, 1000)]   # energy / ZCR, auditok at 100 s and at 1000 samples


def _check_references(handle, videos, auditok, chunk, label, fr=FR, kinds=("bytes", "straddle", "100s", "many")):
    """The session's references under every cut pattern of `kinds` against the one-shot detector, bit for bit."""
    fpw = fr // SR
    want, want_off = _one_shot(handle, videos, auditok, label, chunk, fr)
    for i, kind in enumerate(kinds):
        _begin(handle, auditok, label, chunk, len(videos), expect=[len(v) // 2 for v in videos] if i % 2 else None,
               fr=fr)
        _push_all(lambda v, c: handle.ingest_push([v], [c]), handle.ingest_push, videos, kind, 10 + i,
                  2 * chunk or 2 * 100 * fr, fpw)
        got_w = handle.ingest_windows()
        full = np.diff(want_off)
        assert np.all((got_w == full) | (got_w == full - 1)), (kind, got_w, full)   # at most the unfinished window
        buf, off = _speech_only(handle, len(videos))
        assert np.array_equal(off, want_off), (kind, off, want_off)
        assert np.array_equal(buf[: off[-1]], want), kind
        assert np.all(np.isnan(buf[off[-1]: off[-1] + 16]))


@pytest.mark.parametrize("auditok,chunk", DETECTORS)
@pytest.mark.parametrize("label", [0.0, 0.3])
def test_references_equal_the_one_shot_detector_under_every_cut(handle, auditok, chunk, label):
    _check_references(handle, _videos(3, LENGTHS), auditok, chunk, label)


def _tracks(videos, seed, fr=FR):
    """Two tracks on the fourth video, one on each other video (the empty one included); with fewer videos the last
    one takes the rest."""
    rng = np.random.RandomState(seed)
    tv = np.minimum([0, 1, 2, 3, 3], len(videos) - 1).astype(np.int32)
    starts, ends, off = [], [], [0]
    for v in tv:
        dur = max(len(videos[v]) / fr, 2.0)
        s = np.sort(rng.uniform(0, dur, 12))
        starts += list(s)
        ends += list(s + rng.uniform(0.2, 2.5, 12))
        off.append(len(starts))
    return tv, np.array(starts), np.array(ends), np.array(off, np.int64)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


CASES = [  # (auditok, chunk, label, gss)
    (False, 0, 0.0, False), (False, 0, 0.3, False), (False, 0, 0.0, True), (True, CHUNK_100S, 0.0, False),
    (True, CHUNK_100S, 0.0, True), (True, 1000, 0.3, False), (True, 1000, 0.0, True)]


def _check_sync(handle, videos, auditok, chunk, label, gss, fr=FR, kinds=("many", "straddle", "100s")):
    """The session's sync results (best_*, all_*, gss_ratio / gss_evals with the search, the speech output) under
    every cut pattern of `kinds` against the non-streamed b2_sync_tracks* call over the same PCM, bit for bit."""
    from ffsubsync_b200 import _native as N
    fpw = fr // SR
    pcm = np.concatenate(videos)
    pcm_off = np.concatenate([[0], np.cumsum([len(v) for v in videos])]).astype(np.int64)
    tv, cs, ce, co = _tracks(videos, 7, fr)
    V = len(videos)
    cap = 4 * 10 ** 6

    def with_speech(call):
        buf = np.full(cap, np.nan)
        off = np.full(V + 1, -1, np.int64)
        handle.speech_output(buf, cap, np.arange(V), off, N.B2_HOST)
        try:
            res = call()
        finally:
            handle.speech_output(None, 0, None, None)
        return tuple(res) + (buf[: off[-1]], off)

    kw = dict(want_all=True)
    if auditok:
        want = with_speech(lambda: handle.sync_tracks_auditok(pcm, pcm_off, tv, fr, SR, label, cs, ce, None, co, GRID,
                                                              0.0, MAX_OFF, chunk, gss=gss, want_evals=gss, **kw))
    elif gss:
        want = with_speech(lambda: handle.sync_tracks_gss(pcm, pcm_off, tv, fr, SR, label, THR, -1, -1, cs, ce, None,
                                                          co, GRID, 0.0, MAX_OFF, want_evals=True, **kw))
    else:
        want = with_speech(lambda: handle.sync_tracks(pcm, pcm_off, tv, fr, SR, label, THR, -1, -1, cs, ce, None, co,
                                                      GRID, 0.0, MAX_OFF, **kw))
    assert np.any(want[2] >= 0)
    results = []
    for i, kind in enumerate(kinds):
        _begin(handle, auditok, label, chunk, V, fr=fr)
        _push_all(lambda v, c: handle.ingest_push([v], [c]), handle.ingest_push, videos, kind, 20 + i,
                  2 * chunk or 2 * 100 * fr, fpw)
        got = with_speech(lambda: handle.ingest_sync_tracks(tv, cs, ce, None, co, GRID, 0.0, MAX_OFF, gss=gss,
                                                            want_evals=gss, **kw))
        assert len(got) == len(want)
        for j, (a, b) in enumerate(zip(got, want)):
            assert _same(a, b), (kind, j, a, b)
        results.append(got)
    for r in results[1:]:   # every cut pattern gives the same results
        assert all(_same(a, b) for a, b in zip(r, results[0]))


@pytest.mark.parametrize("auditok,chunk,label,gss", CASES)
def test_sync_equals_the_non_streamed_call(handle, auditok, chunk, label, gss):
    _check_sync(handle, _videos(5, LENGTHS), auditok, chunk, label, gss)


# every length a multiple of the window and none a multiple of the detector call: the flush then closes each video's
# last call with nothing held back (no span of its own), one video alone and several
ALIGNED = [(CHUNK_100S, [CHUNK_100S + FPW * 501]), (CHUNK_100S, [FPW * 50, CHUNK_100S + FPW * 3, 2 * CHUNK_100S + FPW * 11]),
           (1000, [FPW * 1234]), (1000, [FPW * 77, FPW * 1234])]


@pytest.mark.parametrize("chunk,lengths", ALIGNED)
def test_window_aligned_videos_close_their_last_auditok_call(handle, chunk, lengths):
    videos = _videos(41, lengths)
    _check_references(handle, videos, True, chunk, 0.0, kinds=("straddle", "100s"))
    for gss in (False, True):
        _check_sync(handle, videos, True, chunk, 0.0, gss, kinds=("straddle", "100s"))


FR48 = 48000   # the reference's default --frame-rate: 480-sample windows, the lane-group / generic VAD kernels
LENGTHS48 = [0, 301, 7 * FR48 + 77, 2 * 100 * FR48 + 3 * FR48 + 5]


@pytest.mark.parametrize("auditok,chunk,label", [(False, 0, 0.0), (False, 0, 0.3), (True, 100 * FR48, 0.0),
                                                 (True, 1000, 0.3)])
def test_48k_references_equal_the_one_shot_detector(handle, auditok, chunk, label):
    _check_references(handle, _videos(43, LENGTHS48, FR48), auditok, chunk, label, fr=FR48)


@pytest.mark.parametrize("auditok,chunk,label,gss", [(False, 0, 0.0, False), (False, 0, 0.3, False),
                                                     (False, 0, 0.0, True), (True, 100 * FR48, 0.0, True),
                                                     (True, 1000, 0.3, False)])
def test_48k_sync_equals_the_non_streamed_call(handle, auditok, chunk, label, gss):
    _check_sync(handle, _videos(47, LENGTHS48, FR48), auditok, chunk, label, gss, fr=FR48)


def test_push_counts_bytes_of_any_buffer(handle):
    """memoryviews of int16 buffers, int16 arrays, uint8 arrays and bytes all count their bytes: the speech output the
    session sizes from them holds every frame."""
    from ffsubsync_b200.batch import BatchSynchronizer
    videos = _videos(53, [5 * FR + 33, 3 * FR + 160 * 2])
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, max_offset_seconds=60.0)
    want, want_off = _one_shot(bs.handle, videos, False, 0.0, 0)
    s = bs.ingest(2)
    a, b = videos
    s.push(0, memoryview(a[:1001]))
    s.push(0, a[1001:3000])
    s.push(0, a[3000:].view(np.uint8))
    s.push_many([1, 1], [b[:7].tobytes(), memoryview(b[7:])])
    tv, cs, ce, co = _tracks(videos, 3)
    got = s.sync_tracks(tv, cs, ce, co, speech_video=[0, 1])
    speech, off = got[-2], got[-1]
    assert np.array_equal(off, want_off) and np.array_equal(speech, want)


def test_device_outputs_through_the_synchronizer(handle):
    """BatchSynchronizer.ingest with out= tensors returns what sync_device_tracks returns; without, what
    sync_host_tracks returns (several tracks per video, the search, the speech output)."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    videos = _videos(9, LENGTHS)
    pcm = np.concatenate(videos)
    pcm_off = np.concatenate([[0], np.cumsum([len(v) for v in videos])]).astype(np.int64)
    tv, cs, ce, co = _tracks(videos, 11)
    T = len(tv)
    bs = BatchSynchronizer(list(GRID) + [None], frame_rate=FR, max_offset_seconds=60.0)
    want = bs.sync_host_tracks(pcm, pcm_off, tv, cs, ce, co, want_all=True, speech_video=[1, 3])
    s = bs.ingest(len(videos))
    _push_all(s.push, s.push_many, videos, "straddle", 4, 2 * CHUNK_100S)
    got = s.sync_tracks(tv, cs, ce, co, want_all=True, speech_video=[1, 3])
    assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want))
    dev = torch.device("cuda", bs.handle.device)
    out = {"best_score": torch.empty(T, dtype=torch.float64, device=dev),
           "best_offset": torch.empty(T, dtype=torch.int32, device=dev),
           "best_k": torch.empty(T, dtype=torch.int32, device=dev),
           "gss_ratio": torch.empty(T, dtype=torch.float64, device=dev)}
    s = bs.ingest(len(videos), expect_samples=[10] * len(videos))   # a hint far too small: the buffers grow
    _push_all(s.push, s.push_many, videos, "100s", 5, 2 * CHUNK_100S)
    s.sync_tracks(tv, cs, ce, co, out=out)
    torch.cuda.synchronize()
    for k, w in zip(("best_score", "best_offset", "best_k", "gss_ratio"), want[:3] + want[5:6]):
        assert _same(out[k].cpu().numpy(), w), k


def test_more_pushes_than_slots_with_the_buffer_overwritten_at_once(handle):
    """One caller buffer, refilled for every push and scribbled over right after it returns: the library copied it."""
    videos = _videos(13, [40 * FR + 3, 33 * FR + 160 * 7])
    want, _ = _one_shot(handle, videos, False, 0.0, 0)
    _begin(handle, False, 0.0, 0, 2)
    buf = np.empty(2 * FR * 3 + 1, np.uint8)
    raw = [v.tobytes() for v in videos]
    at = [0, 0]
    pushes = 0
    while at[0] < len(raw[0]) or at[1] < len(raw[1]):
        for v in (0, 1):
            m = min(len(buf) - (pushes % 5), len(raw[v]) - at[v])
            if m <= 0:
                continue
            buf[:m] = np.frombuffer(raw[v][at[v]: at[v] + m], np.uint8)
            handle.ingest_push([v], [buf[:m]])
            buf[:] = 0x5A
            at[v] += m
            pushes += 1
    assert pushes > 20
    got, off = _speech_only(handle, 2)
    assert np.array_equal(got[: off[-1]], want)


def test_refusals_leave_the_handle_usable(handle):
    from ffsubsync_b200 import _native as N
    lib, h = handle.lib, handle.h
    videos = _videos(17, [5 * FR + 3, 2 * FR])
    want, _ = _one_shot(handle, videos, False, 0.0, 0)

    def works():
        _begin(handle, False, 0.0, 0, 2)
        for v in (0, 1):
            handle.ingest_push([v], [videos[v].tobytes()])
        got, off = _speech_only(handle, 2)
        assert np.array_equal(got[: off[-1]], want)

    def refused(call, needle):
        with pytest.raises(N.NativeError) as e:
            call()
        assert e.value.status == -1 and needle in str(e.value), str(e.value)

    # without a session
    refused(lambda: handle.ingest_push([0], [b"ab"]), "no open session")
    refused(lambda: handle.ingest_windows(), "no open session")
    refused(lambda: handle.ingest_sync_tracks(np.zeros(0, np.int32), [], [], None, [0], GRID, 0.0, MAX_OFF),
            "no open session")
    works()
    # a second begin
    _begin(handle, False, 0.0, 0, 2)
    refused(lambda: _begin(handle, False, 0.0, 0, 2), "already open")
    handle.ingest_abort()
    works()
    # bad chunks: each refused call pushes nothing, and the session goes on
    _begin(handle, False, 0.0, 0, 2)
    handle.ingest_push([0], [videos[0].tobytes()[:1001]])
    refused(lambda: handle.ingest_push([0, 2], [b"ab", b"cd"]), "chunk 1: video 2 is out of [0, 2)")
    refused(lambda: handle.ingest_push([-1], [b"ab"]), "video -1")
    n = np.array([4, -2], np.int64)
    vid = np.array([1, 1], np.int32)
    data = np.zeros(4, np.uint8)
    ptrs = (ctypes.c_void_p * 2)(data.ctypes.data, data.ctypes.data)
    refused(lambda: handle._check(lib.b2_ingest_push(h, 2, vid.ctypes.data, ptrs, n.ctypes.data), "push"),
            "chunk 1: n_bytes = -2")
    n = np.array([4], np.int64)
    nulls = (ctypes.c_void_p * 1)(None)
    refused(lambda: handle._check(lib.b2_ingest_push(h, 1, vid.ctypes.data, nulls, n.ctypes.data), "push"),
            "chunk 0: null bytes")
    handle.ingest_push([0], [videos[0].tobytes()[1001:]])
    handle.ingest_push([1], [videos[1].tobytes()])
    got, off = _speech_only(handle, 2)
    assert np.array_equal(got[: off[-1]], want)
    works()
    # a detector argument the sync calls refuse, then a bad sync call: the session closes either way
    refused(lambda: handle.ingest_begin(2, FR, 0, 0.0), "bad frame_rate/sample_rate")
    _begin(handle, False, 0.0, 0, 2)
    refused(lambda: handle.ingest_sync_tracks(np.array([3], np.int32), [1.0], [2.0], None, [0, 1], GRID, 0.0, MAX_OFF),
            "track_video[0] = 3")
    refused(lambda: handle.ingest_push([0], [b"ab"]), "no open session")
    works()


_FAKE_FFMPEG = r'''#!/usr/bin/env python3
# stand-in for ffmpeg in tests: "decodes" the input file as raw s16le mono, honouring -ss / -t at the -ar rate
import sys
a = sys.argv[1:]
def hms(v):
    h, m, s = v.split(":")
    return int(h) * 3600 + int(m) * 60 + float(s)
rate = int(a[a.index("-ar") + 1])
ss = hms(a[a.index("-ss") + 1]) if "-ss" in a else 0.0
t = hms(a[a.index("-t") + 1]) if "-t" in a else None
assert a[-1] == "-" and "s16le" in a
data = open(a[a.index("-i") + 1], "rb").read()
lo = 2 * int(round(ss * rate))
hi = len(data) if t is None else lo + 2 * int(round(t * rate))
out = sys.stdout.buffer
for i in range(lo, min(hi, len(data)), 77777):   # a pipe delivers in pieces
    out.write(data[i: min(i + 77777, hi)])
'''


@pytest.mark.parametrize("vad,max_duration", [("energy_zcr", None), ("auditok", 150.0)])
def test_sync_media_with_a_stand_in_ffmpeg(handle, tmp_path, monkeypatch, vad, max_duration):
    from ffsubsync_b200.batch import BatchSynchronizer, sync_media
    exe = tmp_path / "ffmpeg"
    exe.write_text(_FAKE_FFMPEG)
    exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    videos = _videos(21, [3 * FR + 5, 0, 2 * CHUNK_100S + 7 * FR + 3, 61 * FR])
    paths = []
    for i, v in enumerate(videos):
        p = tmp_path / ("movie%d.mkv" % i)
        p.write_bytes(v.tobytes())
        paths.append(str(p))
    tv, cs, ce, co = _tracks(videos, 23)
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, vad=vad, start_seconds=2, max_offset_seconds=60.0)
    # what ffmpeg -ss 2 [-t 150] decodes of each
    cut = []
    for v in videos:
        lo = min(len(v), 2 * FR)
        hi = len(v) if max_duration is None else min(len(v), lo + int(max_duration * FR))
        cut.append(v[lo:hi])
    pcm = np.concatenate(cut)
    pcm_off = np.concatenate([[0], np.cumsum([len(v) for v in cut])]).astype(np.int64)
    want = bs.sync_host_tracks(pcm, pcm_off, tv, cs, ce, co, want_all=True, speech_video=[0, 2])
    got = sync_media(paths, bs, tv, cs, ce, co, max_decoders=2, ffmpeg_path=str(tmp_path),
                     max_duration_seconds=max_duration, want_all=True, speech_video=[0, 2])
    assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want))
    with pytest.raises(RuntimeError, match="status"):   # a decoder that fails aborts the session
        sync_media(paths + [str(tmp_path / "missing.mkv")], bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path))
    import subprocess
    popen = subprocess.Popen

    def failing_popen(cmd, *a, **k):   # a decoder that cannot even start (EMFILE, ENOMEM, ...)
        if any("movie2" in str(x) for x in cmd):
            raise OSError(24, "Too many open files")
        return popen(cmd, *a, **k)

    monkeypatch.setattr(subprocess, "Popen", failing_popen)
    with pytest.raises(RuntimeError, match="Too many open files"):
        sync_media(paths, bs, tv, cs, ce, co, max_decoders=1, ffmpeg_path=str(tmp_path))
    monkeypatch.setattr(subprocess, "Popen", popen)
    s = bs.ingest(1)   # the handle is free again
    s.abort()
