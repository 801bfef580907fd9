"""GPU suite of sampled segments streamed through the batched ingest session (b2_ingest_segments /
_push_segments / _drop_segment, ``IngestSession.push_segment``, ``batch.sync_media(multi_segment=...)``).

Libraries that mix audio videos and segment videos are pushed under several cut patterns (1-byte and odd pushes,
window- and auditok-call-straddling pushes, the reference's 100 s reads, several streams per push call), segments
out of start order and interleaved across videos.  Their segment shapes: overlapping segments (a 5-minute video with
8 x 60 s segments), a short last segment, a segment that starts past the probed end, a segment never pushed, one
dropped after partial pushes, a video whose segments are all dropped, a silent video and a single-segment video.
Every sync result (best_*, all_*, the search's outputs, the speech output) is compared bit for bit with
b2_sync_tracks_seg (B2_HOST) over the live pieces back to back, and every reference frame with the one-shot detector
over each segment's samples placed at its start (later starts win, clipped at int(total * 100) + 2)."""
import logging
import re
import stat
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_ingest import _FAKE_FFMPEG, _cuts, _same, _videos, GRID, MAX_OFF, SR, THR

pytestmark = pytest.mark.gpu

FR = 16000
FR48 = 48000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


class Seg:
    """A segment video: probed duration `total` (seconds), segment starts (whole seconds, increasing), each
    segment's PCM (None: never pushed) and the segments dropped after `partial` of their bytes were pushed."""

    def __init__(self, total, starts, pieces, dropped=()):
        self.total, self.starts, self.pieces, self.dropped = float(total), list(starts), pieces, set(dropped)


def _segment_video(seed, total, fr, duration=60, count=8, never=(), dropped=(), silent=False, starts=None,
                   extra=0):
    """Starts from _segment_starts (or `starts`), pieces of what ``ffmpeg -ss start -t duration`` decodes of a
    video of `total` seconds (plus `extra` samples past the probed end on the last one)."""
    from ffsubsync_b200.batch import ingest_segment_table
    if starts is None:
        starts = list(ingest_segment_table([total], [0], count, duration)["seg_start"])
    n_total = int(round(total * fr))
    pieces = []
    for j, s in enumerate(starts):
        if j in never:
            pieces.append(None)
            continue
        n = max(0, min(duration * fr, n_total - s * fr)) + (extra if j == len(starts) - 1 else 0)
        p = _videos(seed * 17 + j, [n], fr)[0]
        pieces.append(np.zeros(n, np.int16) if silent else p)
    return Seg(total, starts, pieces, dropped)


def _table(library):
    """The whole-call inputs over the live pieces back to back: (pcm, pcm_off, seg dict for sync_tracks_seg)."""
    parts, off = [], [0]
    sv, st, so, ss, lo, hi = [], [], [0], [], [], []
    for v, x in enumerate(library):
        if isinstance(x, Seg):
            at = 0
            for j, (s, p) in enumerate(zip(x.starts, x.pieces)):
                if j in x.dropped:
                    continue
                m = 0 if p is None else len(p)
                if m:
                    parts.append(p)
                ss.append(s)
                lo.append(at)
                hi.append(at + m)
                at += m
            sv.append(v)
            st.append(x.total)
            so.append(len(ss))
            off.append(off[-1] + at)
        else:
            parts.append(x)
            off.append(off[-1] + len(x))
    pcm = np.concatenate(parts) if parts else np.zeros(0, np.int16)
    seg = dict(seg_video=np.array(sv, np.int32), seg_total=np.array(st), seg_off=np.array(so, np.int64),
               seg_start=np.array(ss, np.int64), seg_lo=np.array(lo, np.int64), seg_hi=np.array(hi, np.int64))
    return pcm, np.array(off, np.int64), seg


def _declared(library):
    """The table b2_ingest_segments takes: every segment, dropped ones included."""
    sv, st, so, ss = [], [], [0], []
    for v, x in enumerate(library):
        if isinstance(x, Seg):
            sv.append(v)
            st.append(x.total)
            ss += x.starts
            so.append(len(ss))
    return np.array(sv, np.int32), np.array(st), np.array(so, np.int64), np.array(ss, np.int64)


def _schedule(library, kind, seed, chunk_bytes, fpw):
    """The pushes of a library: (video, segment or None, bytes) in a random interleaving that keeps each stream's
    order, plus ("drop", video, segment) after a dropped segment's first half.  Segments of a video are started in a
    shuffled order."""
    rng = np.random.RandomState(seed)
    streams = []
    for v, x in enumerate(library):
        if isinstance(x, Seg):
            order = list(range(len(x.starts)))
            rng.shuffle(order)
            for j in order:
                p = x.pieces[j]
                if p is None:
                    continue
                raw = p.tobytes()
                if j in x.dropped:
                    raw = raw[: len(raw) // 2 + 1]
                ops, at = [], 0
                for m in _cuts(kind, len(raw), rng, chunk_bytes, fpw):
                    ops.append((v, j, raw[at: at + m]))
                    at += m
                if j in x.dropped:
                    ops.append(("drop", v, j))
                streams.append(ops)
        else:
            raw, ops, at = x.tobytes(), [], 0
            for m in _cuts(kind, len(raw), rng, chunk_bytes, fpw):
                ops.append((v, None, raw[at: at + m]))
                at += m
            streams.append(ops)
    out = []
    while any(streams):
        live = [s for s in streams if s]
        out.append(live[rng.randint(len(live))].pop(0))
    return out


def _run_session(handle, library, kind, seed, fr, auditok, chunk, label, expect=None):
    """Opens a session, declares the segments and pushes the library; "many": several chunks per push call."""
    from ffsubsync_b200 import _native as N
    handle.ingest_begin(len(library), fr, SR, label, detector=N.B2_DETECTOR_AUDITOK if auditok else
                        N.B2_DETECTOR_ENERGY_ZCR, energy_threshold=THR, chunk_samples=chunk, expect_samples=expect)
    handle.ingest_segments(*_declared(library))
    fpw = fr // SR
    pattern = "bytes" if kind == "many" else kind
    ops = _schedule(library, pattern, seed, 2 * chunk or 2 * 100 * fr, fpw)
    rng = np.random.RandomState(seed + 1)
    i = 0
    while i < len(ops):
        op = ops[i]
        if op[0] == "drop":
            handle.ingest_drop_segment(op[1], op[2])
            i += 1
            continue
        k = int(rng.randint(1, 6)) if kind == "many" else 1
        group = []
        while i < len(ops) and len(group) < k and ops[i][0] != "drop" and \
                (ops[i][1] is None) == (op[1] is None):
            group.append(ops[i])
            i += 1
        if op[1] is None:
            handle.ingest_push([g[0] for g in group], [g[2] for g in group])
        else:
            handle.ingest_push([g[0] for g in group], [g[2] for g in group], segments=[g[1] for g in group])


def _tracks(library, fr, seed):
    """One track per video and a second one on the first, cue times inside each video's duration."""
    rng = np.random.RandomState(seed)
    dur = [x.total if isinstance(x, Seg) else max(len(x) / fr, 2.0) for x in library]
    tv = np.array([0] + list(range(len(library))), np.int32)
    starts, ends, off = [], [], [0]
    for v in tv:
        s = np.sort(rng.uniform(0, dur[v], 24))
        starts += list(s)
        ends += list(s + rng.uniform(0.3, 2.5, 24))
        off.append(len(starts))
    return tv, np.array(starts), np.array(ends), np.array(off, np.int64)


def _with_speech(handle, V, call):
    from ffsubsync_b200 import _native as N
    cap = 2 * 10 ** 6
    buf = np.full(cap, np.nan)
    off = np.full(V + 1, -1, np.int64)
    handle.speech_output(buf, cap, np.arange(V), off, N.B2_HOST)
    try:
        res = call()
    finally:
        handle.speech_output(None, 0, None, None)
    return tuple(res) + (buf[: off[-1]], off)


def _one_shot(handle, pcm, fr, auditok, chunk, label):
    off = np.array([0, len(pcm)], np.int64)
    if auditok:
        out, _ = handle.vad_auditok(pcm, off, fr, SR, label, chunk_samples=chunk)
        return out.astype(np.float32).astype(np.float64)
    out, _ = handle.vad_energy_zcr(pcm, off, fr, SR, label, THR)
    return out.astype(np.float64)


def _want_references(handle, library, fr, auditok, chunk, label):
    """Each video's reference: the one-shot detector over an audio video, and over each live segment's samples
    placed at start * 100 in start order (later starts win), clipped at int(total * 100) + 2, 0.0 elsewhere."""
    refs = []
    for x in library:
        if not isinstance(x, Seg):
            refs.append(_one_shot(handle, x, fr, auditok, chunk, label))
            continue
        L = int(x.total * SR) + 2
        r = np.zeros(L)
        for j, (s, p) in enumerate(zip(x.starts, x.pieces)):
            if j in x.dropped or p is None or not len(p):
                continue
            d = _one_shot(handle, p, fr, auditok, chunk, label)
            b = s * SR
            e = min(b + len(d), L)
            if e > b:
                r[b:e] = d[: e - b]
        refs.append(r)
    return refs


def _check(handle, library, fr, auditok, chunk, label, gss, kinds=("many", "straddle")):
    """Session results against b2_sync_tracks_seg over the live pieces, and its references frame for frame."""
    from ffsubsync_b200 import _native as N
    pcm, pcm_off, seg = _table(library)
    tv, cs, ce, co = _tracks(library, fr, 5)
    V = len(library)
    det = N.B2_DETECTOR_AUDITOK if auditok else N.B2_DETECTOR_ENERGY_ZCR
    want = _with_speech(handle, V, lambda: handle.sync_tracks_seg(
        pcm, pcm_off, tv, fr, SR, label, *(seg[k] for k in ("seg_video", "seg_total", "seg_off", "seg_start",
                                                             "seg_lo", "seg_hi")),
        cs, ce, None, co, GRID, 0.0, MAX_OFF, detector=det, energy_threshold=THR, chunk_samples=chunk, gss=gss,
        want_all=True, want_evals=gss))
    refs = _want_references(handle, library, fr, auditok, chunk, label)
    speech, off = want[-2], want[-1]
    for v in range(V):   # the whole call's references are the one-shot detector's, placed
        assert np.array_equal(speech[off[v]: off[v + 1]], refs[v]), v
    for i, kind in enumerate(kinds):
        _run_session(handle, library, kind, 30 + i, fr, auditok, chunk, label,
                     expect=[60 * fr if isinstance(x, Seg) else len(x) for x in library] if i % 2 else None)
        got = _with_speech(handle, V, lambda: handle.ingest_sync_tracks(tv, cs, ce, None, co, GRID, 0.0, MAX_OFF,
                                                                        gss=gss, want_evals=gss, want_all=True))
        assert len(got) == len(want)
        for j, (a, b) in enumerate(zip(got, want)):
            assert _same(a, b), (kind, j, a, b)
    return want


def _library(fr, duration=60):
    """An audio video; a 5-minute video with 8 x 60 s overlapping segments, one never pushed and one dropped after
    partial pushes; a video whose last decode runs past the probed end; an audio video; a video whose last segment
    decodes short."""
    return [_videos(1, [9 * fr + 77], fr)[0],
            _segment_video(2, 300.0, fr, duration, never={3}, dropped={5}),
            _segment_video(3, 3 * duration + 17.5, fr, duration, count=3, extra=fr * 3 + 11),
            _videos(4, [4 * fr + 5], fr)[0],
            _segment_video(19, 200.0, fr, duration, count=2, extra=-(41 * fr + 13))]


CASES = [  # (fr, auditok, chunk, label, gss)
    (FR, False, 0, 0.0, False), (FR, False, 0, 0.3, False), (FR, False, 0, 0.0, True),
    (FR, True, 100 * FR, 0.0, True), (FR, True, 1000, 0.3, False),
    (FR48, False, 0, 0.0, True), (FR48, False, 0, 0.3, False), (FR48, True, 100 * FR48, 0.0, False)]


@pytest.mark.parametrize("fr,auditok,chunk,label,gss", CASES)
def test_sync_equals_the_segment_call(handle, fr, auditok, chunk, label, gss):
    _check(handle, _library(fr), fr, auditok, chunk, label, gss)


@pytest.mark.parametrize("gss", [False, True])
def test_segments_longer_than_a_detector_call(handle, gss):
    """segment_duration 150 s with auditok's 100 s calls: pushes in 100 s reads and straddling ones cross a call
    inside a segment; the call loop restarts at each segment's first sample."""
    lib = [_segment_video(6, 700.0, FR, 150, count=3), _videos(7, [3 * FR], FR)[0]]
    _check(handle, lib, FR, True, 100 * FR, 0.0, gss, kinds=("100s", "straddle"))


def test_a_segment_that_starts_past_the_probed_end(handle):
    """Starts given by the caller (not _segment_starts): the last one lies past int(total * 100) + 2 and is clipped
    away entirely, the one before it partly."""
    lib = [_segment_video(8, 120.0, FR, 60, starts=[0, 100, 130])]
    lib[0].pieces[1] = _videos(9, [30 * FR + 7], FR)[0]
    lib[0].pieces[2] = _videos(9, [20 * FR], FR)[0]
    _check(handle, lib, FR, False, 0, 0.0, False, kinds=("straddle",))


def test_no_speech_videos_get_the_sentinel(handle):
    """A video whose segments are all dropped, a silent video and one whose segments were never pushed: best_k = -3 on
    their tracks, as from b2_sync_tracks_seg; a single-segment video (total <= segment_duration) syncs."""
    from ffsubsync_b200 import _native as N
    lib = [_segment_video(10, 200.0, FR, 60, count=3, dropped={0, 1, 2}),
           _segment_video(11, 200.0, FR, 60, count=3, silent=True),
           _segment_video(12, 200.0, FR, 60, count=3, never={0, 1, 2}),
           _segment_video(13, 45.0, FR, 60)]
    assert len(lib[3].starts) == 1
    want = _check(handle, lib, FR, False, 0, 0.0, False, kinds=("many",))
    tv = _tracks(lib, FR, 5)[0]
    assert list(want[2][tv <= 2]) == [N.B2_BEST_K_NO_SPEECH] * int(np.sum(tv <= 2)) and np.all(want[2][tv == 3] >= 0)


def test_search_at_a_non_zero_label_is_refused_as_by_the_segment_call(handle):
    from ffsubsync_b200 import _native as N
    lib = _library(FR)
    pcm, pcm_off, seg = _table(lib)
    tv, cs, ce, co = _tracks(lib, FR, 5)
    with pytest.raises(N.NativeError) as e0:
        handle.sync_tracks_seg(pcm, pcm_off, tv, FR, SR, 0.3, *(seg[k] for k in ("seg_video", "seg_total", "seg_off",
                                                                              "seg_start", "seg_lo", "seg_hi")),
                               cs, ce, None, co, GRID, 0.0, MAX_OFF, energy_threshold=THR, gss=True)
    _run_session(handle, lib, "100s", 3, FR, False, 0, 0.3)
    with pytest.raises(N.NativeError) as e1:
        handle.ingest_sync_tracks(tv, cs, ce, None, co, GRID, 0.0, MAX_OFF, gss=True)
    assert e0.value.status == e1.value.status == -6 and "label" in str(e1.value)


@pytest.mark.parametrize("auditok,chunk", [(False, 0), (True, 1000)])
def test_serialize_only_run(handle, auditok, chunk):
    """T == 0 with the speech output: the references alone, equal to the placed one-shot detector."""
    lib = _library(FR)
    refs = _want_references(handle, lib, FR, auditok, chunk, 0.0)
    _run_session(handle, lib, "straddle", 9, FR, auditok, chunk, 0.0)
    got = _with_speech(handle, len(lib), lambda: handle.ingest_sync_tracks(np.zeros(0, np.int32), np.zeros(0),
                                                                           np.zeros(0), None, [0], GRID, 0.0, MAX_OFF))
    speech, off = got[-2], got[-1]
    for v in range(len(lib)):
        assert np.array_equal(speech[off[v]: off[v + 1]], refs[v]), v


def test_the_synchronizer_session(handle):
    """IngestSession.push_segment / drop_segment / windows give sync_host_tracks over segment_table(piece_samples=...)
    (speech_video included), the device outputs sync_device_tracks', and the host path raises the reference's
    ValueError for a video without speech."""
    import torch
    from ffsubsync_b200 import _native as N
    from ffsubsync_b200.batch import BatchSynchronizer, ingest_segment_table, segment_table
    bs = BatchSynchronizer(list(GRID) + [None], frame_rate=FR, max_offset_seconds=60.0)
    audio = _videos(14, [6 * FR + 3], FR)[0]
    sv = _segment_video(15, 250.0, FR, 60, count=4)
    table = ingest_segment_table([250.0], [1], 4, 60)
    assert list(table["seg_start"]) == sv.starts
    pcm = np.concatenate([audio] + sv.pieces)
    pcm_off = np.array([0, len(audio), len(pcm)], np.int64)
    whole = segment_table(pcm_off, FR, [1], [250.0], 4, 60, piece_samples=[[len(p) for p in sv.pieces]])
    tv, cs, ce, co = _tracks([audio, sv], FR, 8)
    want = bs.sync_host_tracks(pcm, pcm_off, tv, cs, ce, co, want_all=True, speech_video=[0, 1], **whole)
    s = bs.ingest(2, segments=table)
    for j in (2, 0, 3, 1):
        s.push_segment(1, j, sv.pieces[j][:1001])
    s.push(0, audio)
    s.push_many([1, 1, 1, 1], [sv.pieces[j][1001:] for j in (3, 2, 1, 0)], segments=[3, 2, 1, 0])
    win = s.windows()
    assert win[0] == len(audio) // (FR // SR) and win[1] == sum(-(-len(p) // (FR // SR)) for p in sv.pieces)
    got = s.sync_tracks(tv, cs, ce, co, want_all=True, speech_video=[0, 1])
    assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want))
    T = len(tv)
    dev = torch.device("cuda", bs.handle.device)
    out = {k: torch.empty(T, dtype=d, device=dev) for k, d in (("best_score", torch.float64),
                                                               ("best_offset", torch.int32),
                                                               ("best_k", torch.int32), ("gss_ratio", torch.float64))}
    s = bs.ingest(2, expect_samples=[10, 10], segments=table)   # hints far too small: the regions grow
    s.push(0, audio)
    for j in range(4):
        s.push_segment(1, j, sv.pieces[j])
    s.sync_tracks(tv, cs, ce, co, out=out)
    torch.cuda.synchronize()
    for k, w in zip(("best_score", "best_offset", "best_k", "gss_ratio"), want[:3] + want[5:6]):
        assert _same(out[k].cpu().numpy(), w), k
    s = bs.ingest(2, segments=table)   # every segment dropped: the reference's error on the host
    s.push(0, audio)
    for j in range(4):
        s.push_segment(1, j, sv.pieces[j][:5000])
        s.drop_segment(1, j)
    with pytest.raises(ValueError, match="video 1: Unable to detect speech in any sampled segment"):
        s.sync_tracks(tv, cs, ce, co)
    bs.ingest(1).abort()   # the handle is free again
    assert N.B2_BEST_K_NO_SPEECH == -3


def test_refusals_leave_the_handle_usable(handle):
    from ffsubsync_b200 import _native as N
    lib = [_videos(16, [3 * FR + 5], FR)[0], _segment_video(17, 150.0, FR, 60, count=3)]
    refs = _want_references(handle, lib, FR, False, 0, 0.0)

    def works():
        handle.ingest_begin(2, FR, SR, 0.0, energy_threshold=THR)
        handle.ingest_segments(*_declared(lib))
        handle.ingest_push([0], [lib[0].tobytes()])
        for j, p in enumerate(lib[1].pieces):
            handle.ingest_push([1], [p.tobytes()], segments=[j])
        got = _with_speech(handle, 2, lambda: handle.ingest_sync_tracks(np.zeros(0, np.int32), np.zeros(0),
                                                                        np.zeros(0), None, [0], GRID, 0.0, MAX_OFF))
        assert np.array_equal(got[-2], np.concatenate(refs))

    def refused(call, needle):
        with pytest.raises(N.NativeError) as e:
            call()
        assert e.value.status == -1 and needle in str(e.value), str(e.value)

    decl = _declared(lib)
    refused(lambda: handle.ingest_segments(*decl), "no open session")
    refused(lambda: handle.ingest_drop_segment(1, 0), "no open session")
    refused(lambda: handle.ingest_push([1], [b"ab"], segments=[0]), "no open session")
    works()
    handle.ingest_begin(2, FR, SR, 0.0, energy_threshold=THR)
    handle.ingest_push([1], [b"ab"])
    refused(lambda: handle.ingest_segments(*decl), "video 1 already has pushes")
    handle.ingest_abort()
    handle.ingest_begin(2, FR, SR, 0.0, energy_threshold=THR)
    refused(lambda: handle.ingest_segments(decl[0], decl[1], decl[2], decl[3][::-1].copy()), "not after the previous")
    refused(lambda: handle.ingest_segments(decl[0], [float("inf")], decl[2], decl[3]), "seg_total[0] = inf")
    handle.ingest_segments(*decl)
    refused(lambda: handle.ingest_segments(*decl), "already declared")
    handle.ingest_push([1], [b"abcd"], segments=[2])
    handle.ingest_drop_segment(1, 2)
    refused(lambda: handle.ingest_push([0, 1], [b"ab", b"cd"]), "chunk 1: video 1 has sampled segments")
    refused(lambda: handle.ingest_push([1, 0], [b"ab", b"cd"], segments=[0, 0]), "chunk 1: video 0 has no sampled")
    refused(lambda: handle.ingest_push([1], [b"ab"], segments=[3]), "chunk 0: segment 3 of video 1 is out of [0, 3)")
    refused(lambda: handle.ingest_push([1, 1], [b"ab", b"cd"], segments=[0, 2]), "chunk 1: segment 2 of video 1 was "
                                                                                 "dropped")
    refused(lambda: handle.ingest_drop_segment(0, 0), "video 0 has no sampled segments")
    refused(lambda: handle.ingest_drop_segment(1, 5), "segment 5 of video 1 is out of")
    handle.ingest_abort()
    works()


_FAKE_FFPROBE = r'''#!/usr/bin/env python3
# stand-in for ffprobe in tests: the duration of a raw s16le mono file at %d Hz; fails for names with "noprobe"
import sys
f = sys.argv[-1]
if "noprobe" in f:
    sys.exit(1)
print(len(open(f, "rb").read()) / 2.0 / %d)
''' % (FR, FR)


def test_sync_media_multi_segment(handle, tmp_path, monkeypatch, caplog):
    from ffsubsync_b200.batch import BatchSynchronizer, segment_table, sync_media
    for name, text in (("ffmpeg", _FAKE_FFMPEG), ("ffprobe", _FAKE_FFPROBE)):
        exe = tmp_path / name
        exe.write_text(text)
        exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    videos = _videos(18, [310 * FR + 77, 9 * FR + 3, 140 * FR + 5], FR)
    paths = []
    for i, v in enumerate(videos):
        p = tmp_path / ("movie%d.mkv" % i)
        p.write_bytes(v.tobytes())
        paths.append(str(p))
    lib_tracks = [Seg(len(videos[0]) / FR, [], []), videos[1], Seg(len(videos[2]) / FR, [], [])]
    tv, cs, ce, co = _tracks(lib_tracks, FR, 19)
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, start_seconds=2, max_offset_seconds=60.0)

    def want_of(seg_videos, drop=None, count=8, duration=60):
        """sync_host_tracks over what the stand-in decodes: -ss 2 for audio videos, each segment for the others"""
        parts, totals, pieces = [], [], []
        for v, x in enumerate(videos):
            if v in seg_videos:
                t = len(x) / FR
                table = segment_table(np.array([0, len(x)]), FR, None, [t], count, duration)
                ps = []
                for j, s in enumerate(table["seg_start"]):
                    lo = min(len(x), int(round(s * FR)))
                    p = x[lo: min(len(x), lo + duration * FR)]
                    ps.append(p[:0] if drop == (v, j) else p)
                parts += ps
                totals.append(t)
                pieces.append([len(p) for p in ps])
            else:
                parts.append(x[min(len(x), 2 * FR):])
        pcm = np.concatenate(parts)
        off = np.concatenate([[0], np.cumsum([sum(pieces[seg_videos.index(v)]) if v in seg_videos else
                                              len(videos[v]) - min(len(videos[v]), 2 * FR)
                                              for v in range(len(videos))])]).astype(np.int64)
        table = segment_table(off, FR, seg_videos, totals, count, duration, piece_samples=pieces)
        if drop is not None:   # the dropped segment leaves the table
            i = seg_videos.index(drop[0])
            j = int(table["seg_off"][i]) + drop[1]
            keep = np.arange(len(table["seg_start"])) != j
            for k in ("seg_start", "seg_lo", "seg_hi"):
                table[k] = table[k][keep]
            table["seg_off"] = table["seg_off"] - (np.arange(len(table["seg_off"])) > i)
        return bs.sync_host_tracks(pcm, off, tv, cs, ce, co, want_all=True, speech_video=[0, 1, 2], **table)

    kw = dict(max_decoders=3, ffmpeg_path=str(tmp_path), want_all=True, speech_video=[0, 1, 2])
    want = want_of([0, 2])
    got = sync_media(paths, bs, tv, cs, ce, co, multi_segment=[0, 2], **kw)
    assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want))
    # every video sampled, with 3 segments of 100 s
    want = want_of([0, 1, 2], count=3, duration=100)
    got = sync_media(paths, bs, tv, cs, ce, co, multi_segment=True, segment_count=3, segment_duration=100, **kw)
    assert all(_same(a, b) for a, b in zip(got, want))
    # a segment decoder that exits non-zero after part of its output, and one that cannot start: dropped, logged
    popen = subprocess.Popen
    starts = list(segment_table(np.array([0, len(videos[0])]), FR, None, [len(videos[0]) / FR])["seg_start"])

    def failing_popen(cmd, *a, **k):
        from datetime import timedelta
        if not str(cmd[0]).endswith("ffmpeg"):   # ffprobe runs as it is
            return popen(cmd, *a, **k)
        if "movie0" in " ".join(map(str, cmd)) and str(timedelta(seconds=int(starts[2]))) in cmd:
            return popen([sys.executable, "-c", "import sys; sys.stdout.buffer.write(b'x' * 70001); sys.exit(3)"],
                         *a, **k)
        if "movie2" in " ".join(map(str, cmd)) and "-ss" not in cmd:   # its segment at 0 s
            raise OSError(24, "Too many open files")
        return popen(cmd, *a, **k)

    monkeypatch.setattr(subprocess, "Popen", failing_popen)
    with caplog.at_level(logging.WARNING):
        got = sync_media(paths, bs, tv, cs, ce, co, multi_segment=[0], **kw)
    monkeypatch.setattr(subprocess, "Popen", popen)
    want = want_of([0], drop=(0, 2))
    assert all(_same(a, b) for a, b in zip(got, want))
    assert "failed to extract segment at %ds: ffmpeg exited with status 3" % starts[2] in caplog.text
    monkeypatch.setattr(subprocess, "Popen", failing_popen)
    with caplog.at_level(logging.WARNING):
        got = sync_media(paths, bs, tv, cs, ce, co, multi_segment=[2], **kw)
    monkeypatch.setattr(subprocess, "Popen", popen)
    assert "failed to extract segment at 0s: OSError: [Errno 24] Too many open files" in caplog.text
    assert all(_same(a, b) for a, b in zip(got, want_of([2], drop=(2, 0))))
    # a failing probe raises the reference's error; -t with segments is refused
    bad = str(tmp_path / "noprobe.mkv")
    open(bad, "wb").write(videos[1].tobytes())
    with pytest.raises(ValueError, match=re.escape("multi-segment sync needs the reference duration, but probing '%s' "
                                                   "failed" % bad)):
        sync_media(paths[:2] + [bad], bs, tv, cs, ce, co, multi_segment=[2], ffmpeg_path=str(tmp_path))
    with pytest.raises(ValueError, match="max_duration_seconds"):
        sync_media(paths, bs, tv, cs, ce, co, multi_segment=True, max_duration_seconds=30.0)
    bs.ingest(1).abort()   # the handle is free again
