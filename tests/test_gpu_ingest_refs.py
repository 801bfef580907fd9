"""GPU suite of references that need no audio in the batched ingest session (b2_ingest_sync_refs,
``IngestSession.sync_tracks(**streams)``, ``batch.sync_media`` with stored signals, ``pgs_ref_stream`` and text streams).

Seeded libraries mix audio videos (pushed in 1-byte / window-straddling / 100 s cuts, interleaved), text-stream, PGS,
stored-signal and sampled-segment videos.  Every result (best_*, all_*, the search's outputs) and every speech-output
frame is compared bit for bit with b2_sync_tracks_seg (B2_HOST) over the same tables with the pushed PCM back to back,
for both detectors, labels 0 and 0.3, the grid and --gss, and outputs under B2_HOST and B2_DEVICE.  Further: the
signal and no-speech sentinels, the serialize-only run, every refusal followed by a working session on the same handle,
the call without tables against b2_ingest_sync_tracks on a replay of the same pushes, and sync_media with stand-in
ffmpeg / ffprobe scripts that record what they were asked to do."""
import json
import re
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
CAP = 4 * 10 ** 6


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _pcm(seed, n):
    rng = np.random.RandomState(seed)
    nw = -(-n // FPW)
    cls = np.repeat(rng.choice([0, 1, 2], size=-(-nw // 37) + 1, p=[0.45, 0.45, 0.1]), 37)[:nw].astype(np.uint8)
    return vo.synth_pcm(cls, FPW, seed=seed * 31 + 7)[:n]


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f")


class Lib:
    """A mixed library.  kinds[v]: "audio" (pcm[v]), "text", "pgs", "sig" or "seg" (pieces[v]: its segments' PCM,
    starts[v], total[v]); the reference tables of b2_sync_tracks_sig / _seg over all V videos."""

    def __init__(self, seed, kinds, bad_sig=None, silent_seg=False):
        rng = np.random.RandomState(seed)
        self.kinds = list(kinds)
        V = self.V = len(kinds)
        self.pcm, self.pieces, self.starts, self.total = {}, {}, {}, {}
        cues, pgs, sig = [[] for _ in range(V)], [[] for _ in range(V)], [np.zeros(0)] * V
        for v, k in enumerate(kinds):
            if k == "audio":
                self.pcm[v] = _pcm(seed * 13 + v, int(rng.choice([97, 7 * FR + 77, CHUNK_100S + 3 * FR + 5,
                                                                   2 * CHUNK_100S + 11])))
            elif k == "text":
                s = np.sort(rng.uniform(0, 120, 30))
                cues[v] = list(zip(s, s + rng.uniform(0.3, 3.0, 30)))
            elif k == "pgs":
                s = np.sort(rng.uniform(0, 120, 25))
                pgs[v] = list(zip(s, s + rng.uniform(0.5, 4.0, 25)))
            elif k == "sig":
                x = (rng.rand(int(rng.randint(6000, 14000))) > 0.5).astype(np.float64)
                x[x == 0] = rng.uniform(0, 0.99, int(np.sum(x == 0)))   # stored values < 1.0 become the label
                if bad_sig is not None:
                    x[len(x) // 3] = bad_sig
                    bad_sig = None
                sig[v] = x
            else:   # three segments of 60 s in a 400 s video
                self.total[v] = 400.0
                self.starts[v] = [0, 150, 300]
                self.pieces[v] = [np.zeros(60 * FR, np.int16) if silent_seg else _pcm(seed * 7 + v * 3 + j, 60 * FR)
                                  for j in range(3)]
        u8 = lambda k: np.array([x == k for x in kinds], np.uint8)   # noqa: E731
        cat = lambda lists: np.array([t for lst in lists for t in lst], np.float64).reshape(-1, 2)   # noqa: E731
        off = lambda lists: np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)   # noqa: E731
        c, p = cat(cues), cat(pgs)
        self.tables = dict(ref_is_subs=u8("text"), ref_cue_start_s=c[:, 0].copy(), ref_cue_end_s=c[:, 1].copy(),
                           ref_cue_keep=None, ref_cue_off=off(cues), ref_is_pgs=u8("pgs"), pgs_start_s=p[:, 0].copy(),
                           pgs_end_s=p[:, 1].copy(), pgs_off=off(pgs), ref_is_sig=u8("sig"), x=np.concatenate(sig),
                           sig_off=off(sig))
        # tracks: one per video, two on the first
        tv = np.array([0] + list(range(V)), np.int32)
        starts, ends, o = [], [], [0]
        for v in tv:
            s = np.sort(rng.uniform(0, 100, 14))
            starts += list(s)
            ends += list(s + rng.uniform(0.2, 2.5, 14))
            o.append(len(starts))
        self.tracks = (tv, np.array(starts), np.array(ends), np.array(o, np.int64))

    def whole(self):
        """(pcm, pcm_off, seg table) of b2_sync_tracks_seg: every audio video's and segment's PCM back to back."""
        parts, off = [], [0]
        sv, st, so, ss, lo, hi = [], [], [0], [], [], []
        for v, k in enumerate(self.kinds):
            n = 0
            if k == "audio":
                parts.append(self.pcm[v])
                n = len(self.pcm[v])
            elif k == "seg":
                for s, p in zip(self.starts[v], self.pieces[v]):
                    parts.append(p)
                    ss.append(s)
                    lo.append(n)
                    hi.append(n + len(p))
                    n += len(p)
                sv.append(v)
                st.append(self.total[v])
                so.append(len(ss))
            off.append(off[-1] + n)
        seg = (np.array(sv, np.int32), np.array(st), np.array(so, np.int64), np.array(ss, np.int64),
               np.array(lo, np.int64), np.array(hi, np.int64))
        return np.concatenate(parts + [np.zeros(0, np.int16)]), np.array(off, np.int64), seg

    def pushes(self, kind, seed):
        """(video, segment or None, bytes) of every audio video and segment under a cut pattern, interleaved."""
        rng = np.random.RandomState(seed)
        streams = [(v, None, self.pcm[v].tobytes()) for v in self.pcm]
        streams += [(v, j, p.tobytes()) for v in self.pieces for j, p in enumerate(self.pieces[v])]
        queues = []
        for v, j, raw in streams:
            sizes, left = [], len(raw)
            while left > 0:
                if kind == "bytes":
                    m = 1 if len(sizes) < 500 else int(rng.choice([3, 2 * FPW - 1, 2 * FPW * 700 + 3]))
                elif kind == "straddle":
                    m = int(rng.choice([2 * FPW * 3 + 7, 2 * CHUNK_100S - 3, 2 * CHUNK_100S + 2 * FPW + 1]))
                else:
                    m = 2 * CHUNK_100S
                sizes.append(min(m, left))
                left -= sizes[-1]
            queues.append(sizes)
        order = [i for i, q in enumerate(queues) for _ in q]
        rng.shuffle(order)
        at = [0] * len(streams)
        out = []
        for i in order:
            v, j, raw = streams[i]
            m = queues[i].pop(0)
            out.append((v, j, raw[at[i]: at[i] + m]))
            at[i] += m
        return out

    def declared(self):
        sv = [v for v in range(self.V) if self.kinds[v] == "seg"]
        ss = [s for v in sv for s in self.starts[v]]
        return (np.array(sv, np.int32), np.array([self.total[v] for v in sv]),
                np.concatenate([[0], np.cumsum([len(self.starts[v]) for v in sv])]).astype(np.int64),
                np.array(ss, np.int64))


def _det(auditok):
    from ffsubsync_b200 import _native as N
    return dict(detector=N.B2_DETECTOR_AUDITOK if auditok else N.B2_DETECTOR_ENERGY_ZCR, energy_threshold=THR,
                chunk_samples=CHUNK_100S if auditok else 0)


def _session(handle, lib, auditok, label, kind, seed, drop=()):
    """Opens a session, declares the segments, pushes under the cut pattern (drop: (video, segment) dropped after
    its pushes)."""
    handle.ingest_begin(lib.V, FR, SR, label, **_det(auditok))
    if "seg" in lib.kinds:
        handle.ingest_segments(*lib.declared())
    for v, j, c in lib.pushes(kind, seed):
        handle.ingest_push([v], [c], None if j is None else [j])
    for v, j in drop:
        handle.ingest_drop_segment(v, j)


def _with_speech(handle, V, call, memspace=None):
    from ffsubsync_b200 import _native as N
    buf = np.full(CAP, np.nan)
    off = np.full(V + 1, -1, np.int64)
    handle.speech_output(buf, CAP, np.arange(V), off, N.B2_HOST)
    try:
        res = call()
    finally:
        handle.speech_output(None, 0, None, None)
    return tuple(res) + (buf[: off[-1]], off)


def _whole(handle, lib, auditok, label, gss, tables=None, T=None):
    pcm, off, seg = lib.whole()
    tv, cs, ce, co = lib.tracks if T is None else (lib.tracks[0][:0], lib.tracks[1][:0], lib.tracks[2][:0], [0])
    t = dict(lib.tables if tables is None else tables)
    return handle.sync_tracks_seg(pcm, off, tv, FR, SR, label, *seg, cs, ce, None, co, GRID, 0.0, MAX_OFF, **t,
                                  **_det(auditok), gss=gss, want_all=True, want_evals=gss)


def _ingested(handle, lib, gss, tables=None, T=None):
    tv, cs, ce, co = lib.tracks if T is None else (lib.tracks[0][:0], lib.tracks[1][:0], lib.tracks[2][:0], [0])
    t = dict(lib.tables if tables is None else tables)
    return handle.ingest_sync_tracks(tv, cs, ce, None, co, GRID, 0.0, MAX_OFF, gss=gss, want_all=True,
                                     want_evals=gss, **t)


KINDS = ["audio", "text", "seg", "pgs", "audio", "sig", "audio", "text", "pgs", "sig", "audio"]
CASES = [  # (auditok, label, gss)
    (False, 0.0, False), (False, 0.3, False), (False, 0.0, True), (True, 0.0, False), (True, 0.0, True),
    (True, 0.3, False)]


@pytest.mark.parametrize("auditok,label,gss", CASES)
def test_mixed_library_equals_the_whole_call(handle, auditok, label, gss):
    lib = Lib(3, KINDS)
    want = _with_speech(handle, lib.V, lambda: _whole(handle, lib, auditok, label, gss))
    assert np.any(want[2] >= 0)
    for i, kind in enumerate(("bytes", "straddle", "100s")):
        _session(handle, lib, auditok, label, kind, 40 + i)
        got = _with_speech(handle, lib.V, lambda: _ingested(handle, lib, gss))
        assert len(got) == len(want)
        for j, (a, b) in enumerate(zip(got, want)):
            assert _same(a, b), (kind, j, a, b)


@pytest.mark.parametrize("auditok", [False, True])
def test_the_search_at_a_non_zero_label_is_refused_with_the_whole_calls_message(handle, auditok):
    from ffsubsync_b200 import _native as N
    lib = Lib(4, ["audio", "text", "audio"])
    with pytest.raises(N.NativeError) as want:
        _whole(handle, lib, auditok, 0.3, True)
    _session(handle, lib, auditok, 0.3, "100s", 1)
    with pytest.raises(N.NativeError) as got:
        _ingested(handle, lib, True)
    assert got.value.status == want.value.status == -6
    w, g = str(want.value), str(got.value)
    assert "ingest_sync_refs (search): " in g
    assert g.split("(search): ", 1)[1] == w.split("(search): ", 1)[1], (g, w)
    _session(handle, lib, auditok, 0.0, "100s", 1)   # the handle goes on
    assert all(_same(a, b) for a, b in zip(_ingested(handle, lib, False), _whole(handle, lib, auditok, 0.0, False)))


@pytest.mark.parametrize("auditok,gss", [(False, False), (True, True)])
def test_device_outputs_equal_the_whole_call(handle, auditok, gss):
    import torch
    from ffsubsync_b200 import _native as N
    lib = Lib(5, KINDS)
    want = _with_speech(handle, lib.V, lambda: _whole(handle, lib, auditok, 0.0, gss))
    tv, cs, ce, co = lib.tracks
    T, K = len(tv), len(GRID)
    cols = K + 1 if gss else K
    dev = torch.device("cuda", handle.device)
    out = dict(best_score=torch.empty(T, dtype=torch.float64, device=dev),
               best_offset=torch.empty(T, dtype=torch.int32, device=dev),
               best_k=torch.empty(T, dtype=torch.int32, device=dev),
               all_score=torch.empty(T * cols, dtype=torch.float64, device=dev),
               all_offset=torch.empty(T * cols, dtype=torch.int32, device=dev),
               gss_ratio=torch.empty(T, dtype=torch.float64, device=dev),
               gss_evals=torch.empty(T * N.GSS_EVALS, dtype=torch.float64, device=dev))
    x = torch.from_numpy(lib.tables["x"]).to(dev)
    speech = torch.full((CAP,), float("nan"), dtype=torch.float64, device=dev)
    soff = np.full(lib.V + 1, -1, np.int64)
    _session(handle, lib, auditok, 0.0, "straddle", 9)
    t = dict(lib.tables, x=x.data_ptr())
    handle.speech_output(speech.data_ptr(), CAP, np.arange(lib.V), soff, N.B2_DEVICE)
    try:
        ptrs = {k: v.data_ptr() for k, v in out.items() if gss or k not in ("gss_ratio", "gss_evals")}
        handle.ingest_sync_tracks(tv, cs, ce, None, co, GRID, 0.0, MAX_OFF, gss=gss, memspace=N.B2_DEVICE, **ptrs,
                                  **t)
    finally:
        handle.speech_output(None, 0, None, None)
    handle.synchronize()
    got = [out[k].cpu().numpy() for k in ("best_score", "best_offset", "best_k", "all_score", "all_offset")]
    if gss:
        got += [out["gss_ratio"].cpu().numpy(), out["gss_evals"].cpu().numpy()]
    got += [speech.cpu().numpy()[: soff[-1]], soff]
    assert len(got) == len(want)
    for j, (a, b) in enumerate(zip(got, want)):
        assert _same(a, b), (j, a, b)


def test_synchronizer_session_with_speech_video_equals_sync_host_tracks(handle):
    """IngestSession.sync_tracks(**streams) with the sync methods' keyword arguments, host and device."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    lib = Lib(6, ["audio", "sig", "pgs", "text", "audio", "seg"])
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, vad="subs_then_energy_zcr", max_offset_seconds=60.0)
    t = lib.tables
    V = lib.V
    sig_v = [v for v in range(V) if lib.kinds[v] == "sig"]
    pgs_v = [v for v in range(V) if lib.kinds[v] == "pgs"]
    txt_v = [v for v in range(V) if lib.kinds[v] == "text"]
    # the PGS video has a text stream too (PGS wins), the text video two (the longer wins), the segment video one
    # (dropped)
    assert pgs_v[0] < txt_v[0] < 5
    rs, re_ = t["ref_cue_start_s"], t["ref_cue_end_s"]
    streams = dict(ref_cue_start=np.concatenate([rs[:3], rs, rs[:2], rs[:2]]),
                   ref_cue_end=np.concatenate([re_[:3], re_, re_[:2], re_[:2]]),
                   ref_cue_off=np.array([0, 3, 3 + len(rs), 5 + len(rs), 7 + len(rs)]),
                   ref_stream_video=np.array([pgs_v[0], txt_v[0], txt_v[0], 5]),
                   pgs_start=t["pgs_start_s"], pgs_end=t["pgs_end_s"], pgs_off=[0, len(t["pgs_start_s"])],
                   pgs_video=pgs_v, sig=t["x"], sig_off=[0, len(t["x"])], sig_video=sig_v)
    pcm, off, seg = lib.whole()
    tv, cs, ce, co = lib.tracks
    segd = dict(zip(("seg_video", "seg_total", "seg_off", "seg_start", "seg_lo", "seg_hi"), seg))
    want = bs.sync_host_tracks(pcm, off, tv, cs, ce, co, want_all=True, speech_video=[0, 1, 2, 3, 5],
                               **segd, **streams)
    sess = bs.ingest(V, segments={k: segd[k] for k in ("seg_video", "seg_total", "seg_off", "seg_start")})
    for v, j, c in lib.pushes("100s", 3):
        (sess.push(v, c) if j is None else sess.push_segment(v, j, c))
    got = sess.sync_tracks(tv, cs, ce, co, want_all=True, speech_video=[0, 1, 2, 3, 5], **streams)
    assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want))
    # device: sig as a CUDA tensor
    dev = torch.device("cuda", bs.handle.device)
    T = len(tv)
    out = dict(best_score=torch.empty(T, dtype=torch.float64, device=dev),
               best_offset=torch.empty(T, dtype=torch.int32, device=dev),
               best_k=torch.empty(T, dtype=torch.int32, device=dev))
    sess = bs.ingest(V, segments={k: segd[k] for k in ("seg_video", "seg_total", "seg_off", "seg_start")})
    for v, j, c in lib.pushes("straddle", 4):
        (sess.push(v, c) if j is None else sess.push_segment(v, j, c))
    dstreams = dict(streams, sig=torch.from_numpy(t["x"]).to(dev))
    sess.sync_tracks(tv, cs, ce, co, out=out, speech_video=[1, 2], **dstreams)
    torch.cuda.synchronize(dev)
    for k, w in zip(("best_score", "best_offset", "best_k"), want[:3]):
        assert _same(out[k].cpu().numpy(), w), k
    w_speech, w_off = want[5], want[6]   # listed there: 0, 1, 2, 3, 5
    assert _same(out["speech"].cpu().numpy(), w_speech[w_off[1]: w_off[3]])
    assert _same(out["speech_off"], w_off[1:4] - w_off[1])
    # segment arguments belong to ingest(), and the session is closed by the refusal
    sess = bs.ingest(V)
    with pytest.raises(ValueError, match="declares its segments at ingest"):
        sess.sync_tracks(tv, cs, ce, co, **segd)
    bs.ingest(1).abort()


def test_sentinels_beside_reference_videos(handle):
    from ffsubsync_b200 import _native as N
    from ffsubsync_b200.batch import BatchSynchronizer
    for bad in (1.5, float("nan")):
        lib = Lib(8, ["audio", "sig", "text", "sig", "seg", "pgs"], bad_sig=bad, silent_seg=True)
        _session(handle, lib, False, 0.0, "100s", 2, drop=[(4, 0), (4, 1), (4, 2)])
        got = _with_speech(handle, lib.V, lambda: _ingested(handle, lib, False))
        tv = lib.tracks[0]
        bk = got[2]
        assert set(np.flatnonzero(bk == N.B2_BEST_K_BAD_SIGNAL)) == set(np.flatnonzero(tv == 1))
        assert set(np.flatnonzero(bk == N.B2_BEST_K_NO_SPEECH)) == set(np.flatnonzero(tv == 4))
        # the whole call over the live pieces: the segment video's pieces are all dropped there too
        lib.pieces[4] = [p[:0] for p in lib.pieces[4]]
        want = _with_speech(handle, lib.V, lambda: _whole(handle, lib, False, 0.0, False))
        _session(handle, lib, False, 0.0, "100s", 2)
        got = _with_speech(handle, lib.V, lambda: _ingested(handle, lib, False))
        assert all(_same(a, b) for a, b in zip(got, want))
    # the host method raises the bad signal's ValueError
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, max_offset_seconds=60.0)
    lib = Lib(9, ["audio", "sig"], bad_sig=2.0)
    sess = bs.ingest(2)
    sess.push(0, lib.pcm[0])
    tv, cs, ce, co = lib.tracks
    with pytest.raises(ValueError, match=r"video 1: its serialized signal holds 2\.0 at frame \d+"):
        sess.sync_tracks(tv, cs, ce, co, sig=lib.tables["x"], sig_off=[0, len(lib.tables["x"])], sig_video=[1])


@pytest.mark.parametrize("auditok", [False, True])
def test_serialize_only_writes_the_reference_videos(handle, auditok):
    lib = Lib(10, KINDS)
    want = _with_speech(handle, lib.V, lambda: _whole(handle, lib, auditok, 0.0, False, T=0))
    _session(handle, lib, auditok, 0.0, "bytes", 5)
    got = _with_speech(handle, lib.V, lambda: _ingested(handle, lib, False, T=0))
    assert _same(got[-2], want[-2]) and _same(got[-1], want[-1])
    for v, k in enumerate(lib.kinds):   # the reference videos' frames are there, not left NaN
        if k in ("text", "pgs", "sig"):
            assert not np.any(np.isnan(got[-2][got[-1][v]: got[-1][v + 1]]))


def test_refusals_leave_the_handle_usable(handle):
    import torch
    from ffsubsync_b200 import _native as N
    lib = Lib(12, ["audio", "text", "sig", "pgs", "seg"])

    def works():
        _session(handle, lib, False, 0.0, "100s", 1)
        assert all(_same(a, b) for a, b in zip(_ingested(handle, lib, False), _whole(handle, lib, False, 0.0, False)))

    def refused(prepare, tables, needle, status=-1, **kw):
        _session(handle, lib, False, 0.0, "100s", 1)
        prepare()
        with pytest.raises(N.NativeError) as e:
            _ingested(handle, lib, False, tables=tables, **kw)
        assert e.value.status == status and needle in str(e.value), str(e.value)
        with pytest.raises(N.NativeError, match="no open session"):   # the session closed
            handle.ingest_push([0], [b"ab"])
        works()

    works()
    refused(lambda: handle.ingest_push([2], [b"abc"]), None,
            "ingest_sync_refs: video 2 has a serialized signal reference and received 3 pushed bytes")
    refused(lambda: handle.ingest_push([1], [b"abcd"]), None, "video 1 has a text subtitle reference and received 4")
    seg_pgs = dict(lib.tables, ref_is_pgs=np.array([0, 0, 0, 0, 1], np.uint8),
                   pgs_off=np.array([0, 0, 0, 0, 0, len(lib.tables["pgs_start_s"])]))
    refused(lambda: None, seg_pgs, "video 4 has sampled segments and a PGS reference")
    both = dict(lib.tables, ref_is_subs=np.array([0, 1, 1, 0, 0], np.uint8))
    refused(lambda: None, both, "video 2 is marked both as a signal and as a text subtitle reference")
    _session(handle, lib, False, 0.0, "100s", 1)
    tv, cs, ce, co = lib.tracks
    T = len(tv)
    dev = torch.device("cuda", handle.device)
    o = [torch.empty(T, dtype=dt, device=dev) for dt in (torch.float64, torch.int32, torch.int32)]
    with pytest.raises(N.NativeError) as e:
        handle.ingest_sync_tracks(tv, cs, ce, None, co, GRID, 0.0, MAX_OFF, memspace=N.B2_DEVICE,
                                  best_score=o[0].data_ptr(), best_offset=o[1].data_ptr(), best_k=o[2].data_ptr(),
                                  **lib.tables)
    assert e.value.status == -1 and "ingest_sync_refs: x" in str(e.value), str(e.value)
    works()


def test_no_tables_equals_ingest_sync_tracks_and_the_whole_call(handle):
    """b2_ingest_sync_tracks forwards to b2_ingest_sync_refs, so equality between the two on a replay of the same
    pushes is no evidence on its own; both are also held to the whole calls over the pushed PCM back to back, the
    calls the session's results were pinned to before it took references (b2_sync_tracks / _gss / _auditok for audio
    alone, b2_sync_tracks_seg without tables with segment videos)."""
    from ffsubsync_b200 import _native as N
    for kinds in (["audio", "audio", "audio"], ["audio", "audio", "seg", "audio"]):
        lib = Lib(14, kinds)
        tv, cs, ce, co = lib.tracks
        T, K = len(tv), len(GRID)
        pcm, off, _ = lib.whole()
        for auditok, gss in ((False, False), (False, True), (True, True)):
            if "seg" in kinds:
                whole = lambda: _whole(handle, lib, auditok, 0.0, gss, tables={})   # noqa: E731
            elif auditok:
                whole = lambda: handle.sync_tracks_auditok(pcm, off, tv, FR, SR, 0.0, cs, ce, None, co, GRID,   # noqa: E731
                                                           0.0, MAX_OFF, CHUNK_100S, gss=gss, want_all=True,
                                                           want_evals=gss)
            elif gss:
                whole = lambda: handle.sync_tracks_gss(pcm, off, tv, FR, SR, 0.0, THR, -1, -1, cs, ce, None, co,   # noqa: E731
                                                       GRID, 0.0, MAX_OFF, want_all=True, want_evals=True)
            else:
                whole = lambda: handle.sync_tracks(pcm, off, tv, FR, SR, 0.0, THR, -1, -1, cs, ce, None, co, GRID,   # noqa: E731
                                                   0.0, MAX_OFF, want_all=True)
            want = _with_speech(handle, lib.V, whole)
            _session(handle, lib, auditok, 0.0, "straddle", 6)
            tracks = _with_speech(handle, lib.V, lambda: handle.ingest_sync_tracks(
                tv, cs, ce, None, co, GRID, 0.0, MAX_OFF, gss=gss, want_all=True, want_evals=gss))
            _session(handle, lib, auditok, 0.0, "straddle", 6)
            cols = K + 1 if gss else K
            bs_, bo, bk = np.empty(T), np.empty(T, np.int32), np.empty(T, np.int32)
            a_s, a_o = np.empty(T * cols), np.empty(T * cols, np.int32)
            gr, ge = (np.empty(T), np.empty(T * N.GSS_EVALS)) if gss else (None, None)
            p = lambda a: None if a is None else a.ctypes.data   # noqa: E731
            tv32, cs64, ce64, co64 = (np.ascontiguousarray(tv, np.int32), np.ascontiguousarray(cs),
                                      np.ascontiguousarray(ce), np.ascontiguousarray(co, np.int64))

            def call():
                st = handle.lib.b2_ingest_sync_refs(handle.h, *([None] * 12), p(tv32), T, p(cs64), p(ce64), None,
                                                    p(co64), p(GRID), K, 0.0, MAX_OFF, p(bs_), p(bo), p(bk), p(a_s),
                                                    p(a_o), p(gr), p(ge), N.B2_HOST)
                assert st == 0, handle.lib.b2_last_error(handle.h)
                return (bs_, bo, bk, a_s, a_o) + ((gr, ge) if gss else ())

            refs = _with_speech(handle, lib.V, call)
            assert np.any(want[2] >= 0)
            for j, (a, b, c) in enumerate(zip(refs, tracks, want)):
                assert _same(a, c) and _same(b, c), (kinds, auditok, gss, j)


# ---------------------------------------------------------------------------------------------- sync_media
_FAKE_FFMPEG = r'''#!/usr/bin/env python3
# stand-in for ffmpeg in tests: "decodes" the input file as raw s16le mono, honouring -ss / -t at the -ar rate, and
# appends its input's name to the log next to it
import os, sys
a = sys.argv[1:]
open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "calls.log"), "a").write("ffmpeg %s\n" % a[a.index("-i") + 1])
def hms(v):
    h, m, s = v.split(":")
    return int(h) * 3600 + int(m) * 60 + float(s)
rate = int(a[a.index("-ar") + 1])
ss = hms(a[a.index("-ss") + 1]) if "-ss" in a else 0.0
t = hms(a[a.index("-t") + 1]) if "-t" in a else None
data = open(a[a.index("-i") + 1], "rb").read()
lo = 2 * int(round(ss * rate))
hi = len(data) if t is None else lo + 2 * int(round(t * rate))
for i in range(lo, min(hi, len(data)), 77777):
    sys.stdout.buffer.write(data[i: min(i + 77777, hi)])
'''

# stand-in for ffprobe: a file "<name>.probe.json" beside the input holds {"streams": [...], "packets": [...]};
# "-show_packets" answers the packets (exit 1 when the file has none), otherwise the streams; every call is logged
_FAKE_FFPROBE = r'''#!/usr/bin/env python3
import json, os, sys
a = sys.argv[1:]
f = a[-1]
open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "calls.log"), "a").write("ffprobe %s %s\n" % (f, " ".join(a[:-1])))
meta = json.load(open(f + ".probe.json")) if os.path.exists(f + ".probe.json") else {"streams": []}
if "-show_packets" in a:
    if "packets" not in meta:
        sys.exit(1)
    print(json.dumps({"packets": meta["packets"]}))
else:
    print(json.dumps({"streams": meta["streams"]}))
'''


def _pgs_probe(intervals):
    packets = []
    for s, e in intervals:
        packets.append({"pts_time": "%.6f" % s, "duration_time": "%.6f" % (e - s), "size": "4000"})
        packets.append({"pts_time": "%.6f" % e, "duration_time": "N/A", "size": "30"})
    return {"streams": [{"index": 0, "codec_type": "video"}, {"index": 1, "codec_type": "subtitle",
                                                               "codec_name": "subrip"},
                        {"index": 2, "codec_type": "subtitle", "codec_name": "hdmv_pgs_subtitle"}],
            "packets": packets}


def test_sync_media_takes_signal_pgs_and_text_references_without_decoding_them(handle, tmp_path, monkeypatch):
    from ffsubsync_b200.batch import BatchSynchronizer, sync_media
    from ffsubsync_b200.speech_transformers import PGSSpeechTransformer
    for name, text in (("ffmpeg", _FAKE_FFMPEG), ("ffprobe", _FAKE_FFPROBE)):
        exe = tmp_path / name
        exe.write_text(text)
        exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    log = tmp_path / "calls.log"
    lib = Lib(16, ["audio", "pgs", "sig", "text", "audio"])
    t = lib.tables
    paths = []
    for v, k in enumerate(lib.kinds):
        if k == "sig":
            p = tmp_path / ("ref%d.npz" % v)
            np.savez_compressed(p, speech=t["x"])
        else:
            p = tmp_path / ("movie%d.mkv" % v)
            p.write_bytes(lib.pcm[v].tobytes() if k == "audio" else b"\0\0" * 1000)
        paths.append(str(p))
    iv = list(zip(t["pgs_start_s"], t["pgs_end_s"]))
    (tmp_path / "movie1.mkv.probe.json").write_text(json.dumps(_pgs_probe(iv)))
    tv, cs, ce, co = lib.tracks
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, vad="subs_then_energy_zcr", max_offset_seconds=60.0)
    text = dict(ref_cue_start=t["ref_cue_start_s"], ref_cue_end=t["ref_cue_end_s"],
                ref_cue_off=[0, len(t["ref_cue_start_s"])], ref_stream_video=[3])
    # what the stand-in decodes (start_seconds 0): the audio videos' bytes; the probe's intervals at its precision
    pcm = np.concatenate([lib.pcm[0], lib.pcm[4]])
    off = np.array([0, len(lib.pcm[0]), len(lib.pcm[0]), len(lib.pcm[0]), len(lib.pcm[0]), len(pcm)], np.int64)
    piv = np.array(PGSSpeechTransformer(SR, ffmpeg_path=str(tmp_path), ref_stream="s:1")._probe_intervals(paths[1]))
    want = bs.sync_host_tracks(pcm, off, tv, cs, ce, co, want_all=True, speech_video=[1, 2, 3],
                               pgs_start=piv[:, 0], pgs_end=piv[:, 1], pgs_off=[0, len(piv)], pgs_video=[1],
                               sig=t["x"], sig_off=[0, len(t["x"])], sig_video=[2], **text)
    for spec in (["s:1" if v == 1 else None for v in range(5)], "auto"):
        log.write_text("")
        got = sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), max_decoders=3, want_all=True,
                         speech_video=[1, 2, 3], pgs_ref_stream=spec if spec != "auto" else
                         [None, "auto", None, None, None], **text)
        assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want)), spec
        decoded = sorted(line.split()[1] for line in log.read_text().splitlines() if line.startswith("ffmpeg"))
        assert decoded == sorted([paths[0], paths[4]])   # no decode of the PGS, signal or text videos
    # a subtitle file is refused before anything starts
    log.write_text("")
    with pytest.raises(ValueError, match="subtitle file"):
        sync_media(paths[:4] + [str(tmp_path / "ref.srt")], bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path))
    assert log.read_text() == ""
    bs.ingest(1).abort()
    # keywords other than the text streams are refused before anything starts (PGS and signals have their own forms)
    for bad_kw in (dict(sig=t["x"], sig_off=[0, len(t["x"])], sig_video=[2]),
                   dict(pgs_start=piv[:, 0], pgs_end=piv[:, 1], pgs_off=[0, len(piv)], pgs_video=[1])):
        log.write_text("")
        with pytest.raises(TypeError, match="takes embedded text streams"):
            sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), **text, **bad_kw)
        assert log.read_text() == ""
    # a probed list that PGSSpeechTransformer.fit's raster refuses (a non-finite time): fit's ValueError
    bad_iv = [(1.0, 2.0), (float("inf"), 3.0)]
    (tmp_path / "movie1.mkv.probe.json").write_text(json.dumps(_pgs_probe(bad_iv)))
    bad_probed = PGSSpeechTransformer(SR, ffmpeg_path=str(tmp_path), ref_stream="s:1")._probe_intervals(paths[1])
    with pytest.raises(ValueError) as fit_err:
        PGSSpeechTransformer(SR).fit(bad_probed)
    with pytest.raises(ValueError, match="^%s$" % re.escape(str(fit_err.value))):
        sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), pgs_ref_stream=[None, "s:1", None, None,
                                                                                           None], **text)
    # the reference's three PGS errors
    (tmp_path / "movie1.mkv.probe.json").write_text(json.dumps({"streams": []}))
    spec = [None, "auto", None, None, None]
    with pytest.raises(ValueError, match=re.escape("No hdmv_pgs_subtitle stream found in %s. " % paths[1])):
        sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), pgs_ref_stream=spec, **text)
    with pytest.raises(ValueError, match=re.escape("Failed to get PGS timings via ffprobe for stream 0:s:1 from %s."
                                                   % paths[1])):
        sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), pgs_ref_stream=[None, "s:1", None, None,
                                                                                           None], **text)
    monkeypatch.setattr(PGSSpeechTransformer, "_probe_intervals", lambda self, fname: [])
    with pytest.raises(ValueError, match=re.escape("No subtitle timings found in PGS stream 0:s:1.")):
        sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), pgs_ref_stream=[None, "0:s:1", None, None,
                                                                                           None], **text)
    bs.ingest(1).abort()   # the handle is free again


def test_sync_media_broadcasts_one_pgs_ref_stream_to_every_non_signal_video(handle, tmp_path):
    """pgs_ref_stream as one string ("auto" or "s:N") applies to every video that is not a stored signal: a library of
    PGS videos and a ref.npz runs no decoder at all."""
    from ffsubsync_b200.batch import BatchSynchronizer, sync_media
    from ffsubsync_b200.speech_transformers import PGSSpeechTransformer
    for name, text in (("ffmpeg", _FAKE_FFMPEG), ("ffprobe", _FAKE_FFPROBE)):
        exe = tmp_path / name
        exe.write_text(text)
        exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    log = tmp_path / "calls.log"
    lib = Lib(17, ["pgs", "sig", "pgs"])
    t = lib.tables
    paths = [str(tmp_path / "movie0.mkv"), str(tmp_path / "ref1.npy"), str(tmp_path / "movie2.mkv")]
    np.save(paths[1], t["x"])
    po = t["pgs_off"]
    for v in (0, 2):
        open(paths[v], "wb").write(b"\0\0" * 1000)
        iv = list(zip(t["pgs_start_s"][po[v]: po[v + 1]], t["pgs_end_s"][po[v]: po[v + 1]]))
        open(paths[v] + ".probe.json", "w").write(json.dumps(_pgs_probe(iv)))
    tv, cs, ce, co = lib.tracks
    bs = BatchSynchronizer(list(GRID), frame_rate=FR, max_offset_seconds=60.0)
    probed = [np.array(PGSSpeechTransformer(SR, ffmpeg_path=str(tmp_path))._probe_intervals(paths[v])) for v in (0, 2)]
    want = bs.sync_host_tracks(np.zeros(0, np.int16), np.zeros(4, np.int64), tv, cs, ce, co, want_all=True,
                               speech_video=[0, 1, 2], pgs_start=np.concatenate([p[:, 0] for p in probed]),
                               pgs_end=np.concatenate([p[:, 1] for p in probed]),
                               pgs_off=[0, len(probed[0]), len(probed[0]) + len(probed[1])], pgs_video=[0, 2],
                               sig=t["x"], sig_off=[0, len(t["x"])], sig_video=[1])
    for spec in ("auto", "s:1", "0:s:1"):
        log.write_text("")
        got = sync_media(paths, bs, tv, cs, ce, co, ffmpeg_path=str(tmp_path), want_all=True, speech_video=[0, 1, 2],
                         pgs_ref_stream=spec)
        assert len(got) == len(want) and all(_same(a, b) for a, b in zip(got, want)), spec
        calls = log.read_text().splitlines()
        assert not any(c.startswith("ffmpeg") for c in calls), calls   # nothing decoded
        probes = sorted({c.split()[1] for c in calls if "-show_packets" in c})
        assert probes == sorted([paths[0], paths[2]]), calls   # the signal video is not probed
