"""The batched calls past 32-bit sample and byte indices (run on an H100).

A. Far placement.  One device int16 buffer of 2^32 + 2^26 samples (8.7 GB) holds a few videos of one to five minutes
   at sample offsets just below and above 2^31 (byte 2^32) and 2^32 (byte 2^33), and at the buffer's end; the first
   placement of each mark puts it inside a window of the first video.  Every output of every call there equals, bit
   for bit, the same call on the videos at offset 0 of a buffer of their own, and that call equals the composed
   exact oracle of tests/test_gpu_random_requests.py: b2_vad_energy_zcr and b2_vad_auditok (whose pcm_off[0] must be
   16-byte aligned: an unaligned placement gets a silent filler video in front), b2_sync_batch (B2_DEVICE and
   B2_DEVICE_RESIDENT), b2_sync_tracks on the tiled, run and big aligner paths with packed and float references, one
   and three sub-batches and the lane-group VAD layout, b2_sync_tracks_gss, b2_sync_tracks_auditok and
   b2_sync_tracks_seg (segments of a far video), each with the reference captured (b2_capture_reference) and the
   speech output written (b2_speech_output).

B. One long video.  A 48 kHz video of 2^31 + 4321 samples and a 44.1 kHz one of 2^31 + 88201, made by b2_synth_pcm from
   window classes: silence and voiced speech (whose energy / ZCR and auditok decisions follow from the class for
   every window, see _decided) everywhere, and random classes with loud hiss in bands of windows around sample 2^31
   and around each 100 s read near it, where the decisions are computed exactly from the samples copied back, as
   they are at a seeded sample of windows elsewhere.  Checked: b2_vad_energy_zcr and b2_vad_auditok (100 s reads)
   against that oracle; b2_sync_tracks_sig on the tiled and run paths (energy / ZCR and auditok, every reference kind,
   the long video's cues spread over all 12 h, five ratios, +-60 s) and b2_sync_tracks_gss, reference frame for frame
   and every (track, ratio) score and offset against the exact correlation; the ingest session fed the same video in
   100 s reads against the whole call; b2_sync_tracks_seg with segments from past sample 2^31 against
   segment_oracle.

Each family checks free device memory first and skips when the GPU cannot hold it (the machines are shared).  The
module prints the peak device memory in use at the checkpoints and its wall time."""
import contextlib
import time

import numpy as np
import pytest

import nomination_check as nc
import random_requests as rr
from oracle import auditok_oracle as ad
from oracle import chunk_oracle as co
from oracle import raster_oracle as ro
from oracle import segment_oracle as so
from oracle import vad_oracle as vo
from test_gpu_random_requests import THR, _call, _check_outputs, _gss_trace, _reference, _same, _sub
from test_gpu_reference_exact import _check as check_capture
from test_gpu_reference_exact import _poison
from test_gpu_speech_out import _output as speech_out

pytestmark = pytest.mark.gpu

M31, M32 = 1 << 31, 1 << 32
BUF = M32 + (1 << 26)            # family A's buffer, samples
GB = 1 << 30
STATS = {"peak": 0, "t0": None}


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    STATS["t0"] = time.time()
    yield _native.get_handle()
    print("\ntest_gpu_wide_index: peak device memory in use %.2f GB, wall time %.0f s"
          % (STATS["peak"] / GB, time.time() - STATS["t0"]))


def _need(nbytes):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (nbytes / GB, free / GB))


def _note():
    import torch
    torch.cuda.synchronize()
    free, total = torch.cuda.mem_get_info()
    STATS["peak"] = max(STATS["peak"], total - free)


def _free():
    import gc
    import torch
    gc.collect()
    torch.cuda.empty_cache()


class RunExact(nc.Exact):
    """nc.Exact whose window is summed from the runs of the subtitle signal over prefix sums of the reference: every
    term a multiple of 2^-24 below 2^29, so the sums are exact in float64 whatever the transform length (a 12 h
    reference pads to 2^24 points)."""

    def window(self, ref, sub, w0, n):
        r = 2.0 * np.asarray(ref, np.float64) - 1.0
        s = 2.0 * np.asarray(sub, np.float64) - 1.0
        P = np.concatenate([[0.0], np.cumsum(r)])
        R, S = len(r), len(s)
        cut = np.flatnonzero(np.diff(s)) + 1
        a_run, b_run = np.concatenate([[0], cut]), np.concatenate([cut, [S]])
        o = w0 + np.arange(n, dtype=np.int64)
        lo, hi = np.maximum(0, -o), np.minimum(S, R - o)
        out = np.zeros(n)
        for a, b in zip(a_run, b_run):
            a2, b2 = np.maximum(a, lo), np.minimum(b, hi)
            ok = b2 > a2
            out += s[a] * np.where(ok, P[np.clip(b2 + o, 0, R)] - P[np.clip(a2 + o, 0, R)], 0.0)
        return out


# ============================================================================================ A. far placement

def _video_lengths(fr):
    fpw = fr // 100
    return [62 * fr + 37, rr.chunk_samples(fr) + fpw + 1, 3 * 60 * fr - 1, 5 * 60 * fr + fpw // 2]


def _far_req(entry, fr, knobs, detector="energy_zcr", seed=11):
    """A request in tests/random_requests.py's form: four audio videos of one to five minutes (seg: the second is a
    segment video, a subtitle, PGS and signal video follow), two tracks each, three ratios, +-60 s."""
    rng = np.random.RandomState(seed)
    videos = [dict(kind="audio", n=n) for n in _video_lengths(fr)]
    if entry == "seg":
        n = videos[1]["n"]
        total = n / fr
        starts = [3, 40, 95]
        lo = [s * fr for s in starts]
        videos[1] = dict(kind="seg", n=n, total=total, starts=starts, lo=lo, hi=[min(n, a + 30 * fr) for a in lo])
        st, en = ro.synthetic_cues(seed + 1, 150.0)
        videos.append(dict(kind="subs", starts=st, ends=en, keep=(rng.rand(len(st)) < 0.8).astype(np.uint8)))
        st, en = ro.synthetic_cues(seed + 2, 120.0)
        videos.append(dict(kind="pgs", starts=st + 0.004, ends=en + 0.006))
        videos.append(dict(kind="sig", x=rng.choice([0.0, 0.25, 1.0], 9000).astype(np.float64)))
    for d in videos:
        d["dur"] = d["n"] / fr if "n" in d else 120.0
    tracks = []
    for v, d in enumerate(videos):
        for i in range(1 if entry == "batch" else 2):
            st, en = ro.synthetic_cues(seed * 100 + 7 * v + i, d["dur"] + 5)
            sh = [-2.5, 1.75][i]
            ok = st + sh >= 0
            tracks.append(dict(video=v, starts=np.round(st[ok] + sh, 3), ends=np.round(en[ok] + sh, 3)))
    gss = entry == "gss"
    return dict(seed=seed, entry=entry, fr=fr, videos=videos, tracks=tracks,
                ratios=[1.0, 25 / 23.976, 23.976 / 25], mos=6000, label=0.0 if gss else -0.5, memspace="device",
                knobs=knobs, detector="auditok" if entry == "auditok" else detector, chunk=rr.chunk_samples(fr),
                keep_tracks=False, keep_seed=seed + 17)


def _pcms(req):
    fpw = req["fr"] // 100
    out = []
    for v, d in enumerate(req["videos"]):
        if d["kind"] not in ("audio", "seg"):
            out.append(np.zeros(0, np.int16))
            continue
        rng = np.random.RandomState(req["seed"] * 31 + v)
        W = -(-d["n"] // fpw)
        cls = np.repeat(rng.choice(3, -(-W // 50), p=[0.45, 0.45, 0.1]), 50)[:W].astype(np.uint8)
        out.append(vo.synth_pcm(cls, fpw, req["seed"] + v)[:d["n"]])
    return out


def _placements(total):
    """First samples of the batch in the far buffer: a window of the first video straddles the mark (the start
    16-byte aligned, so the lane kernel stays eligible), then an unaligned start just past it, for elements 2^31 and
    2^32; and the batch ending at the buffer's last sample."""
    return [M31 - 8008, M31 + 3, M32 - 8008, M32 + 5, BUF - total]


def _run_sync(handle, req, a, pcm, speech, cap_n, gss):
    """One call with the reference captured, the speech output of `speech` and (not the search) the nominations."""
    from ffsubsync_b200 import _native as N
    T, K = len(req["tracks"]), len(req["ratios"])
    V = len(req["videos"])
    _poison(handle, cap_n)
    with contextlib.ExitStack() as stack:
        cap = stack.enter_context(handle.capture_reference(cap_n, V + 3))
        nom = None if gss else stack.enter_context(handle.capture_nominations(T * K, 12001))
        sp = stack.enter_context(speech_out(handle, speech, cap_n, N.B2_DEVICE))
        got = _call(handle, req, a, pcm, "device", want_all=True)
    _note()
    return got, cap, sp, nom


FAR_CASES = [
    ("batch", 16000, dict(B2_SUBBATCHES="3")),
    ("tracks", 16000, dict(B2_SUBBATCHES="1", B2_ALIGN_PATH="tiled", B2_REF_PACKED="0")),
    ("tracks", 16000, dict(B2_SUBBATCHES="3", B2_ALIGN_PATH="runs")),
    ("tracks", 48000, dict(B2_SUBBATCHES="3", B2_ALIGN_PATH="big", B2_BIG_WS_MB="64")),
    ("tracks", 16000, dict(B2_SUBBATCHES="3", B2_VAD_LAYOUT="group", B2_REF_PACKED="1")),
    ("gss", 16000, dict(B2_SUBBATCHES="1")),
    ("auditok", 16000, dict(B2_SUBBATCHES="3")),
    ("seg", 48000, dict(B2_SUBBATCHES="3", B2_ALIGN_PATH="tiled")),
    ("seg", 16000, dict(B2_SUBBATCHES="1", B2_ALIGN_PATH="runs")),
]


@pytest.fixture(scope="module")
def far_buffer(handle):
    import torch
    _free()
    _need(2 * BUF + 4 * GB)
    buf = torch.empty(BUF, dtype=torch.int16, device="cuda")
    _note()
    yield buf
    del buf
    _free()


@pytest.mark.parametrize("entry,fr,knobs", FAR_CASES, ids=lambda x: str(x) if not isinstance(x, dict) else
                         "-".join("%s=%s" % (k[3:], v) for k, v in sorted(x.items())))
def test_far_placement_sync(handle, far_buffer, entry, fr, knobs, monkeypatch):
    import torch
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)
    req = _far_req(entry, fr, knobs)
    where = "%s %d %s" % (entry, fr, knobs)
    a = rr.arrays(req)
    pcms = _pcms(req)
    pcm = np.concatenate(pcms)
    refs = [_reference(req, d, pcms[v]) for v, d in enumerate(req["videos"])]
    ref64 = [r.astype(np.float64) for r in refs]
    trk, grid, mos = req["tracks"], req["ratios"], req["mos"]
    for tr in trk:
        tr["keep"] = None
    subs = [[_sub(tr, r, None) for r in grid] for tr in trk]
    exact = RunExact()
    gss = entry == "gss"
    traces = {t: _gss_trace(exact, ref64[tr["video"]], tr, None, mos) for t, tr in enumerate(trk) if gss}
    V = len(req["videos"])
    speech = list(range(V))
    cap_n = int(sum(len(r) for r in refs)) + 4096

    # at offset 0, against the composed oracle
    near = torch.from_numpy(pcm).cuda()
    got, cap, sp, nom = _run_sync(handle, req, a, near.data_ptr(), speech, cap_n, gss)
    check_capture(cap, refs, where=where)
    assert np.array_equal(sp["off"], np.concatenate([[0], np.cumsum([len(r) for r in refs])])), where
    for v in speech:
        assert np.array_equal(sp["buf"][sp["off"][v]:sp["off"][v + 1]], ref64[v]), (where, "speech", v)
    if gss:
        overflow = np.array([[_exact_window_near(exact, ref64[tr["video"]], s, mos) > nc.K_CAND for s in subs[t]]
                             for t, tr in enumerate(trk)], bool)
    else:
        overflow = (nom["cand"] > nc.K_CAND).reshape(len(trk), len(grid))
    _check_outputs(req, a, got, ref64, subs, exact, overflow, traces, where)
    del near
    resident = None
    if entry == "batch":
        hold = []
        near = torch.from_numpy(pcm).cuda()
        resident = _call(handle, req, a, near.data_ptr(), "device", want_all=True, resident=True, keep=hold)
        handle.synchronize()
        names = ("best_score", "best_offset", "best_k", "all_score", "all_offset")
        _same([resident[k].cpu().numpy() for k in names], got, (where, "resident"))
        del near, hold

    # far: every output bit for bit
    for X in _placements(len(pcm)):
        far_buffer[X:X + len(pcm)].copy_(torch.from_numpy(pcm))
        fa = dict(a, pcm_off=a["pcm_off"] + X)
        w = (where, "at", X)
        g2, c2, s2, n2 = _run_sync(handle, req, fa, far_buffer.data_ptr(), speech, cap_n, gss)
        _same(g2, got, w)
        if np.array_equal(c2["packed"], cap["packed"]):
            for k in ("ref", "ref_off"):
                assert np.array_equal(c2[k], cap[k], equal_nan=True), (w, k)
        else:   # an unaligned start leaves the lane kernel, so the reference is not packed there
            check_capture(c2, refs, where=w)
        assert np.array_equal(s2["off"], sp["off"]) and np.array_equal(s2["buf"], sp["buf"], equal_nan=True), w
        if nom is not None:
            for k in nom:
                assert np.array_equal(n2[k], nom[k], equal_nan=True), (w, "nominations", k)
        if entry == "batch":
            hold = []
            r2 = _call(handle, req, fa, far_buffer.data_ptr(), "device", want_all=True, resident=True, keep=hold)
            handle.synchronize()
            _same([r2[k].cpu().numpy() for k in names], got, (w, "resident"))


@pytest.mark.parametrize("fr", [16000, 48000])
@pytest.mark.parametrize("detector", ["energy_zcr", "auditok"])
def test_far_placement_vad(handle, far_buffer, fr, detector):
    """b2_vad_energy_zcr / b2_vad_auditok (B2_DEVICE) over the far batch equal the batch at offset 0, which equals the
    detector oracle per video.  auditok's device pointer is pcm + pcm_off[0], which must be 16-byte aligned: an
    unaligned placement gets a silent video in front from the aligned sample below."""
    import torch
    from ffsubsync_b200 import _native as N
    req = _far_req("tracks", fr, {}, detector=detector)
    pcms = _pcms(req)
    pcm = np.concatenate(pcms)
    off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
    chunk = rr.chunk_samples(fr)

    def run(ptr, pcm_off):
        if detector == "auditok":
            out_off = handle.auditok_out_off(pcm_off, fr, 100, chunk)
            out = torch.full((int(out_off[-1]) + 1,), 7.0, dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()   # the fill and the buffer's copies run on torch's stream, the call on the handle's
            handle.vad_auditok(ptr, pcm_off, fr, 100, -0.5, chunk_samples=chunk, out=out.data_ptr(),
                               memspace=N.B2_DEVICE)
        else:
            fpw = handle.frames_per_window(fr, 100)
            out_off = np.concatenate([[0], np.cumsum((np.diff(pcm_off) + fpw - 1) // fpw)]).astype(np.int64)
            out = torch.full((int(out_off[-1]) + 1,), 7.0, dtype=torch.float32, device="cuda")
            torch.cuda.synchronize()
            handle.vad_energy_zcr(ptr, pcm_off, fr, 100, -0.5, THR, out=out.data_ptr(), memspace=N.B2_DEVICE)
        handle.synchronize()
        _note()
        return out.cpu().numpy(), out_off

    near = torch.from_numpy(pcm).cuda()
    want, want_off = run(near.data_ptr(), off)
    assert want[-1] == 7.0
    for v, p in enumerate(pcms):
        w = want[want_off[v]:want_off[v + 1]]
        if detector == "auditok":
            exp = co.chunk_loop("auditok", p, fr, 100, chunk=chunk, non_speech_label=-0.5)
        else:
            exp = vo.energy_zcr_detect(p, 100, fr, -0.5, THR)
        assert np.array_equal(w, np.asarray(exp, w.dtype)), (fr, detector, v)
    del near
    for X in _placements(len(pcm)):
        far_buffer[X:X + len(pcm)].copy_(torch.from_numpy(pcm))
        pcm_off, skip = off + X, 0
        if detector == "auditok" and X % 8:
            A = X - X % 8
            far_buffer[A:X].zero_()
            pcm_off, skip = np.concatenate([[A], off + X]), 1
        got, got_off = run(far_buffer.data_ptr(), pcm_off)
        got = got[got_off[skip]:]
        if skip and detector == "auditok":
            assert np.all(got_off[1] == (X - A + fr // 100 - 1) // (fr // 100))
        assert np.array_equal(got, want), (fr, detector, X, np.flatnonzero(got != want)[:8])


# ============================================================================================ B. one long video

BAND = 12000          # windows on each side of the window that holds sample 2^31: the 100 s reads around it too


def _long_classes(n, fpw, seed):
    """Window classes of a video of n samples: runs of silence and voiced speech (20 windows to 30 s), random classes
    with loud hiss in the band around sample 2^31 (byte 2^32) and in 40 seeded windows elsewhere."""
    rng = np.random.RandomState(seed)
    W = -(-n // fpw)
    runs = rng.randint(20, 3000, W // 20 + 2)
    cls = np.repeat(np.arange(len(runs)) % 2, runs)[:W].astype(np.uint8)
    c = M31 // fpw
    c1 = min(W, c + BAND)
    cls[c - BAND:c1] = rng.choice(3, c1 - c + BAND, p=[0.4, 0.4, 0.2])
    spots = np.sort(rng.choice(W - 200, 40, replace=False))
    for s in spots:
        cls[s:s + 100] = rng.choice(3, 100, p=[0.4, 0.4, 0.2])
    return cls, [(c - BAND, c1)] + [(int(s), int(s) + 100) for s in spots] + [(W - 300, W)]


def _decided(cls, label):
    """The per-window decision that follows from the class alone: voiced speech has |x| >= 6000 - 2048 with the
    square wave's sign, so E >= fpw * 3952^2 and 11 crossings (within 0 .. 3 fpw / 8) - speech for energy / ZCR and
    above auditok's 50 dB; silence has |x| <= 32 - below both thresholds.  Hiss is decided from its samples."""
    return np.where(cls == 1, 1.0, label)


def _slice(pcm_t, s0, s1):
    return pcm_t[s0:s1].cpu().numpy()


def _energy_ref(pcm_t, n, fpw, cls, bands, label):
    """The energy / ZCR reference (one detector call: the 100 s reads divide into windows at 48 and 44.1 kHz): the
    classes' decisions, with the bands' windows recomputed exactly from their samples."""
    ref = _decided(cls, label)
    W = len(cls)
    ref[W - 1] = label if n % fpw else ref[W - 1]
    for w0, w1 in bands:
        s1 = min(n, w1 * fpw)
        ref[w0:w1] = vo.energy_zcr_detect(_slice(pcm_t, w0 * fpw, s1), 100, fpw * 100, label, THR)
    return ref.astype(np.float32)


def _auditok_ref(pcm_t, n, fpw, cls, bands, chunk, label):
    """auditok over 100 s reads: block validity from the classes (from the samples in the bands and at the end),
    then the tokenizer per read."""
    valid = cls == 1
    floor = ad.energy_floor(fpw)
    for w0, w1 in bands:
        s1 = min(n, w1 * fpw)
        x = _slice(pcm_t, w0 * fpw, s1).astype(np.int64)
        full = len(x) // fpw
        valid[w0:w0 + full] = (x[:full * fpw].reshape(full, fpw) ** 2).sum(1) >= floor
        if len(x) % fpw:
            tail = x[full * fpw:]
            valid[w0 + full] = (tail * tail).sum() >= ad.energy_floor(len(tail))
    per = chunk // fpw
    assert chunk % fpw == 0
    out = []
    for k in range(0, len(valid), per):
        v = valid[k:k + per]
        bs = np.zeros(len(v) + 1)
        for s, e in ad.tokenize(list(v), 20.0, 500, 25.0):
            bs[s] = 1.0
            bs[e + 1] = label - 1.0
        out.append(np.clip(np.cumsum(bs)[:-1], 0.0, 1.0))
    return np.concatenate(out)


def _long_cues(seed, hours, n_sec):
    """A cue every 40 to 80 s over the whole video, 1 to 4 s long."""
    rng = np.random.RandomState(seed)
    st, t = [], 3.0
    while t < n_sec - 10:
        st.append(round(t, 3))
        t += rng.uniform(40, 80)
    st = np.array(st)
    return st, np.round(st + rng.uniform(1, 4, len(st)), 3)


LONG = [(48000, M31 + 4321), (44100, M31 + 2 * 44100 + 1)]


@pytest.fixture(scope="module", params=LONG, ids=["48k", "44k1"])
def long_video(request, handle):
    import torch
    fr, n = request.param
    fpw = int(fr / 100 + 0.5)
    _free()
    _need(2 * n + 6 * GB)
    cls, bands = _long_classes(n, fpw, fr)
    W = len(cls)
    pcm = torch.empty(W * fpw, dtype=torch.int16, device="cuda")
    d_cls = torch.from_numpy(cls).cuda()
    torch.cuda.synchronize()
    from ffsubsync_b200 import _native as N
    handle.synth_pcm(d_cls.data_ptr(), W, fpw, 7, out=pcm.data_ptr(), memspace=N.B2_DEVICE)
    handle.synchronize()
    del d_cls
    # the synthesiser's samples at the bands equal the host generator's
    for w0, w1 in bands[:3]:
        assert np.array_equal(_slice(pcm, w0 * fpw, w1 * fpw), vo.synth_pcm(cls[w0:w1], fpw, 7, w0 * fpw))
    _note()
    yield dict(fr=fr, n=n, fpw=fpw, cls=cls, bands=bands, pcm=pcm)
    del pcm
    _free()


def test_long_video_vad(handle, long_video):
    import torch
    from ffsubsync_b200 import _native as N
    L = long_video
    fr, n, fpw, pcm = L["fr"], L["n"], L["fpw"], L["pcm"]
    want = _energy_ref(pcm, n, fpw, L["cls"], L["bands"], -0.5)
    out = torch.full((len(want) + 1,), 7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()   # the fill runs on torch's stream, the call on the handle's
    handle.vad_energy_zcr(pcm.data_ptr(), [0, n], fr, 100, -0.5, THR, out=out.data_ptr(), memspace=N.B2_DEVICE)
    handle.synchronize()
    got = out.cpu().numpy()
    assert got[-1] == 7.0 and np.array_equal(got[:-1], want), np.flatnonzero(got[:-1] != want)[:8]
    del out
    chunk = rr.chunk_samples(fr)
    want = _auditok_ref(pcm, n, fpw, L["cls"], L["bands"], chunk, -0.5)
    out = torch.full((len(want) + 1,), 7.0, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    handle.vad_auditok(pcm.data_ptr(), [0, n], fr, 100, -0.5, chunk_samples=chunk, out=out.data_ptr(),
                       memspace=N.B2_DEVICE)
    handle.synchronize()
    got = out.cpu().numpy()
    _note()
    assert got[-1] == 7.0 and np.array_equal(got[:-1], want), np.flatnonzero(got[:-1] != want)[:8]


def _long_req(L, entry, detector):
    """The long video, then a text subtitle, a PGS and a stored-signal video; cues over all 12 h on the long video."""
    fr, n = L["fr"], L["n"]
    rng = np.random.RandomState(5)
    videos = [dict(kind="audio", n=n, dur=n / fr)]
    if entry != "gss":
        st, en = ro.synthetic_cues(3, 200.0)
        videos.append(dict(kind="subs", starts=st, ends=en, keep=np.ones(len(st), np.uint8), dur=200.0))
        st, en = ro.synthetic_cues(4, 150.0)
        videos.append(dict(kind="pgs", starts=st + 0.004, ends=en + 0.006, dur=150.0))
        videos.append(dict(kind="sig", x=rng.choice([0.0, 1.0], 15000).astype(np.float64), dur=150.0))
    tracks = []
    for i, sh in enumerate([-12.37, 33.0]):
        st, en = _long_cues(20 + i, 12, n / fr)
        tracks.append(dict(video=0, starts=np.maximum(st + sh, 0.0), ends=np.maximum(en + sh, 0.5)))
    for v in range(1, len(videos)):
        st, en = ro.synthetic_cues(40 + v, 160.0)
        tracks.append(dict(video=v, starts=st + 1.5, ends=en + 1.5))
    K5 = [1.0, 24 / 23.976, 25 / 23.976, 23.976 / 25, 25 / 24.0]
    return dict(seed=5, entry=entry, fr=fr, videos=videos, tracks=tracks, ratios=K5 if entry != "gss" else K5[:2],
                mos=6000, label=0.0, memspace="device", knobs={}, detector=detector, chunk=rr.chunk_samples(fr),
                keep_tracks=False, keep_seed=1)


@pytest.mark.parametrize("entry,detector,path", [("sig", "energy_zcr", "tiled"), ("sig", "energy_zcr", "runs"),
                                                 ("sig", "auditok", "tiled"), ("gss", "energy_zcr", None)])
def test_long_video_sync(handle, long_video, entry, detector, path, monkeypatch):
    """Reference, speech output and every (track, ratio) against the oracle; then the ingest session fed the long
    video in 100 s reads returns the same outputs."""
    import torch
    from ffsubsync_b200 import _native as N
    if path:
        monkeypatch.setenv("B2_ALIGN_PATH", path)
    L = long_video
    fr, n, fpw, pcm = L["fr"], L["n"], L["fpw"], L["pcm"]
    req = _long_req(L, entry, detector)
    where = "%s %s %s %d" % (entry, detector, path, fr)
    a = rr.arrays(req)
    if detector == "auditok":
        long_ref = _auditok_ref(pcm, n, fpw, L["cls"], L["bands"], req["chunk"], req["label"]).astype(np.float32)
    else:
        long_ref = _energy_ref(pcm, n, fpw, L["cls"], L["bands"], req["label"])
    refs = [long_ref] + [_reference(req, d, None) for d in req["videos"][1:]]
    ref64 = [r.astype(np.float64) for r in refs]
    trk, grid, mos = req["tracks"], req["ratios"], req["mos"]
    for tr in trk:
        tr["keep"] = None
    subs = [[_sub(tr, r, None) for r in grid] for tr in trk]
    exact = RunExact()
    gss = entry == "gss"
    traces = {t: _gss_trace(exact, ref64[tr["video"]], tr, None, mos) for t, tr in enumerate(trk) if gss}
    V = len(req["videos"])
    cap_n = int(sum(len(r) for r in refs)) + 4096
    if gss:
        _poison(handle, cap_n)
        with handle.capture_reference(cap_n, V + 3) as cap:
            got = _call(handle, req, a, pcm.data_ptr(), "device", want_all=True)
        sp = None
        overflow = np.array([[_exact_window_near(exact, ref64[tr["video"]], s, mos) > nc.K_CAND for s in subs[t]]
                             for t, tr in enumerate(trk)], bool)
    else:
        got, cap, sp, nom = _run_sync(handle, req, a, pcm.data_ptr(), list(range(V)), cap_n, False)
        overflow = (nom["cand"] > nc.K_CAND).reshape(len(trk), len(grid))
    _note()
    check_capture(cap, refs, where=where)
    if sp is not None:
        for v in range(V):
            assert np.array_equal(sp["buf"][sp["off"][v]:sp["off"][v + 1]], ref64[v]), (where, "speech", v)
    _check_outputs(req, a, got, ref64, subs, exact, overflow, traces, where)
    if gss or path == "runs":
        return

    # the ingest session: the long video in 100 s reads (and two odd-length ones around byte 2^32), the other videos'
    # references from the tables; no capture now, so the outputs are those of the plain whole call
    plain = _call(handle, req, a, pcm.data_ptr(), "device", want_all=True)
    det = dict(detector=N.B2_DETECTOR_AUDITOK if detector == "auditok" else N.B2_DETECTOR_ENERGY_ZCR,
               energy_threshold=THR, chunk_samples=req["chunk"])
    handle.ingest_begin(V, fr, 100, req["label"], **det)
    step = rr.chunk_samples(fr)
    cuts = sorted(set(list(range(0, n, step)) + [M31 - 777, M31 + 1001, n]))
    for s0, s1 in zip(cuts[:-1], cuts[1:]):
        chunk = _slice(pcm, s0, s1)
        b = chunk.view(np.uint8)
        if s1 == M31 - 777:          # an odd byte count: the last sample's high byte arrives with the next push
            handle.ingest_push([0], [b[:-1]])
            held = b[-1:]
            continue
        if s0 == M31 - 777:
            b = np.concatenate([held, b])
        handle.ingest_push([0], [b])
    res = handle.ingest_sync_tracks(a["track_video"], a["cue_start"], a["cue_end"], None, a["cue_off"], grid, 0.0,
                                    mos, want_all=True, ref_is_subs=a["ref_is_subs"],
                                    ref_cue_start_s=a["ref_cue_start"], ref_cue_end_s=a["ref_cue_end"],
                                    ref_cue_keep=a["ref_cue_keep"], ref_cue_off=a["ref_cue_off"],
                                    ref_is_pgs=a["ref_is_pgs"], pgs_start_s=a["pgs_start"], pgs_end_s=a["pgs_end"],
                                    pgs_off=a["pgs_off"], ref_is_sig=a["ref_is_sig"], x=a["x"], sig_off=a["sig_off"])
    _note()
    _same([np.asarray(x) for x in res[:5]], plain[:5], (where, "ingest"))


def _exact_window_near(exact, ref, sub, mos):
    from test_gpu_random_requests import _exact_result
    return _exact_result(exact, ref, sub, mos)[2]


def test_long_video_segments(handle, long_video):
    """b2_sync_tracks_seg with sampled segments of the long video before sample 2^31, across it and from past it to
    the video's end: the reference against segment_oracle over the segments' samples."""
    L = long_video
    fr, n, fpw, pcm = L["fr"], L["n"], L["fpw"], L["pcm"]
    total = n / fr
    mark = M31 // fr                      # the second that holds sample 2^31
    starts = [mark - 20, mark - 1, mark]
    lo = [(mark - 20) * fr, M31 - 1000, M31 + 3]
    hi = [lo[0] + 10 * fr + 7, M31 + 500, n]
    assert hi[1] < n
    videos = [dict(kind="seg", n=n, total=total, starts=starts, lo=lo, hi=hi, dur=total)]
    st, en = _long_cues(9, 12, total)
    req = dict(seed=9, entry="seg", fr=fr, videos=videos, tracks=[dict(video=0, starts=st, ends=en)],
               ratios=[1.0, 25 / 24.0], mos=6000, label=0.0, memspace="device", knobs={}, detector="energy_zcr",
               chunk=rr.chunk_samples(fr), keep_tracks=False, keep_seed=1)
    a = rr.arrays(req)
    # segment_oracle reads the whole video's PCM at its lo / hi: hand it a sparse copy holding just those samples
    sparse = _Sparse(n, {a0: _slice(pcm, a0, b0) for a0, b0 in zip(lo, hi)})
    want = so.segment_reference(sparse, total, starts, lo, hi, 100, non_speech_label=0.0, frame_rate=fr,
                                energy_threshold=THR)
    want = np.asarray(want, np.float64).astype(np.float32)
    _poison(handle, len(want) + 4096)
    with handle.capture_reference(len(want) + 4096, 4) as cap:
        _call(handle, req, a, pcm.data_ptr(), "device", want_all=True)
    _note()
    check_capture(cap, [want], where=("segments", fr))


class _Sparse:
    """The slices segment_oracle takes of a video's PCM, without the rest of it."""

    def __init__(self, n, parts):
        self.n, self.parts = n, parts

    def __len__(self):
        return self.n

    def __getitem__(self, sl):
        assert isinstance(sl, slice) and (sl.step or 1) == 1
        for a0, x in self.parts.items():
            if a0 <= sl.start and sl.stop <= a0 + len(x):
                return x[sl.start - a0:sl.stop - a0]
        raise AssertionError("unexpected slice %r" % sl)
