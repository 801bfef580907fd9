"""GPU tests of the reference signal every batched sync call builds in its detector step (run on an H100).

b2_capture_reference copies a call's whole reference buffer out after its last kernel.  Each test prefills the
capture with NaN and compares every frame of every video with a plain restatement of the operation:
  * energy / ZCR videos: oracle.vad_oracle.energy_zcr_detect, rounded once to float32;
  * auditok videos: the auditok detector over the reference's chunk loop (oracle.auditok_oracle: the energy
    validator and StreamTokenizer), rounded once to float32;
  * text subtitle references: oracle.raster_oracle.rasterize at ratio 1.0 (level 1.0), keep flags and
    start_seconds;
  * PGS references: oracle.pgs_oracle.pgs_signal.
A video whose sub-batch got packed bits holds ceil(R/32) words that must equal the bits (oracle == 1.0f), every bit
past R zero; the rest of its range is not the signal's.  ref_off must be the oracle's lengths, and nothing past
ref_off[V] may be written.  Unlike the outputs, which a wrong frame changes only where a winning offset covers it,
this checks the frames before the window, the tail past the subtitles and every video of every sub-batch.

Each test also checks its premise: packed videos where the run path must run (B2_ALIGN_PATH=runs on the
lane-per-window kernel), and none under auditok, subtitle references, the lane-group kernel or B2_REF_PACKED=0.
The tokenizer tests build PCM from chosen flag strings (a valid block is +-400 alternating: E = 160 000 fpw >=
10^5 fpw; an invalid one is silent) and check both the float64 tokenizer (b2_vad_auditok) and the float32 in-place
one (b2_sync_tracks_auditok)."""
import contextlib
import json
import os

import numpy as np
import pytest

import cases
import test_raster_cpu as rc
from conftest import ROOT
from oracle import auditok_oracle as au
from oracle import pgs_oracle as po
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 25 / 24.0]
MOS = 3000
THR = 100000
LABELS = [0.0, 0.3, 1.0, -0.5]
ENTRIES = ["batch", "tracks", "gss", "auditok", "subs", "pgs"]
DEFAULT_TOK = (20.0, 500, 25.0)   # (0.2, 5, 0.25) s at 100 Hz: the reference's tokenizer


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@contextlib.contextmanager
def _env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _chunk(fr):
    """The Python layer's chunk: (2 fr // 100) * 5000 samples (100 s)."""
    return (2 * fr // 100) * 5000


# ------------------------------------------------------------------------------------------- inputs

def _classes(n, rng):
    """Window classes in runs of 1..60 (0 silence, 1 voiced, 2 loud hiss: energetic, many crossings)."""
    out = np.empty(n, np.uint8)
    i = 0
    while i < n:
        L = rng.randint(1, 61)
        out[i:i + L] = rng.choice(3, p=[0.45, 0.4, 0.15])
        i += L
    return out


def _audio(n_samples, fr, seed):
    w = max(1, fr // 100)
    rng = np.random.RandomState(seed)
    nwin = -(-n_samples // w)
    pcm = vo.synth_pcm(_classes(nwin, rng), w, seed)[:n_samples] if n_samples else np.zeros(0, np.int16)
    if n_samples % w:   # a loud, noisy partial window: speech if it were judged like a full one
        pcm[-(n_samples % w):] = rng.randint(-9000, 9000, n_samples % w).astype(np.int16)
    return pcm


def _track_cues(seed, dur=60.0):
    st, en = cases.synthetic_cues(seed, dur)
    r = np.random.RandomState(seed)
    delta = r.randint(-300, 300) / 100.0
    keep = (r.rand(len(st)) >= 0.1) & (st + delta >= 0)
    return np.round(st[keep] + delta, 3), np.round(en[keep] + delta, 3)


def _corpus(videos, fr=16000, seed=0):
    """videos: list of dicts: kind "audio" (n samples), "subs" (starts, ends, keep) or "pgs" (starts, ends); tracks:
    how many subtitle tracks sync against it (generic 60 s cue lists)."""
    pcms, tv, cs, ce = [], [], [], []
    is_subs, rs, re_, rk, r_off = [], [], [], [], [0]
    is_pgs, ps, pe, p_off = [], [], [], [0]
    for v, d in enumerate(videos):
        kind = d["kind"]
        pcms.append(_audio(d["n"], fr, seed + 31 * v + 7) if kind == "audio" else np.zeros(0, np.int16))
        is_subs.append(int(kind == "subs"))
        is_pgs.append(int(kind == "pgs"))
        if kind == "subs":
            rs.append(np.asarray(d["starts"], np.float64))
            re_.append(np.asarray(d["ends"], np.float64))
            rk.append(np.asarray(d["keep"], np.uint8))
        r_off.append(r_off[-1] + (len(d["starts"]) if kind == "subs" else 0))
        if kind == "pgs":
            ps.append(np.asarray(d["starts"], np.float64))
            pe.append(np.asarray(d["ends"], np.float64))
        p_off.append(p_off[-1] + (len(d["starts"]) if kind == "pgs" else 0))
        for i in range(d.get("tracks", 1)):
            a, b = _track_cues(seed * 1000 + 13 * v + i)
            tv.append(v)
            cs.append(a)
            ce.append(b)
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)   # noqa: E731
    return dict(videos=videos, fr=fr, pcms=pcms, pcm=cat(pcms, np.int16),
                pcm_off=np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64),
                tv=np.array(tv, np.int32), cs=cat(cs, np.float64), ce=cat(ce, np.float64),
                cue_off=np.concatenate([[0], np.cumsum([len(x) for x in cs])]).astype(np.int64),
                is_subs=np.array(is_subs, np.uint8), rs=cat(rs, np.float64), re=cat(re_, np.float64),
                rk=cat(rk, np.uint8), r_off=np.array(r_off, np.int64),
                is_pgs=np.array(is_pgs, np.uint8), ps=cat(ps, np.float64), pe=cat(pe, np.float64),
                p_off=np.array(p_off, np.int64))


def _win_videos(fpw, windows, tracks=1):
    """Audio videos of the given (windows, extra samples); extra samples make a trailing partial window."""
    return [dict(kind="audio", n=w * fpw + x, tracks=tracks) for w, x in windows]


# R mod 32 in {0, 1, 31}, R < 32, trailing partial windows (extra samples are multiples of 8, so every video stays
# 16-byte aligned), an empty video, and one of a single window
LENGTHS = [(32 * 40, 0), (32 * 40 + 1, 0), (32 * 40 + 31, 0), (20, 0), (31, 40), (0, 0), (32 * 7, 8), (1, 0),
           (33, 0), (64 + 5, 120)]


# ------------------------------------------------------------------------------------------- oracles

def _tok_signal(flags, tok, label):
    """The reference's _detect after the validity flags: tokens -> starts 1.0, ends label - 1.0, clipped cumsum."""
    m = np.zeros(len(flags) + 1)
    for s, e in au.tokenize(list(flags), *tok):
        m[s] = 1.0
        m[e + 1] = label - 1.0
    return np.clip(np.cumsum(m)[:-1], 0.0, 1.0)


def _auditok_flags(pcm, block):
    x = pcm.astype(np.int64)
    n_full = len(x) // block
    e = (x[: n_full * block].reshape(n_full, block) ** 2).sum(axis=1)
    fl = list(e >= au.energy_floor(block, 50))
    tail = x[n_full * block:]
    if len(tail):
        fl.append(bool((tail * tail).sum() >= au.energy_floor(len(tail), 50)))
    return fl


def _auditok_oracle(pcm, fr, label, chunk, tok):
    """The reference's chunk loop (speech_transformers.py: one detector call per chunk of chunk samples)."""
    step = chunk if chunk > 0 else max(len(pcm), 1)
    parts = []
    for i in range(0, len(pcm), step):
        seg = pcm[i:i + step]
        if tok == DEFAULT_TOK:
            parts.append(au.auditok_detect_fast(seg.tobytes(), 100, fr, label))
        else:
            parts.append(_tok_signal(_auditok_flags(seg, fr // 100), tok, label))
    return np.concatenate(parts) if parts else np.zeros(0)


def _oracle(c, detector, label, chunk=None, tok=DEFAULT_TOK, ss=0.0):
    """The float32 reference of every video of corpus c."""
    out = []
    chunk = _chunk(c["fr"]) if chunk is None else chunk
    for v, d in enumerate(c["videos"]):
        if d["kind"] == "subs":
            w = ro.rasterize(d["starts"], d["ends"], np.asarray(d["keep"], bool), 100, ss, 1.0)[0]
        elif d["kind"] == "pgs":
            w = po.pgs_signal(list(zip(d["starts"], d["ends"])), 100, ss)
        elif detector == "auditok":
            w = _auditok_oracle(c["pcms"][v], c["fr"], label, chunk, tok)
        else:
            w = vo.energy_zcr_detect(c["pcms"][v], 100, c["fr"], label, THR)
        out.append(np.asarray(w, np.float64).astype(np.float32))
    return out


def _words(w32):
    """ceil(R/32) uint32 words of the bits (r == 1.0f), bit i of word k = frame 32k + i, zero past R."""
    n = len(w32)
    bits = np.zeros(-(-n // 32) * 32, np.uint64)
    bits[:n] = w32 == np.float32(1.0)
    return (bits.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)


def _check(cap, want, packed=None, where="", tail=True):
    """cap: a capture_reference dict; want: per-video float32 oracle.  packed: None (not checked), True (every
    non-empty video packed), False (none).  tail: nothing past ref_off[V] was written (one call only)."""
    V = len(want)
    ref, ref_off, pk = cap["ref"], cap["ref_off"], cap["packed"]
    lens = np.array([len(w) for w in want], np.int64)
    assert np.array_equal(ref_off[: V + 1], np.concatenate([[0], np.cumsum(lens)])), (where, ref_off[: V + 1], lens)
    assert set(pk[:V].tolist()) <= {0, 1}, (where, pk[:V])
    if packed is not None:
        assert all(bool(pk[v]) == packed for v in range(V) if lens[v] > 0), (where, "premise: packed", pk[:V])
    words = ref.view(np.uint32)
    for v, w in enumerate(want):
        a = int(ref_off[v])
        if pk[v]:
            got, exp = words[a: a + -(-len(w) // 32)], _words(w)
        else:
            got, exp = ref[a: a + len(w)], w
        assert len(got) == len(exp), (where, "video", v, len(got), len(exp))
        bad = np.flatnonzero(got != exp)   # the oracle has no NaN: a frame the call did not write fails
        assert len(bad) == 0, (where, "video", v, "packed", int(pk[v]), "R", len(w), "first bad", bad[:8].tolist(),
                               got[bad[:8]].tolist(), exp[bad[:8]].tolist())
    if tail:
        rest = ref[int(ref_off[V]):]
        assert np.isnan(rest).all(), (where, "written past ref_off[V]", np.flatnonzero(~np.isnan(rest))[:8])


def _capacity(want):
    return int(sum(len(w) for w in want)) + 4096


# ------------------------------------------------------------------------------------------- calls

def _device_args(c, entry):
    """Corpus c's PCM uploaded and the outputs of an `entry` call allocated with torch, then a device synchronise:
    (pcm pointer, output pointers, the tensors, which must outlive the call)."""
    import torch
    T = len(c["tv"])
    pcm_t = torch.from_numpy(c["pcm"]).cuda() if len(c["pcm"]) else None
    t = dict(best_score=torch.empty(T, dtype=torch.float64, device="cuda"),
             best_offset=torch.empty(T, dtype=torch.int32, device="cuda"),
             best_k=torch.empty(T, dtype=torch.int32, device="cuda"))
    if entry == "gss":
        t["gss_ratio"] = torch.empty(T, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    return (pcm_t.data_ptr() if pcm_t is not None else None), {k: v.data_ptr() for k, v in t.items()}, (pcm_t, t)


def _call(handle, c, entry, label=0.0, memspace=None, chunk=None, tok=DEFAULT_TOK, ss=0.0, detector="energy",
          want_all=True, keep=None, dev=None):
    """One batched sync call of `entry` over corpus c.  Device memspaces take `dev` (_device_args, nothing is
    synchronised then) or upload the PCM and allocate the outputs here (kept alive in `keep` until the caller
    synchronises the handle)."""
    from ffsubsync_b200 import _native as N
    memspace = N.B2_HOST if memspace is None else memspace
    fr = c["fr"]
    chunk = _chunk(fr) if chunk is None else chunk
    pcm = c["pcm"]
    outs = {}
    if memspace != N.B2_HOST:
        if dev is None:
            dev = _device_args(c, entry)
            if keep is not None:
                keep.append(dev[2])
        pcm, outs = dev[0], dev[1]
        want_all = False
    common = dict(memspace=memspace, want_all=want_all, **outs)
    tk = dict(min_length=tok[0], max_length=tok[1], max_continuous_silence=tok[2])
    det = 1 if detector == "auditok" else 0
    if entry == "batch":
        return handle.sync_batch(pcm, c["pcm_off"], fr, 100, label, THR, -1, -1, c["cs"], c["ce"], None, c["cue_off"],
                                 GRID, ss, MOS, **common)
    if entry in ("tracks", "gss"):
        f = handle.sync_tracks if entry == "tracks" else handle.sync_tracks_gss
        if entry == "gss":
            common["want_evals"] = want_all
        return f(pcm, c["pcm_off"], c["tv"], fr, 100, label, THR, -1, -1, c["cs"], c["ce"], None, c["cue_off"], GRID,
                 ss, MOS, **common)
    if entry == "auditok":
        return handle.sync_tracks_auditok(pcm, c["pcm_off"], c["tv"], fr, 100, label, c["cs"], c["ce"], None,
                                          c["cue_off"], GRID, ss, MOS, chunk, **tk, **common)
    if entry == "subs":
        return handle.sync_tracks_subs(pcm, c["pcm_off"], c["tv"], fr, 100, label, c["is_subs"], c["rs"], c["re"],
                                       c["rk"], c["r_off"], c["cs"], c["ce"], None, c["cue_off"], GRID, ss, MOS,
                                       detector=det, energy_threshold=THR, chunk_samples=chunk, **tk, **common)
    assert entry == "pgs"
    return handle.sync_tracks_pgs(pcm, c["pcm_off"], c["tv"], fr, 100, label, c["is_pgs"], c["ps"], c["pe"],
                                  c["p_off"], c["cs"], c["ce"], None, c["cue_off"], GRID, ss, MOS,
                                  ref_is_subs=c["is_subs"], ref_cue_start_s=c["rs"], ref_cue_end_s=c["re"],
                                  ref_cue_keep=c["rk"], ref_cue_off=c["r_off"], detector=det, energy_threshold=THR,
                                  chunk_samples=chunk, **tk, **common)


_POISON = {}


def _poison(handle, n_frames):
    """Fill the first n_frames of the handle's reference buffer with -7.0, a value no reference holds: one 8 kHz
    silent video at label -7, as floats.  A frame the next call fails to write then cannot pass for one that an
    identical earlier call wrote."""
    import torch
    from ffsubsync_b200 import _native as N
    n = n_frames * 80
    if _POISON.get("pcm") is None or _POISON["pcm"].numel() < n:
        _POISON["pcm"] = torch.zeros(max(n, 1 << 20), dtype=torch.int16, device="cuda")
        _POISON["out"] = torch.empty(4, dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
    out = _POISON["out"].data_ptr()
    with _env(B2_REF_PACKED=0, B2_SUBBATCHES=1):
        handle.sync_tracks(_POISON["pcm"].data_ptr(), [0, n], [0], 8000, 100, -7.0, THR, -1, -1, [0.5], [1.5], None,
                           [0, 1], [1.0], 0.0, 100, best_score=out, best_offset=out + 8, best_k=out + 16,
                           memspace=N.B2_DEVICE)
    handle.synchronize()


def _captured(handle, c, want, run):
    _poison(handle, _capacity(want))
    with handle.capture_reference(_capacity(want), len(want) + 3) as cap:
        keep = []
        run(keep)
    return cap


# ------------------------------------------------------------------------------- entry points, memory

def _mixed_corpus(pgs, fr=16000, seed=5):
    """Audio videos (lengths of LENGTHS), text references and (pgs) PGS references in one call."""
    fpw = fr // 100
    rng = np.random.RandomState(seed)
    vids = _win_videos(fpw, LENGTHS[:5])
    st, en = cases.synthetic_cues(seed, 90.0)
    vids.insert(1, dict(kind="subs", starts=st, ends=en, keep=rng.rand(len(st)) < 0.8, tracks=2))
    if pgs:
        vids.insert(4, dict(kind="pgs", starts=st[::2] + 0.004, ends=en[::2] + 0.006, tracks=1))
    vids.append(dict(kind="subs", starts=np.zeros(0), ends=np.zeros(0), keep=np.zeros(0), tracks=1))
    vids += _win_videos(fpw, LENGTHS[5:])
    return _corpus(vids, fr, seed)


@pytest.fixture(scope="module")
def energy_corpus():
    return _corpus(_win_videos(160, LENGTHS, tracks=1), 16000, 1)


@pytest.fixture(scope="module")
def mixed_corpus():
    """The corpus of each subtitle entry point: text references for b2_sync_tracks_subs, text and PGS for _pgs."""
    return {"subs": _mixed_corpus(False), "pgs": _mixed_corpus(True)}


@pytest.mark.parametrize("memspace", ["host", "device", "resident"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_entry_points_and_memory(handle, energy_corpus, mixed_corpus, entry, memspace):
    """Every entry point under every memory space, on the run path: the energy entry points' references packed,
    auditok's and the subtitle calls' (subtitle references in the one sub-batch) as floats."""
    from ffsubsync_b200 import _native as N
    ms = {"host": N.B2_HOST, "device": N.B2_DEVICE, "resident": N.B2_DEVICE_RESIDENT}[memspace]
    c = mixed_corpus[entry] if entry in ("subs", "pgs") else energy_corpus
    detector = "auditok" if entry == "auditok" else "energy"
    want = _oracle(c, detector, 0.0)
    with _env(B2_ALIGN_PATH="runs"):
        cap = _captured(handle, c, want, lambda keep: _call(handle, c, entry, 0.0, ms, detector=detector, keep=keep))
    _check(cap, want, packed=entry in ("batch", "tracks", "gss"), where=(entry, memspace))


@pytest.mark.parametrize("entry", ["subs", "pgs"])
def test_subtitle_calls_with_auditok(handle, mixed_corpus, entry):
    """The subtitle calls with the auditok detector: the tokenizer's chunk tables skip the subtitle videos."""
    c = mixed_corpus[entry]
    want = _oracle(c, "auditok", 0.0, chunk=160 * 333)
    cap = _captured(handle, c, want, lambda keep: _call(handle, c, entry, 0.0, detector="auditok", chunk=160 * 333))
    _check(cap, want, packed=False, where=entry)


# --------------------------------------------------------------------- sub-batches, partitioned VAD

@pytest.mark.parametrize("mode", ["packed", "floats", "auditok"])
@pytest.mark.parametrize("n_sub", [1, 2, 3, 4])
def test_sub_batches_on_few_sms(handle, energy_corpus, n_sub, mode):
    """B2_SUBBATCHES = 1..4 with B2_VAD_SMS=8: the later sub-batches' lane kernel on 8 CTAs, writing packed words,
    floats (B2_REF_PACKED=0) or auditok's energy flags."""
    detector = "auditok" if mode == "auditok" else "energy"
    entry = "tracks" if detector == "energy" else "auditok"
    knobs = dict(B2_SUBBATCHES=n_sub, B2_VAD_SMS=8, B2_ALIGN_PATH="runs")
    if mode == "floats":
        knobs["B2_REF_PACKED"] = "0"
    want = _oracle(energy_corpus, detector, 0.0)
    with _env(**knobs):
        cap = _captured(handle, energy_corpus, want, lambda keep: _call(handle, energy_corpus, entry, 0.0))
    _check(cap, want, packed=mode == "packed", where=(n_sub, mode))


def test_default_call_with_96_tracks(handle):
    """>= 96 tracks: the default pipeline.  The launch count shows that the call was cut into sub-batches; the plan
    cuts a call without B2_SUBBATCHES only where it also gives the later sub-batches' VAD 54 % of the SMs, so this is
    the partitioned launch at its default size (test_sub_batches_on_few_sms pins it on 8 SMs)."""
    c = _corpus(_win_videos(160, [(3000 + 37 * i, 8 * (i % 3)) for i in range(32)], tracks=3), 16000, 96)
    assert len(c["tv"]) == 96
    want = _oracle(c, "energy", 0.0)
    n = []
    for knobs in (dict(B2_SUBBATCHES=1), {}):
        n0 = handle.launch_count
        with _env(**knobs):
            _call(handle, c, "tracks", 0.0)
        n.append(handle.launch_count - n0)
    assert n[1] > n[0], n   # premise: the default call was cut into sub-batches
    cap = _captured(handle, c, want, lambda keep: _call(handle, c, "tracks", 0.0))
    _check(cap, want, where="96 tracks")


# ----------------------------------------------------------------------------------- resident chains

@pytest.fixture(scope="module")
def chain_corpora():
    """Four different corpora: a buffer's previous content is never the reference the next call writes there.  The
    second and fourth have one track per video (b2_sync_batch)."""
    a = _corpus(_win_videos(160, [(30000, 0), (12345, 40), (32 * 500 + 1, 0), (31, 0)], tracks=2), 16000, 71)
    b = _corpus(_win_videos(160, [(20000 + 32, 0), (0, 0), (32 * 300 + 31, 8), (25000, 0), (7, 0)], tracks=1),
                16000, 72)
    c = _corpus(_win_videos(160, [(28001, 8), (32 * 400, 0), (5, 0)], tracks=3), 16000, 73)
    d = _corpus(_win_videos(160, [(32 * 700 + 31, 0), (31000, 40), (0, 0), (19, 0)], tracks=1), 16000, 74)
    return a, b, c, d


@pytest.mark.parametrize("n_calls", [1, 2, 3, 4])
def test_resident_chain(chain_corpora, n_calls, capfd):
    """The capture set once, then n resident calls (two sub-batches each, so they chain) over four corpora and two
    entry points, enqueued with no synchronisation between them: the last call's reference, from WS_SIG_REF (odd n)
    or WS_SIG_REF2 (even n).  A sleep kernel on the caller's stream ahead of every call but the last holds that
    call's chains back, so each later call finds its predecessor still running: its sub-batch 0 starts behind the
    predecessor's fence, on the SM partition (B2_VAD_SMS=8, like sub-batch 1 of every call), and writes the other
    buffer while the predecessor's chains and capture copy are still queued.  The last call runs with
    B2_PIPE_TRACE=1, whose line proves the premise (chained, predecessor busy, two sub-batches, 8 VAD SMs); every
    corpus is shown to be cut in two by its launch count."""
    import torch
    from ffsubsync_b200 import _native as N
    seq = list(zip(chain_corpora, ["tracks", "batch", "tracks", "batch"]))
    want = _oracle(seq[n_calls - 1][0], "energy", 0.0)
    cap_n = max(_capacity(_oracle(x, "energy", 0.0)) for x, _ in seq)
    stream = torch.cuda.Stream()
    handle = N.Handle(torch.cuda.current_device())   # on a stream of its own, which the sleeps can delay
    handle.set_stream(stream.cuda_stream)
    try:
        devs = [_device_args(x, e) for x, e in seq]
        with _env(B2_ALIGN_PATH="runs"):
            for (x, e), dev in zip(seq, devs):   # premise: every corpus is cut into two sub-batches
                n = []
                for n_sub in (1, 2):
                    with _env(B2_SUBBATCHES=n_sub):
                        n0 = handle.launch_count
                        _call(handle, x, e, 0.0, N.B2_DEVICE, dev=dev)
                        n.append(handle.launch_count - n0)
                assert n[1] > n[0], (e, n)
            with _env(B2_SUBBATCHES=2, B2_VAD_SMS=8):
                for (x, e), dev in zip(seq, devs):   # grow both buffers and every workspace before the chain
                    _call(handle, x, e, 0.0, N.B2_DEVICE_RESIDENT, dev=dev)
                handle.synchronize()
                _poison(handle, cap_n)
                capfd.readouterr()
                with handle.capture_reference(cap_n, 8) as cap:
                    for i, ((x, e), dev) in enumerate(zip(seq[:n_calls], devs)):
                        last = i == n_calls - 1
                        if not last:
                            with torch.cuda.stream(stream):
                                torch.cuda._sleep(200_000_000)   # about 0.1 s
                        with _env(B2_PIPE_TRACE=1) if last else contextlib.nullcontext():
                            _call(handle, x, e, 0.0, N.B2_DEVICE_RESIDENT, dev=dev)
        err = capfd.readouterr().err
    finally:
        handle.close()
        torch.cuda.synchronize()
    lines = [ln for ln in err.splitlines() if ln.startswith("[b2 pipe] V=")]
    assert len(lines) == 1, err
    chained = n_calls > 1
    premise = " n_sub=2 vad_sms=8 chained=%d prev_busy=%d;" % (chained, chained)
    assert premise in lines[0], (premise, lines[0])
    _check(cap, want, packed=True, where=("chain", n_calls), tail=n_calls == 1)


# ----------------------------------------------------------------------------------- rates, labels

@pytest.mark.parametrize("cfg", ["16k", "8k", "16k-group", "48k", "44.1k", "22.05k", "11.025k", "16k-unaligned"])
def test_rates_and_layouts(handle, cfg):
    """The lane kernel at 16 and 8 kHz (packed), the lane-group kernel (B2_VAD_LAYOUT=group, other rates, and a
    video that starts off the 8-sample grid) with floats."""
    fr = {"16k": 16000, "8k": 8000, "16k-group": 16000, "48k": 48000, "44.1k": 44100, "22.05k": 22050,
          "11.025k": 11025, "16k-unaligned": 16000}[cfg]
    fpw = int(fr / 100 + 0.5)
    vids = _win_videos(fpw, LENGTHS[:6] + [(50, 3)])
    if cfg == "16k-unaligned":
        vids.insert(1, dict(kind="audio", n=1605, tracks=1))   # every later pcm_off is 5 mod 8
    c = _corpus(vids, fr, 200 + fr % 97)
    knobs = dict(B2_ALIGN_PATH="runs")
    if cfg == "16k-group":
        knobs["B2_VAD_LAYOUT"] = "group"
    for label in (0.0, 0.3):
        want = _oracle(c, "energy", label)
        with _env(**knobs):
            cap = _captured(handle, c, want, lambda keep: _call(handle, c, "tracks", label))
        _check(cap, want, packed=cfg in ("16k", "8k"), where=(cfg, label))


@pytest.mark.parametrize("layout", ["lane", "group"])
@pytest.mark.parametrize("label", LABELS)
def test_labels(handle, energy_corpus, label, layout):
    """At label 1.0 every window is 1.0, the partial ones too (all bits set up to R); at -0.5 and 0.3 the
    non-speech frames hold the label."""
    knobs = dict(B2_ALIGN_PATH="runs")
    if layout == "group":
        knobs["B2_VAD_LAYOUT"] = "group"
    want = _oracle(energy_corpus, "energy", label)
    with _env(**knobs):
        cap = _captured(handle, energy_corpus, want, lambda keep: _call(handle, energy_corpus, "tracks", label))
    _check(cap, want, packed=layout == "lane", where=(label, layout))
    if label == 1.0:
        assert all((w == 1.0).all() for w in want)


@pytest.mark.parametrize("label", [0.0, 0.3])
def test_auditok_labels(handle, energy_corpus, label):
    want = _oracle(energy_corpus, "auditok", label, chunk=160 * 1000)
    cap = _captured(handle, energy_corpus, want,
                    lambda keep: _call(handle, energy_corpus, "auditok", label, chunk=160 * 1000))
    _check(cap, want, packed=False, where=label)


def test_long_reference_tail(handle):
    """A 20-minute video whose tracks cover its first minute: the 118 800 frames past the subtitles and the window
    are checked too, at 16 kHz packed and floats, and under auditok."""
    c = _corpus([dict(kind="audio", n=120000 * 160 + 40, tracks=2), dict(kind="audio", n=31 * 160, tracks=1)],
                16000, 1200)
    for knobs, packed in ((dict(B2_ALIGN_PATH="runs"), True), (dict(B2_REF_PACKED=0), False)):
        want = _oracle(c, "energy", 0.0)
        with _env(**knobs):
            cap = _captured(handle, c, want, lambda keep: _call(handle, c, "tracks", 0.0))
        _check(cap, want, packed=packed, where=knobs)
    want = _oracle(c, "auditok", 0.0)
    cap = _captured(handle, c, want, lambda keep: _call(handle, c, "auditok", 0.0))
    _check(cap, want, packed=False, where="auditok")


# ----------------------------------------------------------------------------------- auditok chunking

@pytest.mark.parametrize("fr,chunk", [(16000, 0), (16000, None), (16000, 160 * 3200), (16000, 160 * 3201),
                                      (16000, 160 * 3231), (22050, None), (8000, 80 * 1057)])
def test_auditok_chunking(handle, fr, chunk):
    """chunk_samples of 0 (one call per video), of the default, and of 3200 / 3201 / 3231 blocks (0, 1, 31 mod
    32); at 22.05 kHz the default chunk is 10 022.7 blocks.  Subtitle videos sit between the audio videos."""
    block = fr // 100
    vids = [dict(kind="audio", n=n, tracks=1) for n in (block * 12000 + 77, block * 3231 * 2 + 5, 0, block * 40)]
    st, en = cases.synthetic_cues(fr, 50.0)
    vids.insert(1, dict(kind="subs", starts=st, ends=en, keep=np.ones(len(st)), tracks=1))
    vids.insert(4, dict(kind="subs", starts=st[:3], ends=en[:3], keep=np.ones(3), tracks=1))
    vids.append(dict(kind="audio", n=block * 25000 + 11, tracks=1))
    c = _corpus(vids, fr, 300 + fr % 89)
    want = _oracle(c, "auditok", 0.0, chunk=chunk)
    cap = _captured(handle, c, want, lambda keep: _call(handle, c, "subs", 0.0, detector="auditok", chunk=chunk))
    _check(cap, want, packed=False, where=(fr, chunk))


# ----------------------------------------------------------------------------------- text and PGS edges

def _pgs_rows():
    with open(os.path.join(ROOT, "tests", "golden", "pgs.json")) as fh:
        g = json.load(fh)
    return [r for r in g["pgs_signals"] if not r["error"] and r["start_seconds"] == 0]


@pytest.mark.parametrize("ss", [0.0, 3.0, -2.0, 0.005, 12.345])
def test_text_and_pgs_edges(handle, ss):
    """Text references from the rasteriser's edge catalogue at ratio 1.0 (half-microsecond ties, half frames, every
    slice case: cues before start_seconds wrap to the end) and the PGS rounding-edge interval lists, between audio
    videos, at labels 0 and 0.5."""
    rng = np.random.RandomState(int(ss * 1000) % 9973 + 5)
    vids = _win_videos(160, [(2000, 0), (33, 40)])
    t = rc.half_us_times(rng, 1.0, 1, 700, 40000)[:300]
    other = t + np.where(t >= 0, 1.0, -1.0) * rng.uniform(0, 5, len(t))
    texts = [(t, other), (other, t)]
    texts.append(rc.half_frame_cues(rng, 1.0, ss, 300, 0, 60000))
    for n in (1, 2, 31, 32, 33, 1000):
        texts.append(rc.slice_case_cues(rng, 1.0, ss, n, 60))
    for a, b in texts:
        vids.append(dict(kind="subs", starts=a, ends=b, keep=rng.rand(len(a)) < 0.85, tracks=1))
    for row in _pgs_rows():
        vids.append(dict(kind="pgs", starts=row["starts"], ends=row["ends"], tracks=1))
    vids += _win_videos(160, [(32 * 10 + 1, 8)])
    c = _corpus(vids, 16000, 400)
    for label in (0.0, 0.5):
        want = _oracle(c, "energy", label, ss=ss)
        cap = _captured(handle, c, want, lambda keep: _call(handle, c, "pgs", label, ss=ss))
        _check(cap, want, packed=False, where=(ss, label))


# ----------------------------------------------------------------------------------- tokenizer edges

TOKS = [(1.0, 1, 0.0), (1.0, 2, 0.5), (3.0, 32, 0.0), (2.0, 31, 30.0), (1.0, 33, 31.5), (1.0, 64, 0.0), DEFAULT_TOK]


def _flag_pcm(flags, fpw):
    """A valid block is +-400 alternating (E = 160 000 fpw), an invalid one silent."""
    alt = np.where(np.arange(len(flags) * fpw) % 2 == 0, 400, -400).astype(np.int16)
    return np.where(np.repeat(np.asarray(flags, bool), fpw), alt, np.int16(0)).astype(np.int16)


def _edge_flags(rng, L, ml, mcs):
    """L flags of valid runs and gaps whose lengths sit at max_length, at 32-frame steps and at the silence rule's
    edge, starting near frames 31 / 32 / 33 of a step."""
    runs = sorted({1, 2, 31, 32, 33, 63, 64, 65, max(1, ml - 1), ml, ml + 1, 2 * ml - 1, 2 * ml, 2 * ml + 1})
    gaps = sorted({1, 2, 31, 32, 33, max(1, int(mcs)), int(mcs) + 1, int(mcs) + 2})
    out = [0] * int(rng.choice([0, 1, 30, 31, 32, 33, 63, 64, 65]))
    while len(out) < L:
        out += [1] * int(rng.choice(runs))
        out += [0] * int(rng.choice(gaps))
    return out[:L]


@pytest.fixture(scope="module")
def tok_inputs():
    fpw = 160
    all12 = ((np.arange(4096)[:, None] >> np.arange(12)) & 1).astype(bool)   # every flag string of length 12
    lc = 160   # long chunks: 160 frames (0 mod 32); the videos' last chunks are 1, 31, 33, 97 and 128 frames
    longs = [dict(tail=t, n_chunks=k) for t, k in ((1, 3), (31, 2), (33, 4), (97, 1), (128, 5), (0, 6))]
    return dict(fpw=fpw, all12=all12, lc=lc, longs=longs)


def _tok_case(ti, tok):
    """(pcm videos, chunk_samples, per-video oracle flags per chunk) of the two shapes."""
    fpw = ti["fpw"]
    cases_ = [([ti["all12"].reshape(-1)], 12 * fpw, 12)]
    rng = np.random.RandomState(int(tok[1]) * 7 + int(tok[2] * 2))
    vids = []
    for d in ti["longs"]:
        L = ti["lc"] * d["n_chunks"] + d["tail"]
        vids.append(np.array(_edge_flags(rng, L, tok[1], tok[2]), bool))
    cases_.append((vids, ti["lc"] * fpw, ti["lc"]))
    return cases_


@pytest.mark.parametrize("tok", TOKS, ids=["1-1-0", "1-2-0.5", "3-32-0", "2-31-30", "1-33-31.5", "1-64-0", "default"])
def test_tokenizer_edges(handle, tok_inputs, tok):
    """Both tokenizer instantiations against au.tokenize: every flag string of length 12 as its own chunk, and long
    chunks whose runs sit at step and max_length boundaries."""
    fpw = tok_inputs["fpw"]
    for flag_videos, chunk, step in _tok_case(tok_inputs, tok):
        want64 = []
        for fl in flag_videos:
            parts = [_tok_signal(fl[i:i + step], tok, 0.0) for i in range(0, len(fl), step)]
            want64.append(np.concatenate(parts) if parts else np.zeros(0))
        pcms = [_flag_pcm(fl, fpw) for fl in flag_videos]
        pcm_off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
        pcm = np.concatenate(pcms)
        # the float64 instantiation (b2_vad_auditok)
        out, out_off = handle.vad_auditok(pcm, pcm_off, 16000, 100, 0.0, min_length=tok[0], max_length=tok[1],
                                          max_continuous_silence=tok[2], chunk_samples=chunk)
        for v, w in enumerate(want64):
            got = out[out_off[v]:out_off[v + 1]]
            bad = np.flatnonzero(got != w)
            assert len(got) == len(w) and len(bad) == 0, (tok, chunk, v, bad[:8].tolist())
        # the float32 in-place instantiation (b2_sync_tracks_auditok's reference)
        vids = [dict(kind="audio", n=len(p), tracks=1) for p in pcms]
        c = dict(videos=vids, fr=16000, pcms=pcms, pcm=pcm, pcm_off=pcm_off, tv=np.arange(len(pcms), dtype=np.int32),
                 cs=np.repeat([0.5], len(pcms)), ce=np.repeat([1.5], len(pcms)),
                 cue_off=np.arange(len(pcms) + 1, dtype=np.int64))
        want = [w.astype(np.float32) for w in want64]
        cap = _captured(handle, c, want, lambda keep: _call(handle, c, "auditok", 0.0, chunk=chunk, tok=tok))
        _check(cap, want, packed=False, where=(tok, chunk))


# ----------------------------------------------------------------------------------- capture on / off

def _host_outputs(r):
    return [None if x is None else np.array(x, copy=True) for x in r]


@pytest.mark.parametrize("entry", ENTRIES)
def test_capture_changes_nothing(handle, energy_corpus, mixed_corpus, entry):
    """Outputs bit-identical and launch counts equal with and without the capture, with two sub-batches; an
    undersized capture (frames or videos) fails the call with B2_ERR_BAD_ARG and copies nothing."""
    from ffsubsync_b200 import _native as N
    c = mixed_corpus[entry] if entry in ("subs", "pgs") else energy_corpus
    detector = "auditok" if entry == "auditok" else "energy"
    want = _oracle(c, detector, 0.0)
    with _env(B2_SUBBATCHES=2):
        n0 = handle.launch_count
        off = _host_outputs(_call(handle, c, entry, 0.0, detector=detector))
        n_off = handle.launch_count - n0
        _poison(handle, _capacity(want))
        with handle.capture_reference(_capacity(want), len(want)) as cap:
            n0 = handle.launch_count
            on = _host_outputs(_call(handle, c, entry, 0.0, detector=detector))
            n_on = handle.launch_count - n0
    assert n_on == n_off, (entry, n_on, n_off)
    for x, y in zip(on, off):
        if x is not None or y is not None:
            assert np.array_equal(x, y, equal_nan=True) and x.dtype == y.dtype, entry
    _check(cap, want, where=entry)
    total = int(sum(len(w) for w in want))
    for capacity, max_videos in ((total - 1, len(want)), (total, len(want) - 1)):
        with pytest.raises(N.NativeError) as e:
            with handle.capture_reference(capacity, max_videos) as bad:
                _call(handle, c, entry, 0.0, detector=detector)
        assert e.value.status == -1, (entry, capacity, max_videos)
        assert np.isnan(bad["ref"]).all() and (bad["ref_off"] == -1).all(), (entry, capacity, max_videos)
