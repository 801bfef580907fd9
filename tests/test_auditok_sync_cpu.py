"""CPU suite for the auditok detector inside the batched sync (b2_sync_tracks_auditok).

Checks what can be checked without a GPU: the symbol and its ctypes signature against the header, the
front end's argument checks, the chunk table / reference-length arithmetic of the C planner (against the lengths
the oracle's chunk loop produces), and the two-level property of the auditok signal at
label 0 that lets the run path and the golden-section search read it."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import auditok_oracle as au
from sync_plan import plan


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


# ---------------------------------------------------------------- ABI

_CTYPE = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "double": ctypes.c_double}


def _prototype(header: str, name: str):
    m = re.search(r"\bint\s+%s\s*\((.*?)\);" % name, header, re.S)
    assert m, name
    body = re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S)
    return [" ".join(a.split()) for a in body.split(",")]


def test_sync_tracks_auditok_is_exported_with_the_header_signature(built):
    from ffsubsync_b200 import _native
    assert "b2_sync_tracks_auditok" in _native.EXPORTS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), "b2_sync_tracks_auditok")
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    args = _prototype(header, "b2_sync_tracks_auditok")
    want = []
    for a in args:
        t = a.rsplit(" ", 1)[0]
        want.append(ctypes.c_void_p if ("*" in a or t == "b2_handle") else _CTYPE[t])
    got = _native.load().b2_sync_tracks_auditok.argtypes
    assert len(got) == len(want) == 30
    for i, (g, w) in enumerate(zip(got, want)):
        assert g is w, (i, args[i], g, w)
    # a handle-less call is refused before anything is read
    assert _native.load().b2_sync_tracks_auditok(None, None, None, 0, None, 0, 16000, 100, 0.0, 50.0, 20.0, 500, 25.0,
                                                 0, None, None, None, None, None, 1, 0.0, 0, None, None, None, None,
                                                 None, None, None, 0) == -1


# ---------------------------------------------------------------- front end

def _make(ratios, **kw):
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    try:
        return BatchSynchronizer(ratios, **kw)
    except _native.NativeError:   # no GPU here: the arguments were accepted before the handle was made
        return None


def test_batch_synchronizer_vad_argument():
    from ffsubsync_b200.batch import BatchSynchronizer
    for bad in ("webrtc", "silero", "AUDITOK", "", None):
        with pytest.raises(ValueError):
            BatchSynchronizer([1.0], vad=bad)
    # the energy detector's knobs are not silently ignored with auditok
    for kw in (dict(energy_threshold=1), dict(z_lo=0), dict(z_hi=40)):
        with pytest.raises(ValueError):
            BatchSynchronizer([1.0], vad="auditok", **kw)
    for vad in ("energy_zcr", "auditok"):
        _make([1.0], vad=vad)
        _make([1.0, None], vad=vad)
    _make([1.0], vad="energy_zcr", energy_threshold=1, z_lo=0, z_hi=40)


def test_chunk_samples_is_the_chunk_loop_read_size():
    from ffsubsync_b200.constants import detector_chunk_bytes
    from ffsubsync_b200.speech_transformers import VideoSpeechTransformer
    for fr in (8000, 16000, 22050, 44100, 48000):
        assert detector_chunk_bytes(fr, 100) == (2 * fr // 100) * 10000
        assert detector_chunk_bytes(fr, 100) // 2 == (2 * fr // 100) * 5000
        assert ((2 * fr // 100) * 5000) % 8 == 0   # chunk starts keep 16-byte alignment
    assert VideoSpeechTransformer.CHUNK_WINDOWS == 10000


# ---------------------------------------------------------------- chunk table

def _chunk_table(pcm_off, fr, chunk_samples):
    """The planner's table (csrc/sync_plan.h, build_chunk_table, as b2_sync_tracks_auditok plans it with one track
    per video): returns (chunk pcm offsets, chunk block offsets, first chunk of each video, ref_off)."""
    V = len(pcm_off) - 1
    p = plan(who="sync_tracks_auditok", detector=1, frame_rate=fr, sample_rate=100, chunk_samples=chunk_samples,
             pcm_off=pcm_off, cue_start=[], cue_end=[], cue_off=[0] * (V + 1), ratios=[1.0])
    assert p["status"] == 0, p["err"]
    return p["ch_pcm"].tolist(), p["ch_out"].tolist(), p["ch_first"].tolist(), p["ref_off"].tolist()


@pytest.mark.parametrize("fr", [8000, 16000, 22050, 44100, 48000])
def test_reference_length_is_the_oracle_chunk_loop_length(fr):
    sr = 100
    fpw = fr // sr
    chunk = (2 * fr // sr) * 5000
    lengths = [0, 1, fpw - 1, fpw, chunk - 1, chunk, chunk + 1, 2 * chunk, 3 * chunk + 7, 2 * chunk - fpw + 1]
    pcm_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    ch_pcm, ch_out, first, ref_off = _chunk_table(list(pcm_off), fr, chunk)
    silent = np.zeros(max(lengths), np.int16)
    for v, n in enumerate(lengths):
        # the reference's chunk loop: one detector call per chunk, outputs concatenated
        want = sum(len(au.auditok_detect_fast(silent[s: min(n, s + chunk)].tobytes(), sr, fr, 0.0))
                   for s in range(0, n, chunk))
        assert ref_off[v + 1] - ref_off[v] == want, (fr, n)
        # the closed form the Python layer uses for vad_auditok's out_off
        assert want == n // chunk * ((chunk + fpw - 1) // fpw) + (n % chunk + fpw - 1) // fpw
        # chunks tile the video, start on multiples of chunk_samples, at most chunk_samples long
        c0, c1 = first[v], first[v + 1]
        assert ch_pcm[c0] == pcm_off[v] and ch_pcm[c1] == pcm_off[v + 1]
        assert all(0 < ch_pcm[c + 1] - ch_pcm[c] <= chunk for c in range(c0, c1))
        assert all((ch_pcm[c] - pcm_off[v]) % chunk == 0 for c in range(c0, c1))
    # 22.05 kHz: a chunk is not a whole number of blocks, so ceil(n/fpw) is too short
    if fr == 22050:
        assert chunk % fpw != 0
        assert ref_off[9] - ref_off[8] == (lengths[8] + fpw - 1) // fpw + 1


def test_chunk_samples_zero_is_one_call_per_video():
    pcm_off = [0, 0, 1, 161, 16000 * 300 + 5]
    _, _, first, ref_off = _chunk_table(pcm_off, 16000, 0)
    assert np.diff(first).tolist() == [0, 1, 1, 1]
    assert np.diff(ref_off).tolist() == [0, 1, 1, (16000 * 300 + 5 - 161 + 159) // 160]


# ---------------------------------------------------------------- two levels

def _flags_pcm(valid, fpw=160, seed=0):
    """PCM whose blocks pass the 50 dB test exactly where valid is set (a final partial block too)."""
    rng = np.random.RandomState(seed)
    out = np.where(np.repeat(valid, fpw), rng.choice([-2000, 2000], len(valid) * fpw),
                   rng.randint(-3, 4, len(valid) * fpw)).astype(np.int16)
    return out


def _chunked(pcm, fr, label, chunk):
    return np.concatenate([au.auditok_detect_fast(pcm[s: s + chunk].tobytes(), 100, fr, label)
                           for s in range(0, len(pcm), chunk)])


def _two_level_inputs():
    chunk_w = 700   # blocks per chunk in these inputs
    cases = []
    v = np.zeros(3000, bool)
    v[100:1300] = True            # 12 s of speech: truncated 5 s tokens, contiguous follow-ups
    v[1350:1372] = True           # a short token
    v[1390:1394] = True           # shorter than min_length
    v[chunk_w - 30: chunk_w + 40] = True   # a token cut by a chunk end
    v[2 * chunk_w - 510: 2 * chunk_w + 3] = True   # a 5 s token ending right at a chunk boundary
    cases.append(v)
    rng = np.random.RandomState(4)
    cases.append(rng.rand(3000) < 0.7)         # dense: many tokens ending in trailing silence
    w = np.zeros(2600, bool)
    for k in range(0, 1000, 80):
        w[k: k + 30] = True                    # separate tokens
    w[1000:1501] = True                        # 501 blocks: one truncated token plus a 1-block follow-up
    cases.append(w)
    return chunk_w, cases


def test_auditok_signal_is_two_level_only_at_label_zero():
    chunk_w, cases = _two_level_inputs()
    fr, fpw = 16000, 160
    saw_truncation = False
    for i, valid in enumerate(cases):
        pcm = _flags_pcm(valid, fpw, seed=i)[:-37]   # a short last block too
        chunk = chunk_w * fpw
        sig0 = _chunked(pcm, fr, 0.0, chunk)
        assert set(np.unique(sig0).tolist()) <= {0.0, 1.0}, i
        # truncated tokens were exercised: a 5 s run of ones is followed by a contiguous token
        toks = au.tokenize(list(valid[:chunk_w]), 20, 500, 25)
        saw_truncation |= any(b[0] == a[1] + 1 for a, b in zip(toks, toks[1:]))
        s03 = _chunked(pcm, fr, 0.3, chunk)
        s1 = _chunked(pcm, fr, 1.0, chunk)
        if i != 1:   # (case 1 is one chain of contiguous tokens: its cumsum never falls below 1 before the end)
            assert len(set(np.unique(s03).tolist()) - {0.0, 1.0}) > 0, i
            assert not np.array_equal(s1, sig0)
        # label 1: ends add 0, so every frame after the first token start is 1 within its chunk
        for c0 in range(0, len(s1), chunk_w):
            part = s1[c0: c0 + chunk_w]
            nz = np.nonzero(part)[0]
            if len(nz):
                assert np.all(part[nz[0]:] == 1.0)
    assert saw_truncation
    # the levels a non-zero label produces: 0.3 accumulates 0.3, 0.6, 0.9 over consecutive tokens
    s = au.auditok_detect_fast(_flags_pcm(cases[2][:300], fpw, seed=0).tobytes(), 100, fr, 0.3)
    vals = set(np.round(np.unique(s), 6).tolist())
    assert {0.3, 0.6, 0.9} <= vals


def test_chunk_restart_changes_the_signal():
    """A token that crosses a chunk boundary: the chunked signal differs from one detector call over the whole
    video (the tokenizer restarts in every call)."""
    fr, fpw, chunk_w = 16000, 160, 700
    valid = np.zeros(2000, bool)
    valid[chunk_w - 12: chunk_w + 13] = True   # 25 blocks across the boundary
    pcm = _flags_pcm(valid, fpw, seed=9)
    whole = au.auditok_detect_fast(pcm.tobytes(), 100, fr, 0.0)
    chunked = _chunked(pcm, fr, 0.0, chunk_w * fpw)
    assert len(whole) == len(chunked) and not np.array_equal(whole, chunked)
    # the 12 blocks the first call ends on are too short a token; the second call's 13 blocks plus their
    # trailing silence are long enough
    assert whole[chunk_w - 12] == 1.0 and chunked[chunk_w - 12] == 0.0 and chunked[chunk_w] == 1.0
