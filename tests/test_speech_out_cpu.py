"""CPU suite of the speech output of the batched sync calls (b2_speech_output, ``--serialize-speech``).

Checks what can be checked without a GPU: speech_out_kernel's loop nest run thread by thread on the CPU against a
numpy unpack (tests/host_emul/speech_out_emul), the symbols and their ctypes signatures against the header, the
Python layer's reference lengths against the planner's ref_off for every reference kind (sync_plan.h through the
emulator's plan mode, with and without tracks), and save_serialized_speech's round trip through the loaders."""
import os
import re
import struct
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import ROOT

EMUL = os.path.join(ROOT, "tests", "host_emul", "speech_out_emul")


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


# ---------------------------------------------------------------- the kernel, thread by thread

def _words(x):
    """ceil(R/32) uint32 words of the bits (x == 1.0f), bit i of word k = frame 32k + i, zero past R."""
    bits = np.zeros(-(-len(x) // 32) * 32, np.uint64)
    bits[: len(x)] = x == np.float32(1.0)
    return (bits.reshape(-1, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)


def _buffer(videos, rng):
    """A reference buffer of videos (R, packed, low) at ragged starts: returns (uint32 words, src per video, signals)."""
    words, src, sigs = [rng.randint(0, 2 ** 32, rng.randint(0, 40), dtype=np.uint64).astype(np.uint32)], [], []
    for R, packed, low in videos:
        x = np.where(rng.rand(R) < 0.5, np.float32(1.0), np.float32(low) if packed else
                     rng.choice([np.float32(low), np.float32(0.25), np.float32(-3.5)], R)).astype(np.float32)
        at = sum(len(w) for w in words)
        src.append(at)
        words.append(_words(x) if packed else x.view(np.uint32))
        sigs.append(x)
        words.append(rng.randint(0, 2 ** 32, rng.randint(0, 37), dtype=np.uint64).astype(np.uint32))   # a gap
    return np.concatenate(words), src, sigs


def _emul_kernel(words, src, lows, packed, lens):
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    n = len(lens)
    with tempfile.TemporaryDirectory() as d:
        a, b = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(a, "wb") as f:
            f.write(struct.pack("<iq", n, len(words)))
            f.write(off.tobytes())
            for s, lo, p in zip(src, lows, packed):
                f.write(struct.pack("<qfi", int(s), float(lo), int(p)))
            f.write(np.ascontiguousarray(words, np.uint32).tobytes())
        subprocess.check_call([EMUL, "kernel", a, b])
        return np.fromfile(b, np.float64), off


# R mod 32 in {0, 1, 31}, R < 32, empty videos, and videos longer than one tile
LENGTHS = [32 * 40, 32 * 40 + 1, 32 * 40 + 31, 20, 0, 1, 33, 4096 * 3 + 17, 0, 64 + 5, 4095, 4097]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_emulated_kernel(built, seed):
    rng = np.random.RandomState(seed)
    vids = [(R, bool(rng.rand() < 0.5), float(np.float32(rng.choice([0.0, 0.3, -0.5, 1.0])))) for R in LENGTHS]
    words, src, sigs = _buffer(vids, rng)
    for pick in (np.arange(len(vids)), np.array([1, 4, 7, 8, 11]), np.array([4]), np.array([7])):
        got, off = _emul_kernel(words, [src[i] for i in pick], [vids[i][2] for i in pick], [vids[i][1] for i in pick],
                                [vids[i][0] for i in pick])
        want = np.concatenate([sigs[i].astype(np.float64) for i in pick] + [np.zeros(0)])
        assert len(got) == off[-1] == len(want)
        assert np.array_equal(got, want), (seed, pick.tolist())


def test_emulated_kernel_packed_low_level(built):
    """A clear bit reads as the video's low level, a set bit as 1.0, side by side with float videos."""
    x = np.array([1.0, 0.0, 1.0] * 23, np.float32)
    words = np.concatenate([_words(x), x.view(np.uint32), _words(x)])
    nw = len(_words(x))
    got, _ = _emul_kernel(words, [0, nw, nw + len(x)], [-0.5, 7.0, 0.0], [1, 0, 1], [len(x)] * 3)
    assert np.array_equal(got[: len(x)], np.where(x == 1.0, 1.0, np.float64(np.float32(-0.5))))
    assert np.array_equal(got[len(x): 2 * len(x)], x.astype(np.float64))
    assert np.array_equal(got[2 * len(x):], x.astype(np.float64))


# ---------------------------------------------------------------- ABI

def test_export_and_header_signature(built):
    from ffsubsync_b200 import _native
    hdr = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    lib = _native.load()
    for name, n in (("b2_speech_output", 7), ("b2_segment_length", 2)):
        m = re.search(r"\b%s\((.*?)\);" % name, hdr, re.S)
        assert m and name in _native.EXPORTS
        params = [p for p in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",") if p.strip()]
        assert len(getattr(lib, name).argtypes) == len(params) == n
    # a handle-less call is refused before anything is read (bad pointers everywhere else)
    assert lib.b2_speech_output(None, 8, 10, 16, 3, 24, 1) == -1
    assert lib.b2_segment_length(100.0, 100) == 10002 and lib.b2_segment_length(float("nan"), 100) == -1


# ---------------------------------------------------------------- lengths against the planner

def _plan(**req):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            for k, v in req.items():
                vals = [v] if np.isscalar(v) or isinstance(v, str) else list(np.asarray(v).ravel())
                f.write("%s %d %s\n" % (k, len(vals), " ".join(
                    x if isinstance(x, str) else repr(float(x)) if isinstance(x, (float, np.floating)) else str(int(x))
                    for x in vals)))
        subprocess.check_call([EMUL, "plan", src, dst])
        out = {}
        for line in open(dst).read().splitlines():
            k, _, rest = line.partition(" ")
            out[k] = int(rest) if k == "status" else rest if k == "err" else np.array(rest.split(), np.int64)
        return out


FR = 16000


def _mixed(tracks=True):
    """Six videos: energy audio, text stream, PGS list, signal, segments, audio with a partial window."""
    from ffsubsync_b200.batch import segment_table
    pcm_off = np.array([0, 3000 * 160 + 7, 3000 * 160 + 7, 3000 * 160 + 7, 3000 * 160 + 7, 3000 * 160 + 7 + 200 * FR,
                        3000 * 160 + 7 + 200 * FR + 12345], np.int64)
    tab = segment_table(pcm_off, FR, videos=[4], segment_count=3, segment_duration=20)
    st, en = np.array([1.0, 5.5, 60.25]), np.array([2.0, 7.125, 61.5])
    return dict(pcm_off=pcm_off, ref_is_subs=[0, 1, 0, 0, 0, 0], ref_cue_start=st, ref_cue_end=en,
                ref_cue_off=[0, 0, 3, 3, 3, 3, 3], ref_is_pgs=[0, 0, 1, 0, 0, 0], pgs_start=[0.5, 10.0],
                pgs_end=[1.25, 12.345], pgs_off=[0, 0, 0, 2, 2, 2, 2], ref_is_sig=[0, 0, 0, 1, 0, 0],
                sig_off=[0, 0, 0, 0, 777, 777, 777], **{k: v for k, v in tab.items()},
                track_video=list(range(6)) if tracks else [], cue_start=[1.0] * (6 if tracks else 0),
                cue_end=[2.0] * (6 if tracks else 0), cue_off=list(range(7)) if tracks else [0], ratios=[1.0])


def _python_lengths(req, vad):
    """BatchSynchronizer._reference_lengths over the request's references."""
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200 import _native

    class _Sync(BatchSynchronizer):   # the length rules need the library, not a device
        def __init__(self):
            self.handle = _native.Handle.__new__(_native.Handle)
            self.handle.lib = _native.load()
            self.vad, self.detector, self.subs_then = vad, vad, False
            self.frame_rate, self.sample_rate = FR, 100
            from ffsubsync_b200.constants import detector_chunk_bytes
            self.chunk_samples = detector_chunk_bytes(FR, 100) // 2
            self.start_seconds = 0.0

    s = _Sync()
    V = len(req["pcm_off"]) - 1
    refs = (np.array(req["ref_is_subs"], np.uint8), np.asarray(req["ref_cue_start"]), np.asarray(req["ref_cue_end"]),
            None, np.asarray(req["ref_cue_off"], np.int64))
    pgs = (np.array(req["ref_is_pgs"], np.uint8), np.asarray(req["pgs_start"]), np.asarray(req["pgs_end"]),
           np.asarray(req["pgs_off"], np.int64))
    sig = (np.array(req["ref_is_sig"], np.uint8), np.zeros(777), np.asarray(req["sig_off"], np.int64))
    seg = (req["seg_video"], req["seg_total"], req["seg_off"], req["seg_start"], req["seg_lo"], req["seg_hi"])
    assert V == 6
    return s._reference_lengths(req["pcm_off"], refs, pgs, sig, seg)


@pytest.mark.parametrize("tracks", [True, False])
@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
def test_lengths_equal_the_planner(built, det, tracks):
    req = _mixed(tracks)
    p = _plan(detector=1 if det == "auditok" else 0, chunk_samples=(2 * FR // 100) * 5000 if det == "auditok" else 0,
              speech_out=1, **req)
    assert p["status"] == 0, p["err"]
    assert np.array_equal(np.diff(p["ref_off"]), _python_lengths(req, det)), (p["ref_off"], det)
    if not tracks:   # the serialize-only plan: one sub-batch of floats, no tracks
        assert p["cut"].tolist() == [0, 6] and p["ref_packed"].tolist() == [0] and not p["trk_off"].any()


def test_no_tables_without_the_output(built):
    p = _plan(detector=0, **_mixed(False))
    assert p["status"] == 0 and len(p["ref_off"]) == 0 and len(p["cut"]) == 0


# ---------------------------------------------------------------- saving

def test_save_round_trip(built):
    from ffsubsync_b200.batch import load_serialized_speech, save_serialized_speech
    from ffsubsync_b200.speech_transformers import load_stored_speech
    rng = np.random.RandomState(3)
    x = np.concatenate([np.where(rng.rand(1000) < 0.5, 1.0, 0.3), np.zeros(0), np.where(rng.rand(33) < 0.5, 1.0, -0.5)])
    off = np.array([0, 1000, 1000, 1033], np.int64)
    with tempfile.TemporaryDirectory() as d:
        paths = [os.path.join(d, "v%d.npz" % i) for i in range(3)]
        save_serialized_speech(paths, x, off)
        for i, p in enumerate(paths):
            assert np.array_equal(load_stored_speech(p), x[off[i]: off[i + 1]])
            with np.load(p) as z:
                assert list(z.keys()) == ["speech"] and z["speech"].dtype == np.float64
        y, y_off = load_serialized_speech(paths, stored=True)
        assert np.array_equal(y, x) and np.array_equal(y_off, off)
        # a segment video without a frame > 0 is refused before anything is written; a non-segment one is not
        paths2 = [os.path.join(d, "w%d.npz" % i) for i in range(3)]
        z = np.concatenate([x[:1000], np.full(33, -0.5)])
        with pytest.raises(ValueError, match="video 7: Unable to detect speech"):
            save_serialized_speech(paths2, z, off, speech_video=[3, 5, 7], seg_video=[3, 7])
        assert not any(os.path.exists(p) for p in paths2)
        save_serialized_speech(paths2, z, off, speech_video=[3, 5, 7], seg_video=[3])
        assert np.array_equal(load_stored_speech(paths2[2]), z[1000:])
        # the segment check needs the listed videos, one per path
        with pytest.raises(ValueError, match="needs speech_video"):
            save_serialized_speech(paths2, z, off, seg_video=[3])
        with pytest.raises(ValueError, match="2 entries for 3 paths"):
            save_serialized_speech(paths2, z, off, speech_video=[3, 5], seg_video=[3])
        with pytest.raises(ValueError, match="paths"):
            save_serialized_speech(paths[:2], x, off)
