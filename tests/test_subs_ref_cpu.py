"""CPU suite for embedded subtitle streams as references in the batched sync (b2_sync_tracks_subs, the
``subs_then_`` detectors).

Checks what can be checked without a GPU: the symbol and its ctypes signature against the header, the front
end's stream selection and keep flags against fixtures recorded from the reference's
VideoSpeechTransformer(vad="subs_then_webrtc").fit (tests/golden/make_golden_subs_ref.py), the oracle
rasteriser reproducing the recorded reference signals frame for frame, the oracle aligner reproducing the
recorded MaxScoreAligner result over the ratio grid, and the front end's argument checks."""
import ctypes
import json
import os
import re
import sys

import numpy as np
import pytest

from conftest import ROOT
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro

GOLDEN = os.path.join(ROOT, "tests", "golden", "subs_ref.json")


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


def _streams(row):
    """The fixture row's streams as the flat arrays the front end takes (one video)."""
    st = row["streams"]
    starts = np.array([t for s in st for t in s["starts"]], dtype=np.float64)
    ends = np.array([t for s in st for t in s["ends"]], dtype=np.float64)
    content = [c for s in st for c in s["contents"]]
    off = np.concatenate([[0], np.cumsum([len(s["starts"]) for s in st])]).astype(np.int64)
    return starts, ends, content, off


def _runs(x):
    nz = np.asarray(x) != 0
    d = np.diff(np.concatenate([[0], nz.astype(np.int8), [0]]))
    return list(np.flatnonzero(d == 1)), list(np.flatnonzero(d == -1))


# ---------------------------------------------------------------- ABI

_CTYPE = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "double": ctypes.c_double}


def test_sync_tracks_subs_is_exported_with_the_header_signature(built):
    from ffsubsync_b200 import _native
    assert "b2_sync_tracks_subs" in _native.EXPORTS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), "b2_sync_tracks_subs")
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    m = re.search(r"\bint\s+b2_sync_tracks_subs\s*\((.*?)\);", header, re.S)
    assert m
    args = [" ".join(a.split()) for a in re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")]
    want = [ctypes.c_void_p if ("*" in a or a.startswith("b2_handle")) else _CTYPE[a.rsplit(" ", 1)[0]] for a in args]
    got = _native.load().b2_sync_tracks_subs.argtypes
    assert len(got) == len(want) == 39
    for i, (g, w) in enumerate(zip(got, want)):
        assert g is w, (i, args[i], g, w)
    assert "B2_DETECTOR_ENERGY_ZCR = 0" in header and "B2_DETECTOR_AUDITOK = 1" in header
    # a handle-less call is refused before anything is read
    assert _native.load().b2_sync_tracks_subs(None, None, None, 0, None, 0, 16000, 100, 0, 0.0, 0, -1, -1, 50.0, 20.0,
                                              500, 25.0, 0, None, None, None, None, None, None, None, None, None,
                                              None, 1, 0.0, 0, None, None, None, None, None, None, None, 0) == -1


def test_batch_vads_carry_the_subs_then_detectors():
    from ffsubsync_b200.constants import BATCH_VADS
    assert BATCH_VADS == ("energy_zcr", "auditok", "subs_then_energy_zcr", "subs_then_auditok")


# ---------------------------------------------------------------- fixtures of the reference

def test_fixture_cases_are_present(golden):
    names = {r["name"] for r in golden["subs_ref"]}
    assert {"tie", "start_seconds", "metadata", "one_and_empty", "empty_only", "two_hours"} <= names
    tie = [r for r in golden["subs_ref"] if r["name"] == "tie"][0]
    assert tie["max_time"][0] == tie["max_time"][1] and tie["chosen"] == 0


def test_stream_selection_and_keep_flags_match_the_reference(golden):
    from ffsubsync_b200.batch import select_reference_streams
    from ffsubsync_b200.speech_transformers import _is_metadata
    for row in golden["subs_ref"]:
        starts, ends, content, off = _streams(row)
        S = len(off) - 1
        is_subs, rs, re_, rk, roff = select_reference_streams(1, starts, ends, off, np.zeros(S, np.int64),
                                                              row["start_seconds"], content=content)
        assert list(is_subs) == [1] and len(roff) == 2, row["name"]
        ch = row["streams"][row["chosen"]]
        assert list(rs) == ch["starts"] and list(re_) == ch["ends"], row["name"]
        n = len(ch["starts"])
        assert list(rk) == [int(not _is_metadata(c, i == 0 or i + 1 == n)) for i, c in enumerate(ch["contents"])]
        assert list(rk) == [int(not ro.is_metadata(c, i == 0 or i + 1 == n)) for i, c in enumerate(ch["contents"])]


def test_stream_selection_over_several_videos(golden):
    """The rows as one batch of videos (plus one without streams): each video picks its own stream."""
    from ffsubsync_b200.batch import select_reference_streams
    rows = [r for r in golden["subs_ref"] if r["start_seconds"] == 0]
    parts, vid, content = [], [], []
    V = len(rows) + 1
    for v, row in enumerate(rows):
        for s in row["streams"]:
            parts.append(s)
            vid.append(v + 1)          # video 0 has no stream
            content += s["contents"]
    starts = np.array([t for s in parts for t in s["starts"]])
    ends = np.array([t for s in parts for t in s["ends"]])
    off = np.concatenate([[0], np.cumsum([len(s["starts"]) for s in parts])]).astype(np.int64)
    is_subs, rs, re_, rk, roff = select_reference_streams(V, starts, ends, off, vid, 0.0, content=content)
    assert list(is_subs) == [0] + [1] * len(rows)
    assert roff[1] == 0
    for v, row in enumerate(rows):
        assert list(rs[roff[v + 1]:roff[v + 2]]) == row["streams"][row["chosen"]]["starts"], row["name"]


def test_oracle_raster_reproduces_the_reference_signals(golden):
    for row in golden["subs_ref"]:
        ch = row["streams"][row["chosen"]]
        n = len(ch["starts"])
        keep = [not ro.is_metadata(c, i == 0 or i + 1 == n) for i, c in enumerate(ch["contents"])]
        x, max_time, _, _ = ro.rasterize(ch["starts"], ch["ends"], keep, 100, row["start_seconds"], 1.0)
        assert len(x) == row["length"], row["name"]
        assert max_time == row["max_time"][row["chosen"]], row["name"]
        rs, re_ = _runs(x)
        assert rs == row["run_starts"] and re_ == row["run_stops"], row["name"]
        assert set(np.unique(x)) <= {0.0, 1.0}


def test_oracle_aligner_reproduces_the_reference_grid(golden):
    ms = golden["subs_ref_maxscore"]
    row = [r for r in golden["subs_ref"] if r["name"] == ms["video"]][0]
    ch = row["streams"][row["chosen"]]
    ref, _, _, _ = ro.rasterize(ch["starts"], ch["ends"], None, 100, 0, 1.0)
    import cases
    mos = ms["max_offset_seconds"] * 100
    best = None
    for k, (r, want) in enumerate(zip(cases.ratio_grid(), ms["per_ratio"])):
        sub, _, _, _ = ro.rasterize(ms["in_starts"], ms["in_ends"], None, 100, 0, r)
        score, off = ao.fft_align(ref, sub, mos)
        assert off == want["offset"], k
        assert abs(score - want["score"]) <= 1e-9 * abs(want["score"]), k
        if abs(off) <= mos and (best is None or score > best[0]):
            best = (score, off, k)
    assert best[1:] == (ms["best"]["offset"], ms["best"]["index"])


# ---------------------------------------------------------------- front end

class _FakeHandle:
    device = 0

    def __init__(self):
        self.calls = []

    def sync_tracks_subs(self, *a, **kw):
        self.calls.append((a, kw))
        T = len(a[2])
        return (np.zeros(T), np.zeros(T, np.int32), np.zeros(T, np.int32), None, None)


@pytest.fixture
def fake(monkeypatch):
    from ffsubsync_b200 import _native
    h = _FakeHandle()
    monkeypatch.setattr(_native, "get_handle", lambda device=None: h)
    return h


def test_front_end_argument_checks(fake):
    from ffsubsync_b200.batch import BatchSynchronizer
    for kw in (dict(energy_threshold=1), dict(z_lo=0), dict(z_hi=40)):
        with pytest.raises(ValueError):
            BatchSynchronizer([1.0], vad="subs_then_auditok", **kw)
    BatchSynchronizer([1.0], vad="subs_then_energy_zcr", energy_threshold=1, z_lo=0, z_hi=40)
    pcm, pcm_off = np.zeros(0, np.int16), np.array([0, 0])
    cues = (np.array([1.0]), np.array([2.0]), np.array([0, 1]))
    streams = dict(ref_cue_start=[1.0], ref_cue_end=[3.0], ref_cue_off=[0, 1], ref_stream_video=[0])
    # streams with a detector that does not read them
    with pytest.raises(ValueError):
        BatchSynchronizer([1.0], vad="energy_zcr").sync_host(pcm, pcm_off, *cues, **streams)
    with pytest.raises(TypeError):
        BatchSynchronizer([1.0], vad="subs_then_energy_zcr").sync_host(pcm, pcm_off, *cues, ref_cue_stat=[1.0])
    bs = BatchSynchronizer([1.0], vad="subs_then_energy_zcr")
    with pytest.raises(ValueError):
        bs.sync_host(pcm, pcm_off, *cues, ref_cue_content=["a"], ref_cue_keep=[1], **streams)
    with pytest.raises(ValueError):
        bs.sync_host(pcm, pcm_off, *cues, **dict(streams, ref_stream_video=[1]))   # no video 1
    with pytest.raises(ValueError):
        bs.sync_device_candidate_sharded(None, pcm_off, *cues)
    assert not fake.calls


def test_front_end_hands_the_chosen_streams_to_the_call(fake):
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    bs = BatchSynchronizer([1.0, 1.04], vad="subs_then_auditok", start_seconds=0.0)
    pcm = np.zeros(3200, np.int16)
    pcm_off = np.array([0, 0, 3200, 3200])          # videos 0 and 2 have streams, video 1 audio
    # video 0: two one-cue streams, the second ends later; video 2: the first stream ends later
    ref = dict(ref_cue_start=[1.0, 2.0, 5.0, 0.5], ref_cue_end=[3.0, 4.0, 9.0, 1.5], ref_cue_off=[0, 1, 2, 3, 4],
               ref_stream_video=[0, 0, 2, 2], ref_cue_content=["a", "b", "c", "[music]"])
    bs.sync_host_tracks(pcm, pcm_off, [0, 1, 2], np.array([1.0] * 3), np.array([2.0] * 3), [0, 1, 2, 3], **ref)
    (a, kw), = fake.calls
    is_subs, rs, re_, rk, roff = a[6:11]
    assert list(is_subs) == [1, 0, 1]
    assert list(rs) == [2.0, 5.0] and list(re_) == [4.0, 9.0] and list(rk) == [1, 1]
    assert list(roff) == [0, 1, 1, 2]
    assert kw["detector"] == _native.B2_DETECTOR_AUDITOK and kw["chunk_samples"] == bs.chunk_samples
    # without streams the detector's own call runs (b2_sync_tracks_auditok, not this one)
    fake.calls.clear()
    fake.sync_tracks_auditok = lambda *a, **kw: fake.calls.append(("auditok", kw)) or (None,) * 5
    bs.sync_host_tracks(pcm, pcm_off, [1], np.array([1.0]), np.array([2.0]), [0, 1])
    assert fake.calls[0][0] == "auditok"
