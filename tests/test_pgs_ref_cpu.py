"""CPU suite for PGS (bitmap subtitle) display intervals as references (b2_rasterize_pgs, b2_sync_tracks_pgs,
``--pgs-ref-stream``).

Checks what can be checked without a GPU: the oracle and the host helpers against fixtures recorded from the
reference's PGS path (tests/golden/make_golden_pgs.py), the symbols and their ctypes signatures against the header,
the kernels' interval arithmetic (raster_math.cuh) run on the CPU against the oracle at the rounding edges and at
10^6 seeded random times, the planner's PGS checks and tables, and the front end's argument checks."""
import ctypes
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from oracle import aligner_oracle as ao
from oracle import pgs_oracle as po
from oracle import raster_oracle as ro

GOLDEN = os.path.join(ROOT, "tests", "golden", "pgs.json")
EMUL = os.path.join(ROOT, "tests", "host_emul", "pgs_emul")


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


def _runs(x):
    nz = np.asarray(x) != 0
    d = np.diff(np.concatenate([[0], nz.astype(np.int8), [0]]))
    return [int(v) for v in np.flatnonzero(d == 1)], [int(v) for v in np.flatnonzero(d == -1)]


# ---------------------------------------------------------------- oracle and helpers vs the reference

def test_fixture_cases_are_present(golden):
    names = {r["name"] for r in golden["pgs_signals"]}
    assert {"edges", "negative_zero_overlap_unsorted", "end_clamp", "max_end_negative", "negative_length",
            "two_hours"} <= names
    assert {r["start_seconds"] for r in golden["pgs_signals"]} == {0, 3, -2}
    two_h = [r for r in golden["pgs_signals"] if r["name"] == "two_hours"][0]
    assert len(two_h["starts"]) > 1000 and two_h["length"] > 100 * 3600


def test_oracle_reproduces_the_reference_signals(golden):
    for row in golden["pgs_signals"]:
        iv = list(zip(row["starts"], row["ends"]))
        if row["error"]:
            with pytest.raises(ValueError):
                po.pgs_signal(iv, 100, row["start_seconds"])
            continue
        x = po.pgs_signal(iv, 100, row["start_seconds"])
        assert len(x) == row["length"], row["name"]
        assert _runs(x) == (row["run_starts"], row["run_stops"]), (row["name"], row["start_seconds"])


def test_oracle_rounding_edges():
    assert [po.pgs_frame(t, 0, 100) for t in (0.125, 7200.125, 0.285, -0.015, 1234.565)] == \
        [12, 720012, 28, -2, 123456]
    assert po.pgs_length(-0.015, 100) == 1 and po.pgs_length(-0.025, 100) == 0 and po.pgs_length(-0.035, 100) == -1


def test_helpers_match_the_reference(golden):
    from ffsubsync_b200.speech_transformers import find_pgs_stream, pgs_timings_from_packets
    for row in golden["pgs_packets"]:
        want = None if row["timings"] is None else [tuple(t) for t in row["timings"]]
        assert pgs_timings_from_packets({"packets": row["packets"]}) == want, row["name"]
        assert po.pgs_timings(row["packets"]) == want, row["name"]
    for row in golden["pgs_streams"]:
        assert find_pgs_stream(row["probe"]) == row["stream"], row["name"]
        assert po.find_pgs_stream(row["probe"]) == row["stream"], row["name"]


def test_oracle_aligner_reproduces_the_reference_grid(golden):
    ms = golden["pgs_maxscore"]
    row = [r for r in golden["pgs_signals"] if r["name"] == "two_hours" and r["start_seconds"] == 0][0]
    ref = po.pgs_signal(list(zip(row["starts"], row["ends"])), 100, 0)
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
    g = golden["pgs_gss"]
    assert g["per_candidate"][:len(ms["per_ratio"])] == ms["per_ratio"]
    assert 0.9 <= g["gss_ratio"] <= 1.1


# ---------------------------------------------------------------- ABI

_CTYPE = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "double": ctypes.c_double}


@pytest.mark.parametrize("name,n_args", [("b2_rasterize_pgs_lengths", 5), ("b2_rasterize_pgs", 10),
                                         ("b2_sync_tracks_pgs", 43)])
def test_exported_with_the_header_signature(built, name, n_args):
    from ffsubsync_b200 import _native
    assert name in _native.EXPORTS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), name)
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    m = re.search(r"\bint\s+%s\s*\((.*?)\);" % name, header, re.S)
    assert m
    args = [" ".join(a.split()) for a in re.sub(r"/\*.*?\*/", "", m.group(1), flags=re.S).split(",")]
    want = [ctypes.c_void_p if ("*" in a or a.startswith("b2_handle")) else _CTYPE[a.rsplit(" ", 1)[0]] for a in args]
    got = getattr(_native.load(), name).argtypes
    assert len(got) == len(want) == n_args
    for i, (g, w) in enumerate(zip(got, want)):
        assert g is w, (i, args[i], g, w)


def _lengths(end, off, sr=100):
    from ffsubsync_b200 import _native
    end = np.ascontiguousarray(end, dtype=np.float64)
    off = np.ascontiguousarray(off, dtype=np.int64)
    out = np.zeros(len(off) - 1, dtype=np.int64)
    st = _native.load().b2_rasterize_pgs_lengths(end.ctypes.data, off.ctypes.data, len(off) - 1, sr, out.ctypes.data)
    return st, out


def test_lengths_on_the_host(built, golden):
    """b2_rasterize_pgs_lengths runs on the host: the fixture's lengths, and B2_ERR_BAD_ARG for every case the
    reference raises for."""
    ends, off, want = [], [0], []
    for row in golden["pgs_signals"]:
        if row["error"] or row["start_seconds"] != 0:
            continue
        ends += row["ends"]
        off.append(len(ends))
        want.append(row["length"])
    st, got = _lengths(ends, off)
    assert st == 0 and list(got) == want
    for end, off in (([], [0, 0]), ([np.nan], [0, 1]), ([np.inf], [0, 1]), ([1.0, -np.inf], [0, 2]),
                     ([1e10], [0, 1]), ([-0.05], [0, 1]), ([1.0, 2.0], [0, 2, 1])):
        assert _lengths(end, off)[0] == -1, (end, off)
    assert _lengths([1.0], [0, 1], sr=0)[0] == -1
    assert _lengths([1.0], [0, 1], sr=(1 << 28) + 1)[0] == -1
    assert _lengths([-0.035], [0, 1])[0] == -1 and _lengths([-0.025], [0, 1]) == (0, [0])
    # a null array behind a non-monotone table is never read: the whole table is checked first
    from ffsubsync_b200 import _native
    off = np.array([0, 5, 0], dtype=np.int64)
    out = np.zeros(2, dtype=np.int64)
    assert _native.load().b2_rasterize_pgs_lengths(None, off.ctypes.data, 2, 100, out.ctypes.data) == -1
    for o in ([0, 1, 2], [3, 3, 4]):   # and a null array under a monotone, non-empty table is refused
        o = np.array(o, dtype=np.int64)
        assert _native.load().b2_rasterize_pgs_lengths(None, o.ctypes.data, 2, 100, out.ctypes.data) == -1
    # a handle-less rasterisation is refused before anything is read
    from ffsubsync_b200 import _native
    assert _native.load().b2_rasterize_pgs(None, None, None, None, 0, 100, 0.0, None, None, 0) == -1


# ---------------------------------------------------------------- the kernels' arithmetic on the CPU

def _emul_bounds(t0, t1, ss, sr, n):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.int64(len(t0)).tobytes() + np.int32(sr).tobytes() + np.int64(n).tobytes())
            f.write(np.stack([t0, t1, ss], axis=1).astype(np.float64).tobytes())
        subprocess.check_call([EMUL, "bounds", src, dst])
        return np.fromfile(dst, dtype=np.int64).reshape(-1, 3)


def _oracle_bounds(t0, t1, ss, sr, n):
    first = np.maximum(np.rint((t0 - ss) * sr), 0).astype(np.int64)
    last = np.minimum(np.rint((t1 - ss) * sr), n).astype(np.int64)
    return first, last, np.trunc(t1 * sr).astype(np.int64) + 2


def test_emulated_bounds_at_the_edges(built):
    edges = np.array([0.125, 7200.125, 0.285, -0.015, 1234.565, 0.005, 0.015, -0.005, 2.5e-3, 0.0, -0.0, 1e-9,
                      -1e-9, 86400.005, 1e6 + 0.125, 9007199254.0])
    for ss in (0.0, 3.0, -2.0, 0.5, 1e-3):
        t0 = np.repeat(edges, len(edges))
        t1 = np.tile(edges, len(edges))
        s = np.full(len(t0), ss)
        got = _emul_bounds(t0, t1, s, 100, 720014)
        f, l_, n = _oracle_bounds(t0, t1, s, 100, 720014)
        assert np.array_equal(got[:, 0], f) and np.array_equal(got[:, 1], l_) and np.array_equal(got[:, 2], n)
    # python's own round / int on the issue's values
    got = _emul_bounds(np.array([0.125, 7200.125, 0.285, -0.015, 1234.565]), np.array([-0.015] * 5),
                       np.zeros(5), 100, 10 ** 9)
    assert list(got[:, 0]) == [12, 720012, 28, 0, 123456]   # -2 clamped to 0
    assert list(got[:, 2]) == [1] * 5


def test_emulated_bounds_on_random_times(built):
    rng = np.random.RandomState(20261016)
    m = 1_000_000
    # decimal times at ms / half-frame resolution (where the rounding ties are), plus raw doubles
    t0 = np.concatenate([np.round(rng.uniform(-10, 7300, m // 2), 3),
                         rng.uniform(-100, 7300, m // 4),
                         (rng.randint(-2000, 1_500_000, m // 4) + 0.5) / 200.0])
    t1 = t0 + np.where(rng.rand(m) < 0.9, np.round(rng.uniform(0, 6, m), 3), rng.uniform(-3, 3, m))
    ss = rng.choice([0.0, 3.0, -2.0, 0.25, 1.005], m)
    for sr in (100, 48000):
        got = _emul_bounds(t0, t1, ss, sr, 730000 * (sr // 100))
        f, l_, n = _oracle_bounds(t0, t1, ss, sr, 730000 * (sr // 100))
        assert np.array_equal(got[:, 0], f) and np.array_equal(got[:, 1], l_) and np.array_equal(got[:, 2], n), sr
    # the oracle's vectorised form is Python's round / int
    for i in rng.randint(0, m, 2000):
        assert po.pgs_frame(t0[i], ss[i], 100) == int(np.rint((t0[i] - ss[i]) * 100))
        assert po.pgs_length(t1[i], 100) == int(np.trunc(t1[i] * 100)) + 2


# ---------------------------------------------------------------- the planner

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
            if k == "status":
                out[k] = int(rest)
            elif k == "err":
                out[k] = rest
            elif k == "two_level":
                a, b = rest.split()
                out[k], out["ref_label"] = bool(int(a)), float(b)
            else:
                out[k] = [int(x) for x in rest.split()]
        return out


def _base(**kw):
    # three videos: 0 PGS, 1 audio (160 windows at 16 kHz / 100 Hz), 2 PGS; one track each
    req = dict(pcm_off=[0, 0, 25600, 25600], track_video=[0, 1, 2], cue_start=[1.0, 1.0, 1.0],
               cue_end=[2.0, 2.0, 2.0], cue_off=[0, 1, 2, 3], ratios=[1.0], ref_is_pgs=[1, 0, 1],
               pgs_start=[0.125, 5.0, -1.0], pgs_end=[3.0, 4.0, -0.015], pgs_off=[0, 2, 2, 3])
    req.update(kw)
    return req


def test_plan_tables(built):
    p = _plan(**_base())
    assert p["status"] == 0, p["err"]
    assert p["pgs_video"] == [0, 2] and p["sub_video"] == []
    # lengths int(max_end * 100) + 2: 402, 160 windows, int(-1.5) + 2 = 1
    assert p["ref_off"] == [0, 402, 562, 563]
    assert p["two_level"] and p["ref_label"] == 0.0 and p["ref_packed"] == [0]
    # auditok: the PGS videos are one empty chunk each, left out of the tokenizer
    a = _plan(**_base(detector=1))
    assert a["status"] == 0, a["err"]
    assert a["ch_out"] == [0, 402, 562, 563] and a["tok_off"] == [402]
    # PGS and text references on different videos; the text video's length is b2_rasterize's
    m = _plan(**_base(pcm_off=[0, 0, 0, 0], ref_is_pgs=[1, 0, 0], pgs_off=[0, 2, 2, 2], ref_is_subs=[0, 1, 1],
                      ref_cue_start=[1.0, 2.0], ref_cue_end=[1.5, 7.25], ref_cue_off=[0, 0, 1, 2]))
    assert m["status"] == 0, m["err"]
    assert m["pgs_video"] == [0] and m["sub_video"] == [1, 2] and m["ref_off"] == [0, 402, 554, 1281]
    # start_seconds moves no length
    assert _plan(**_base(start_seconds=-2.0))["ref_off"] == p["ref_off"]
    # a non-zero label with audio and PGS videos: three levels, not two
    t = _plan(**_base(label=0.25))
    assert t["status"] == 0 and not t["two_level"]
    g = _plan(**_base(label=0.25, gss=1))
    assert g["status"] == -6 and "three levels" in g["err"]
    # the lane kernel on a call with PGS videos still keeps the float reference
    assert _plan(**_base(lane=1))["ref_packed"] == [0]


@pytest.mark.parametrize("kw,msg", [
    (dict(pgs_off=[0, 2, 1, 3]), "pgs_off not monotone at 1"),
    (dict(ref_is_pgs=[1, 0, 0]), "video 2 has PGS intervals but no PGS reference"),
    (dict(pcm_off=[0, 160, 25600, 25600]), "video 0 has a PGS reference and a non-empty PCM range"),
    (dict(ref_is_subs=[1, 0, 0], ref_cue_start=[1.0], ref_cue_end=[2.0], ref_cue_off=[0, 1, 1, 1]),
     "video 0 is marked both as a PGS and as a text subtitle reference"),
    (dict(pgs_off=[0, 2, 2, 2], pgs_start=[0.125, 5.0], pgs_end=[3.0, 4.0]), "empty interval list (list 2"),
    (dict(pgs_end=[3.0, float("nan"), -0.015]), "interval end time is not finite or too large (index 1"),
    (dict(pgs_start=[float("inf"), 5.0, -1.0]), "interval start time is not finite or too large (index 0"),
    (dict(pgs_end=[3.0, 9007199254.740992, -0.015]), "interval end time is not finite or too large (index 1"),
    (dict(pgs_end=[3.0, 4.0, -0.035]), "negative signal length"),
    (dict(start_seconds=float("nan")), "start_seconds is not finite"),
    (dict(sample_rate=(1 << 28) + 1), "sample_rate"),
])
def test_plan_bad_arguments(built, kw, msg):
    p = _plan(**_base(**kw))
    assert p["status"] == -1 and msg in p["err"], p["err"]
    assert p["err"].startswith("sync_tracks_pgs: ")


# ---------------------------------------------------------------- front end

class _FakeHandle:
    device = 0

    def __init__(self):
        self.calls = []

    def _call(self, name):
        def f(*a, **kw):
            self.calls.append((name, a, kw))
            T = len(a[2])
            return (np.zeros(T), np.zeros(T, np.int32), np.zeros(T, np.int32), None, None)
        return f

    def __getattr__(self, name):
        if name.startswith("sync_"):
            return self._call(name)
        raise AttributeError(name)


@pytest.fixture
def fake(monkeypatch):
    from ffsubsync_b200 import _native
    h = _FakeHandle()
    monkeypatch.setattr(_native, "get_handle", lambda device=None: h)
    return h


def test_front_end_argument_checks(fake):
    from ffsubsync_b200.batch import BatchSynchronizer
    pcm, pcm_off = np.zeros(0, np.int16), np.array([0, 0, 0])
    cues = (np.array([1.0, 1.0]), np.array([2.0, 2.0]), np.array([0, 1, 2]))
    pgs = dict(pgs_start=[1.0, 2.0], pgs_end=[3.0, 4.0], pgs_off=[0, 1, 2], pgs_video=[0, 1])
    bs = BatchSynchronizer([1.0], vad="energy_zcr")
    for bad in (dict(pgs_video=[1, 1]), dict(pgs_video=[1, 0]), dict(pgs_video=[0, 2]), dict(pgs_video=[0]),
                dict(pgs_off=[0, 2, 1]), dict(pgs_off=[0, 1, 3]), dict(pgs_end=None)):
        with pytest.raises(ValueError):
            bs.sync_host(pcm, pcm_off, *cues, **dict(pgs, **bad))
    with pytest.raises(TypeError):
        bs.sync_host(pcm, pcm_off, *cues, pgs_stat=[1.0])
    with pytest.raises(ValueError):
        bs.sync_device_candidate_sharded(None, pcm_off, *cues, **pgs)
    assert not fake.calls


@pytest.mark.parametrize("vad", ["energy_zcr", "auditok", "subs_then_energy_zcr", "subs_then_auditok"])
def test_front_end_hands_the_intervals_to_the_call(fake, vad):
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    bs = BatchSynchronizer([1.0, 1.04], vad=vad)
    pcm = np.zeros(3200, np.int16)
    pcm_off = np.array([0, 0, 3200, 3200])   # videos 0 and 2 have PGS intervals, video 1 audio
    pgs = dict(pgs_start=[1.0, 2.0, 5.0], pgs_end=[3.0, 4.0, 9.0], pgs_off=[0, 2, 3], pgs_video=[0, 2])
    bs.sync_host(pcm, pcm_off, np.array([1.0] * 3), np.array([2.0] * 3), [0, 1, 2, 3], **pgs)
    (name, a, kw), = fake.calls
    assert name == "sync_tracks_pgs"
    is_pgs, ps, pe, poff = a[6:10]
    assert list(is_pgs) == [1, 0, 1] and list(ps) == [1.0, 2.0, 5.0] and list(pe) == [3.0, 4.0, 9.0]
    assert list(poff) == [0, 2, 2, 3]
    want = _native.B2_DETECTOR_AUDITOK if vad.endswith("auditok") else _native.B2_DETECTOR_ENERGY_ZCR
    assert kw["detector"] == want and "ref_is_subs" not in kw


def test_front_end_prefers_pgs_over_a_text_stream(fake):
    from ffsubsync_b200.batch import BatchSynchronizer
    bs = BatchSynchronizer([1.0], vad="subs_then_energy_zcr")
    pcm_off = np.array([0, 0, 0, 0])
    text = dict(ref_cue_start=[1.0, 2.0, 5.0], ref_cue_end=[3.0, 4.0, 9.0], ref_cue_off=[0, 1, 2, 3],
                ref_stream_video=[0, 1, 2], ref_cue_keep=[1, 1, 1])
    pgs = dict(pgs_start=[0.5], pgs_end=[7.0], pgs_off=[0, 1], pgs_video=[1])
    bs.sync_host(None, pcm_off, np.array([1.0] * 3), np.array([2.0] * 3), [0, 1, 2, 3], **text, **pgs)
    (name, a, kw), = fake.calls
    assert name == "sync_tracks_pgs"
    assert list(a[6]) == [0, 1, 0]
    assert list(kw["ref_is_subs"]) == [1, 0, 1] and list(kw["ref_cue_start_s"]) == [1.0, 5.0]
    assert list(kw["ref_cue_off"]) == [0, 1, 1, 2] and list(kw["ref_cue_keep"]) == [1, 1]


def test_transformer_interface():
    from ffsubsync_b200.speech_transformers import PGSSpeechTransformer
    t = PGSSpeechTransformer(100, start_seconds=3, ffmpeg_path=None, ref_stream="s:1", gui_mode=False)
    assert t.num_frames is None and t.sample_rate == 100 and t.start_seconds == 3 and t.ref_stream == "s:1"
    with pytest.raises(ValueError):
        t.fit([])
