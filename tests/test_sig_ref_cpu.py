"""CPU suite for serialized speech signals as references (b2_sync_tracks_sig, ``ffs ref.npz -i in.srt``).

Checks what can be checked without a GPU: the float64 oracle against fixtures recorded from the reference's
DeserializeSpeechTransformer (tests/golden/make_golden_signal_ref.py), the stored-value loader, the symbol and its
ctypes signature against the header, the planner's signal tables, checks and level / path / packed rules
(sync_plan.h, through tests/host_emul/sig_ref_emul), and sig_ref_kernel's arithmetic and word layout run thread by
thread on the CPU at the edges."""
import json
import math
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from oracle import sig_oracle as so

GOLDEN = os.path.join(ROOT, "tests", "golden", "signal_ref.json")
EMUL = os.path.join(ROOT, "tests", "host_emul", "sig_ref_emul")


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


# ---------------------------------------------------------------- oracle and loader vs the reference

def test_fixture_cases_are_present(golden):
    rows, stored = golden["signals"], golden["stored"]
    # every stored signal at every label, read back from both file formats (the generator checks they agree)
    assert {(r["name"], r["label"]) for r in rows} == {(s["name"], lb) for s in stored for lb in (0.0, 0.5, -0.5)}
    assert all(r["formats"] == ["npz", "npy"] for r in rows)
    lengths = {s["length"] for s in stored}
    assert {32, 33, 63, 0} <= lengths and any(n < 32 for n in lengths if n) and max(lengths) >= 100 * 7200
    levels = {float(v) for s in stored for v in s["levels"]}
    assert {1.0 - 2.0 ** -53, 1.0 - 2.0 ** -25, 1.0, -np.inf, 0.5, 0.0} <= levels and min(levels) < 0


def test_oracle_reproduces_the_reference(golden):
    for r in golden["signals"]:
        x = so.stored_signal(golden, r["name"])
        want = so.from_runs(r["out_levels"], r["out_starts"], r["length"])
        got = so.deserialize(x, r["label"])
        assert got.dtype == np.float64 and np.array_equal(got, want), (r["name"], r["label"])
        # the domain: two levels, 1.0 and the label
        assert set(np.unique(want).tolist()) <= {1.0, r["label"]}
        assert so.first_bad_frame(x) == -1
    # the rounding edge: the rule in float64 keeps 1 - 2^-25 non-speech, rounding first would not
    x = np.array([1.0 - 2.0 ** -25, 1.0 - 2.0 ** -53, 1.0, np.nextafter(1.0, 0.0)])
    assert so.frames(x, 0.0).tolist() == [0.0, 0.0, 1.0, 0.0]
    assert np.float32(1.0 - 2.0 ** -25) == np.float32(1.0)
    assert so.first_bad_frame([0.0, 1.0, np.nextafter(1.0, 2.0)]) == 2 and so.first_bad_frame([np.nan]) == 0


def test_stored_values_loader(golden, tmp_path):
    from ffsubsync_b200.batch import load_serialized_speech
    from ffsubsync_b200.speech_transformers import DeserializeSpeechTransformer
    rows = [s for s in golden["stored"] if s["length"] < 10000]
    paths, xs = [], []
    for i, r in enumerate(rows):
        x = so.from_runs(r["levels"], r["starts"], r["length"])
        p = str(tmp_path / ("s%d.%s" % (i, "npz" if i % 2 else "npy")))
        np.savez(p, speech=x) if i % 2 else np.save(p, x)
        paths.append(p)
        xs.append(x)
    vals, off = load_serialized_speech(paths, stored=True)
    assert vals.dtype == np.float64 and np.array_equal(vals, np.concatenate(xs))
    assert off.tolist() == np.concatenate([[0], np.cumsum([len(x) for x in xs])]).tolist()
    # the default output is unchanged: DeserializeSpeechTransformer's, rounded to float32
    sig, off2 = load_serialized_speech(paths, 0.5)
    want = np.concatenate([DeserializeSpeechTransformer(0.5).fit(p).transform() for p in paths]).astype(np.float32)
    assert sig.dtype == np.float32 and np.array_equal(sig, want) and np.array_equal(off, off2)
    assert np.array_equal(sig, so.frames(vals, 0.5))


# ---------------------------------------------------------------- ABI

def test_export_and_header_signature(built):
    from ffsubsync_b200 import _native
    hdr = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    m = re.search(r"int b2_sync_tracks_sig\((.*?)\);", hdr, re.S)
    assert m
    params = [p for p in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",") if p.strip()]
    lib = _native.load()
    assert len(lib.b2_sync_tracks_sig.argtypes) == len(params) == 46
    assert "b2_sync_tracks_sig" in _native.EXPORTS
    assert re.search(r"#define B2_BEST_K_BAD_SIGNAL \(-2\)", hdr) and _native.B2_BEST_K_BAD_SIGNAL == -2
    # the signal arguments follow the PGS ones, as documented
    names = [re.findall(r"(\w+)\s*$", p.strip())[0] for p in params]
    assert names[27:30] == ["ref_is_sig", "x", "sig_off"] and names[23:27] == ["ref_is_pgs", "pgs_start_s",
                                                                             "pgs_end_s", "pgs_off"]
    # refused without a handle, before anything is read
    assert lib.b2_sync_tracks_sig(*([None] * 3 + [0, None, 0, 16000, 100, 0, 0.0, 0, -1, -1, 50.0, 0.0, 0, 0.0, 0]
                                    + [None] * 17 + [1, 0.0, 0] + [None] * 7 + [0])) == -1


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
    # four videos: 0 signal (500 frames), 1 audio (160 windows at 16 kHz / 100 Hz), 2 signal (33), 3 empty signal;
    # one track each
    req = dict(pcm_off=[0, 0, 25600, 25600, 25600], track_video=[0, 1, 2, 3], cue_start=[1.0] * 4, cue_end=[2.0] * 4,
               cue_off=[0, 1, 2, 3, 4], ratios=[1.0], ref_is_sig=[1, 0, 1, 1], sig_off=[0, 500, 500, 533, 533])
    req.update(kw)
    return req


def test_plan_tables(built):
    p = _plan(**_base())
    assert p["status"] == 0, p["err"]
    assert p["sig_video"] == [0, 2, 3] and p["sub_video"] == [] and p["pgs_video"] == []
    assert p["ref_off"] == [0, 500, 660, 693, 693]   # R = sig_off[v+1] - sig_off[v]; 160 windows
    assert p["audio_samples"] == [25600]
    # auditok: each signal video one empty chunk spanning its frames, left out of the tokenizer's table
    a = _plan(**_base(detector=1))
    assert a["status"] == 0, a["err"]
    assert a["ch_out"] == [0, 500, 660, 693, 693] and a["ch_first"] == [0, 1, 2, 3, 4] and a["tok_off"] == [500]
    assert a["ref_off"] == p["ref_off"]
    # signals alone and no audio: no PCM read
    s = _plan(**_base(pcm_off=[0, 0, 0, 0, 0], ref_is_sig=[1, 1, 1, 1], sig_off=[0, 500, 600, 633, 633]))
    assert s["status"] == 0 and s["ref_off"] == [0, 500, 600, 633, 633] and s["audio_samples"] == [0]
    # start_seconds moves no length
    assert _plan(**_base(start_seconds=-2.0))["ref_off"] == p["ref_off"]
    # signal, PGS and text references on different videos
    m = _plan(**_base(pcm_off=[0] * 5, ref_is_sig=[1, 0, 0, 0], sig_off=[0, 500, 500, 500, 500],
                      ref_is_pgs=[0, 1, 0, 0], pgs_start=[0.125], pgs_end=[3.0], pgs_off=[0, 0, 1, 1, 1],
                      ref_is_subs=[0, 0, 1, 0], ref_cue_start=[1.0], ref_cue_end=[7.25], ref_cue_off=[0, 0, 0, 1, 1]))
    assert m["status"] == 0, m["err"]
    assert m["sig_video"] == [0] and m["pgs_video"] == [1] and m["sub_video"] == [2]
    assert m["ref_off"][:4] == [0, 500, 802, 1529]


@pytest.mark.parametrize("kw,msg", [
    (dict(sig_off=[0, 500, 400, 533, 533]), "sig_off not monotone at 1"),
    (dict(ref_is_sig=[1, 0, 0, 1], sig_off=[0, 500, 500, 533, 533]), "video 2 has signal values but no signal reference"),
    (dict(pcm_off=[0, 160, 25760, 25760, 25760]), "video 0 has a signal reference and a non-empty PCM range (160"),
    (dict(ref_is_pgs=[1, 0, 0, 0], pgs_start=[1.0], pgs_end=[2.0], pgs_off=[0, 1, 1, 1, 1]),
     "video 0 is marked both as a signal and as a PGS reference"),
    (dict(ref_is_subs=[0, 0, 1, 0], ref_cue_start=[1.0], ref_cue_end=[2.0], ref_cue_off=[0, 0, 0, 1, 1]),
     "video 2 is marked both as a signal and as a text subtitle reference"),
    (dict(x_null=1), "null signal values x with 533 values"),
])
def test_bad_arguments(built, kw, msg):
    p = _plan(**_base(**kw))
    assert p["status"] == -1 and msg in p["err"], p["err"]
    assert p["err"].startswith("sync_tracks_sig: ")


def test_null_values_without_values_are_fine(built):
    p = _plan(**_base(x_null=1, ref_is_sig=[1, 0, 1, 1], sig_off=[0, 0, 0, 0, 0]))
    assert p["status"] == 0 and p["ref_off"] == [0, 0, 160, 160, 160]


def _levels(p, label):
    return p["two_level"], p["ref_label"]


@pytest.mark.parametrize("label", [0.0, 0.3, -0.5])
def test_level_and_path_rules(built, label):
    """A signal video counts like a detector video: levels 1.0 and the label."""
    pgs = dict(ref_is_pgs=[0, 0, 0, 1], pgs_start=[0.5], pgs_end=[2.0], pgs_off=[0, 0, 0, 0, 1],
               ref_is_sig=[1, 0, 1, 0], sig_off=[0, 500, 500, 533, 533])
    sig_only = dict(pcm_off=[0] * 5, ref_is_sig=[1, 1, 1, 1], sig_off=[0, 500, 600, 633, 633])
    for det, lab in ((0, dict(label=label)), (1, dict(auditok_label=label))):
        # signals alone: two-level with either detector, ref_label = the label; the search runs
        for gss in (0, 1):
            p = _plan(**_base(detector=det, gss=gss, **sig_only, **lab))
            assert p["status"] == 0 and p["two_level"] and p["ref_label"] == pytest.approx(label, abs=1e-7), (det, p)
        # with audio: two-level with energy audio at any label, with auditok audio only at label 0
        p = _plan(**_base(detector=det, **lab))
        assert p["status"] == 0 and p["ref_label"] == pytest.approx(label, abs=1e-7)
        assert p["two_level"] == (det == 0 or label == 0.0), (det, label)
        g = _plan(**_base(detector=det, gss=1, **lab))
        assert g["status"] == (0 if det == 0 or label == 0.0 else -6), (det, label, g["err"])
        # with a PGS video: three levels at a non-zero label, whichever the detector
        m = _plan(**_base(detector=det, **pgs, **lab))
        assert m["status"] == 0 and m["two_level"] == (label == 0.0)
        g = _plan(**_base(detector=det, gss=1, **pgs, **lab))
        assert g["status"] == (0 if label == 0.0 else -6), g["err"]
        if label != 0.0:
            assert "three levels" in g["err"] or "more than two levels" in g["err"]


def _chain_runs(req, p, i):
    from test_ref_packed_cpu import _chain_takes_runs
    K = len(req["ratios"])
    v0, v1 = p["cut"][i], p["cut"][i + 1]
    t0, t1 = p["trk_off"][v0], p["trk_off"][v1]
    R = np.diff(p["ref_off"][v0:v1 + 1])
    S = np.diff(p["sub_off"][t0 * K:t1 * K + 1])
    cue_n = np.diff(np.asarray(req["cue_off"]))
    trk = np.asarray(p["trk_off"][v0:v1 + 1]) - p["trk_off"][v0]
    return _chain_takes_runs(R, S, cue_n[t0:t1], trk, K, 6000, req)


def _expected_packed(req, p):
    """A sub-batch is packed when its chain takes the run path and every video in it is a signal video or
    lane-eligible energy audio; text / PGS references, auditok audio and lane-group audio keep floats."""
    V = len(p["ref_off"]) - 1
    z = [0] * V
    is_sig, is_subs, is_pgs = (np.asarray(req.get(k, z)) != 0 for k in ("ref_is_sig", "ref_is_subs", "ref_is_pgs"))
    auditok = req.get("detector", 0) == 1
    out = []
    for i in range(len(p["cut"]) - 1):
        v0, v1 = p["cut"][i], p["cut"][i + 1]
        videos_ok = all(is_sig[v] or (not auditok and req.get("lane", 0) and not is_subs[v] and not is_pgs[v])
                        for v in range(v0, v1))
        ok = (videos_ok and req.get("ref_packed") != "0" and p["two_level"] and math.isfinite(p["ref_label"])
              and _chain_runs(req, p, i))
        out.append(int(bool(ok)))
    return out


def _mixed(V, kinds, **kw):
    """V videos of kinds ("sig", "audio", "pgs", "text") by index, 2 tracks each, 30 s signals / audio."""
    pcm, sig = [0], [0]
    for v in range(V):
        k = kinds[v % len(kinds)]
        pcm.append(pcm[-1] + (3000 * 160 if k == "audio" else 0))
        sig.append(sig[-1] + (3000 + v if k == "sig" else 0))
    T = 2 * V
    req = dict(pcm_off=pcm, track_video=np.repeat(np.arange(V), 2), cue_start=np.tile([1.0, 5.0], T),
               cue_end=np.tile([2.0, 9.0], T), cue_off=np.arange(0, 2 * T + 1, 2), ratios=[1.0, 25 / 24.0],
               ref_is_sig=[int(kinds[v % len(kinds)] == "sig") for v in range(V)], sig_off=sig)
    if "pgs" in kinds:
        pv = [v for v in range(V) if kinds[v % len(kinds)] == "pgs"]
        req.update(ref_is_pgs=[int(v in pv) for v in range(V)], pgs_start=[0.5] * len(pv), pgs_end=[20.0] * len(pv),
                   pgs_off=np.concatenate([[0], np.cumsum([int(v in pv) for v in range(V)])]))
    if "text" in kinds:
        tv = [v for v in range(V) if kinds[v % len(kinds)] == "text"]
        req.update(ref_is_subs=[int(v in tv) for v in range(V)], ref_cue_start=[0.5] * len(tv),
                   ref_cue_end=[25.0] * len(tv), ref_cue_off=np.concatenate([[0], np.cumsum([int(v in tv)
                                                                                           for v in range(V)])]))
    req.update(kw)
    return req


@pytest.mark.parametrize("kinds", [("sig",), ("sig", "audio"), ("audio", "sig", "sig"), ("sig", "pgs"),
                                   ("sig", "sig", "text", "sig"), ("audio",)])
@pytest.mark.parametrize("det,lane,label,subs,packed_env", [
    (0, 1, 0.0, "3", None), (0, 1, 0.3, "4", None), (0, 0, 0.0, "3", None), (1, 0, 0.0, "3", None),
    (1, 0, 0.3, "2", None), (0, 1, -0.5, "3", "0"), (0, 1, 0.0, "1", None)])
def test_packed_flag_per_sub_batch(built, kinds, det, lane, label, subs, packed_env):
    extra = dict(detector=det, lane=lane, subbatches=subs)
    extra.update(dict(label=label) if det == 0 else dict(auditok_label=label))
    if packed_env is not None:
        extra["ref_packed"] = packed_env
    req = _mixed(12, kinds, **extra)
    p = _plan(**req)
    assert p["status"] == 0, p["err"]
    assert len(p["cut"]) - 1 == int(subs)
    assert p["ref_packed"] == _expected_packed(req, p), (kinds, p["cut"], p["ref_packed"])
    if kinds == ("sig",) and packed_env is None:
        assert p["ref_packed"] == [1] * int(subs)   # signals alone are packed with either detector


# ---------------------------------------------------------------- sig_ref_kernel on the CPU

def _emul_kernel(x, label, packed):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.int64(len(x)).tobytes() + np.float32(label).tobytes() + np.int32(packed).tobytes())
            f.write(np.asarray(x, dtype=np.float64).tobytes())
        subprocess.check_call([EMUL, "kernel", src, dst])
        raw = np.fromfile(dst, dtype=np.uint8)
        first = int(raw[:8].view(np.int64)[0])
        body = raw[8:].view(np.uint32 if packed else np.float32)
        return first, body


EDGE = np.array([1.0 - 2.0 ** -53, 1.0 - 2.0 ** -25, 1.0, 0.0, -0.5, -np.inf, 0.999, np.nextafter(1.0, 0.0),
                 -0.0, 1e-300, -1e308, 0.5])


@pytest.mark.parametrize("n", [0, 1, 7, 31, 32, 33, 63, 64, 95, 255, 256, 257, 8191, 8192, 8193, 20000])
def test_emulated_kernel_at_the_edges(built, n):
    rng = np.random.RandomState(n)
    x = EDGE[rng.randint(0, len(EDGE), n)]
    x[rng.rand(n) < 0.45] = 1.0
    for label in (0.0, 0.3, -0.5, 1.0):
        f = so.frames(x, label)
        first, frames = _emul_kernel(x, label, 0)
        assert first == -1 and np.array_equal(frames, f), (n, label)
        first, words = _emul_kernel(x, label, 1)
        assert first == -1 and np.array_equal(words, so.packed_words(f)), (n, label)
        assert len(words) == (n + 31) // 32
        if n % 32:   # zero bits past R, even where every frame is 1.0
            assert words[-1] >> (n % 32) == 0


@pytest.mark.parametrize("where", [[0], [31], [32], [8191, 8192], [9000, 300], [19999], [5, 17000, 12]])
def test_emulated_kernel_flags_the_first_out_of_domain_frame(built, where):
    x = np.where(np.arange(20000) % 3 == 0, 1.0, 0.25)
    for i, w in enumerate(where):
        x[w] = [2.0, np.nan, np.inf, np.nextafter(1.0, 2.0)][i % 4]
    for packed in (0, 1):
        first, body = _emul_kernel(x, 0.0, packed)
        assert first == min(where) == so.first_bad_frame(x)
    # out-of-domain frames are written as the label: the chain still sees two levels
    _, frames = _emul_kernel(x, -0.5, 0)
    assert set(np.unique(frames).tolist()) <= {1.0, -0.5}
