"""CPU suite for sampled segments as references (b2_sync_tracks_seg, ``--multi-segment-sync``).

Checks what can be checked without a GPU: the float64 oracle against the reference's assembly fixture, the table
helper's starts against the reference's ``_segment_starts`` fixture, the symbol and its ctypes signature against the
header, the planner's segment tables, owned frames, lengths, checks and level / packed rules (sync_plan.h, through
tests/host_emul/seg_ref_emul), and seg_ref_kernel's loop nest run thread by thread on the CPU."""
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from oracle import segment_oracle as so

GOLDEN = os.path.join(ROOT, "tests", "golden", "golden.json")
EMUL = os.path.join(ROOT, "tests", "host_emul", "seg_ref_emul")


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


# ---------------------------------------------------------------- oracle and helper vs the reference

def test_oracle_assembly_matches_the_reference(golden):
    for c in golden["segment_assembly"]:
        from ffsubsync_b200.speech_transformers import MultiSegmentVideoSpeechTransformer
        t = MultiSegmentVideoSpeechTransformer(vad="webrtc", sample_rate=100, frame_rate=48000, non_speech_label=0.0,
                                               segment_count=c["count"], segment_duration=c["duration"])
        starts = t._segment_starts(c["total"])
        outs = [(s, np.full(c["duration"] * 100, (s % 7 + 1) / 8.0)) for s in starts if s != c["failing"]]
        x = so.assemble(c["total"], 100, outs)
        want = np.zeros(c["len"])
        for a, b, v in c["runs"]:
            want[a:b] = v
        assert len(x) == c["len"] == so.length(c["total"], 100) and np.array_equal(x, want), c


def test_oracle_overlap_order_and_speech():
    # 100 s video, three 60 s segments: later starts win where they overlap; uncovered frames stay 0.0
    x = so.assemble(100.0, 100, [(0, np.full(6000, 0.25)), (20, np.full(6000, 0.5)), (40, np.full(10, 1.0))])
    assert len(x) == 10002 and x[0] == 0.25 and x[1999] == 0.25 and x[2000] == 0.5
    assert x[4000:4010].tolist() == [1.0] * 10 and x[4010] == 0.5 and x[7999] == 0.5 and x[8000] == 0.0
    assert so.has_speech(x) and not so.has_speech(np.zeros(5)) and not so.has_speech(np.full(3, -0.5))
    # a segment past the end writes nothing
    assert not so.has_speech(so.assemble(1.0, 100, [(5, np.ones(100))]))


def test_helper_starts_match_the_reference(golden):
    from ffsubsync_b200.batch import segment_table
    for c in golden["segment_starts"]:
        n = int(round(c["total"] * 100))   # a 100 Hz "PCM" of that length
        tab = segment_table([0, n], 100, totals=[c["total"]], segment_count=c["count"],
                            segment_duration=c["duration"], skip_intro_outro=c["skip"])
        assert tab["seg_start"].tolist() == c["starts"], c
        assert tab["seg_off"].tolist() == [0, len(c["starts"])] and tab["seg_total"].tolist() == [c["total"]]
        lo = np.minimum(n, np.round(np.array(c["starts"]) * 100).astype(np.int64))
        assert tab["seg_lo"].tolist() == lo.tolist()
        assert tab["seg_hi"].tolist() == np.minimum(n, lo + c["duration"] * 100).tolist()


def test_helper_layouts():
    from ffsubsync_b200.batch import segment_table
    fr = 16000
    pcm_off = [0, 7200 * fr, 7200 * fr, 7200 * fr + 40 * fr + 7]
    full = segment_table(pcm_off, fr, videos=[0, 2], segment_count=3)
    assert full["seg_video"].tolist() == [0, 2] and full["seg_off"].tolist() == [0, 3, 4]
    assert full["seg_total"].tolist() == [7200.0, (40 * fr + 7) / fr]   # samples / frame_rate by default
    assert full["seg_start"].tolist() == [0, 3570, 7140, 0]
    assert full["seg_lo"].tolist() == [0, 3570 * fr, 7140 * fr, 0]
    assert full["seg_hi"].tolist() == [60 * fr, 3630 * fr, 7200 * fr, 40 * fr + 7]   # a short video: clipped
    # decoded windows back to back: the pieces' own sample counts
    pieces = [[60 * fr, 60 * fr - 3, 60 * fr], [40 * fr + 7]]
    dec = segment_table([0, 180 * fr - 3, 180 * fr - 3, 220 * fr + 4], fr, videos=[0, 2], totals=[7200.0, 40.0],
                        segment_count=3, piece_samples=pieces)
    assert dec["seg_start"].tolist() == full["seg_start"].tolist() and dec["seg_total"].tolist() == [7200.0, 40.0]
    assert dec["seg_lo"].tolist() == [0, 60 * fr, 120 * fr - 3, 0]
    assert dec["seg_hi"].tolist() == [60 * fr, 120 * fr - 3, 180 * fr - 3, 40 * fr + 7]
    with pytest.raises(ValueError, match="decoded pieces"):
        segment_table([0, 100], fr, totals=[7200.0], piece_samples=[[100]])


# ---------------------------------------------------------------- ABI

def test_export_and_header_signature(built):
    from ffsubsync_b200 import _native
    hdr = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    m = re.search(r"int b2_sync_tracks_seg\((.*?)\);", hdr, re.S)
    assert m
    params = [p for p in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",") if p.strip()]
    lib = _native.load()
    assert len(lib.b2_sync_tracks_seg.argtypes) == len(params) == 53
    assert "b2_sync_tracks_seg" in _native.EXPORTS
    assert re.search(r"#define B2_BEST_K_NO_SPEECH \(-3\)", hdr) and _native.B2_BEST_K_NO_SPEECH == -3
    names = [re.findall(r"(\w+)\s*$", p.strip())[0] for p in params]
    assert names[27:37] == ["ref_is_sig", "x", "sig_off", "n_seg_videos", "seg_video", "seg_total", "seg_off",
                            "seg_start", "seg_lo", "seg_hi"]
    assert lib.b2_sync_tracks_seg(*([None] * 3 + [0, None, 0, 16000, 100, 0, 0.0, 0, -1, -1, 50.0, 0.0, 0, 0.0, 0]
                                    + [None] * 12 + [0] + [None] * 11 + [1, 0.0, 0] + [None] * 7 + [0])) == -1


# ---------------------------------------------------------------- the planner

def _plan(env=None, **req):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            for k, v in req.items():
                vals = [v] if np.isscalar(v) or isinstance(v, str) else list(np.asarray(v).ravel())
                f.write("%s %d %s\n" % (k, len(vals), " ".join(
                    x if isinstance(x, str) else repr(float(x)) if isinstance(x, (float, np.floating)) else str(int(x))
                    for x in vals)))
        subprocess.check_call([EMUL, "plan", src, dst], env=None if env is None else dict(os.environ, **env))
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


FR = 16000


def _base(**kw):
    # three videos at 16 kHz / 100 Hz: 0 segments (a 100 s full decode: starts 0, 20, 40 of 60 s - overlapping), 1
    # audio (160 windows), 2 segments (decoded pieces back to back: 2 x 10 s at 0 s and 3590 s of a 3600 s video, the
    # last one short); one track each
    req = dict(pcm_off=[0, 100 * FR, 100 * FR + 25600, 100 * FR + 25600 + 20 * FR - 5], track_video=[0, 1, 2],
               cue_start=[1.0] * 3, cue_end=[2.0] * 3, cue_off=[0, 1, 2, 3], ratios=[1.0],
               seg_video=[0, 2], seg_total=[100.0, 3600.0], seg_off=[0, 3, 5], seg_start=[0, 20, 40, 0, 3590],
               seg_lo=[0, 20 * FR, 40 * FR, 0, 10 * FR], seg_hi=[60 * FR, 80 * FR, 100 * FR, 10 * FR, 20 * FR - 5])
    req.update(kw)
    return req


def test_plan_tables(built):
    p = _plan(**_base())
    assert p["status"] == 0, p["err"]
    assert p["seg_video"] == [0, 2]
    # reference lengths: int(total * 100) + 2 for segment videos, the windows for audio
    assert p["ref_off"] == [0, 10002, 10162, 10162 + 360002]
    # the main launch leaves the segment videos empty
    assert p["det_end"] == [0, 100 * FR + 25600, 100 * FR + 25600]
    # one item per segment, absolute samples, compact scratch
    a2 = 100 * FR + 25600
    assert p["item_start"][:5] == [0, 20 * FR, 40 * FR, a2, a2 + 10 * FR]
    assert p["item_end"] == [60 * FR, 80 * FR, 100 * FR, a2 + 10 * FR, a2 + 20 * FR - 5]
    assert p["item_out"] == [0, 6000, 12000, 18000, 19000, 20000]   # ceil((10 s - 5) / 160) = 1000
    assert p["item_first"] == [0, 3, 3, 5] and p["item_tail"] == [0] * 5
    # owned frames: video 0 = seg 0 [0, 2000), seg 1 [2000, 4000), seg 2 [4000, 10000), 0.0 after
    assert p["run_first"] == [0, 4, 8]
    assert p["run_lo"][:4] == [0, 2000, 4000, 10000] and p["run_src"][:4] == [0, 6000, 12000, -1]
    # video 2: seg 0 [0, 1000), 0.0 up to 359000, seg 1 [359000, 360000), 0.0 for the last two frames
    assert p["run_lo"][4:] == [0, 1000, 359000, 360000] and p["run_src"][4:] == [18000, -1, 19000, -1]
    # only segment samples count (overlapping ones as often as the detector reads them), and B2_HOST stages only
    # what the detector reads
    assert p["audio_samples"] == [180 * FR + 25600 + 20 * FR - 5]
    assert p["stage_lo"] == [0] and p["stage_hi"] == [100 * FR + 25600 + 20 * FR - 5]
    # a full decode of the second video: gaps are not staged
    q = _plan(**_base(pcm_off=[0, 100 * FR, 100 * FR + 25600, 100 * FR + 25600 + 3600 * FR],
                      seg_lo=[0, 20 * FR, 40 * FR, 0, 3590 * FR], seg_hi=[60 * FR, 80 * FR, 100 * FR, 10 * FR,
                                                                           3600 * FR]))
    assert q["status"] == 0, q["err"]
    assert q["stage_lo"] == [0, a2 + 3590 * FR] and q["stage_hi"] == [a2 + 10 * FR, a2 + 3600 * FR]
    assert q["audio_samples"] == [180 * FR + 25600 + 20 * FR]
    # start_seconds moves no segment
    assert _plan(**_base(start_seconds=-2.0))["run_lo"] == p["run_lo"]


def test_plan_auditok_items(built):
    p = _plan(**_base(detector=1, chunk_samples=25 * FR))
    assert p["status"] == 0, p["err"]
    # 60 s segments in chunks of 25 s from their own first sample: 25 + 25 + 10 s
    assert p["item_start"][:3] == [0, 25 * FR, 50 * FR] and p["item_end"][:3] == [25 * FR, 50 * FR, 60 * FR]
    assert p["item_out"][:4] == [0, 2500, 5000, 6000]
    assert p["item_first"] == [0, 9, 9, 11] and p["item_tail"][-1] > 0   # the short last block of the 10 s - 5 piece
    # the segment videos are one empty chunk each in the main table, left out of the tokenizer's
    assert p["ch_out"][:2] == [0, 10002] and p["ref_off"] == [0, 10002, 10162, 370164]
    assert p["det_end"][0] == 0 and p["tok_off"] == [10002]


def test_plan_overlaps_and_clipping(built):
    # segments longer than the reference: clipped at L; a later short segment inside an earlier one splits it
    p = _plan(**_base(seg_total=[30.0, 3600.0], seg_start=[0, 10, 20, 0, 3590],
                      seg_hi=[60 * FR, 20 * FR + 100 * 160, 100 * FR, 10 * FR, 20 * FR - 5]))
    assert p["status"] == 0, p["err"]
    L = 3002
    assert p["ref_off"][1] == L
    # segment 1 has 100 frames: [1000, 1100) from it, then segment 0 again up to 2000 where segment 2 starts
    assert p["run_lo"] == [0, 1000, 1100, 2000] + p["run_lo"][4:] and p["run_src"][:4] == [0, 6000, 1100, 6100]
    assert p["run_first"][1] == 4   # [2000, L) all segment 2's: no zero run
    p = _plan(**_base(seg_start=[0, 10, 50, 0, 3590], seg_hi=[60 * FR, 20 * FR + 100 * 160, 100 * FR, 10 * FR,
                                                               20 * FR - 5]))
    assert p["run_lo"][:4] == [0, 1000, 1100, 5000] and p["run_first"][1] == 4   # segment 2 clipped at L = 10002
    assert p["run_src"][:4] == [0, 6000, 1100, 6100]


@pytest.mark.parametrize("kw,msg", [
    (dict(seg_off=[0, 3, 2]), "seg_off not monotone at 1"),
    (dict(seg_video=[0, 0]), "seg_video[1] = 0 is out of [0, 3) or not increasing"),
    (dict(seg_video=[0, 3]), "seg_video[1] = 3 is out of [0, 3)"),
    (dict(seg_total=[float("nan"), 3600.0]), "seg_total[0] = nan (video 0) is not finite"),
    (dict(seg_total=[100.0, -1.0]), "gives a negative signal length"),
    (dict(seg_total=[100.0, 1e300]), "seg_total[1]"),
    (dict(seg_start=[0, 20, 40, -1, 3590]), "segment 3 of video 2 starts at -1 s, outside"),
    (dict(seg_start=[0, 20, 20, 0, 3590]), "segment 2 of video 0 starts at 20 s, not after the previous one (20 s)"),
    (dict(seg_hi=[60 * FR, 80 * FR, 100 * FR + 1, 10 * FR, 20 * FR - 5]),
     "segment 2 of video 0 has the sample range [640000, 1600001), not inside the video's PCM range [0, 1600000)"),
    (dict(seg_lo=[0, 20 * FR, 40 * FR, -1, 10 * FR]), "segment 3 of video 2 has the sample range [-1,"),
    (dict(ref_is_sig=[1, 0, 0], sig_off=[0, 5, 5, 5]),
     "video 0 has sampled segments and a serialized signal reference; a video has one reference"),
    (dict(ref_is_pgs=[0, 0, 1], pgs_start=[1.0], pgs_end=[2.0], pgs_off=[0, 0, 0, 1]),
     "video 2 has sampled segments and a PGS reference"),
    (dict(ref_is_subs=[1, 0, 0], ref_cue_start=[1.0], ref_cue_end=[2.0], ref_cue_off=[0, 1, 1, 1]),
     "video 0 has sampled segments and a text subtitle reference"),
])
def test_bad_arguments(built, kw, msg):
    p = _plan(**_base(**kw))
    assert p["status"] == -1 and msg in p["err"], p["err"]
    assert p["err"].startswith("sync_tracks_seg: ")


@pytest.mark.parametrize("label", [0.0, 0.3, -0.5])
def test_level_rules(built, label):
    """A segment reference is two-level only at label 0, where it mixes like a subtitle reference."""
    # segment videos only (video 1 is a segment video without segments)
    only = dict(pcm_off=[0, 100 * FR, 100 * FR, 100 * FR + 20 * FR - 5], seg_video=[0, 1, 2], seg_total=[100.0, 1.0,
                3600.0], seg_off=[0, 3, 3, 5])
    for det, lab in ((0, dict(label=label)), (1, dict(auditok_label=label))):
        for extra in (only, {}):
            p = _plan(**_base(detector=det, **extra, **lab))
            assert p["status"] == 0 and p["two_level"] == (label == 0.0), (det, extra, p)
            g = _plan(**_base(detector=det, gss=1, **extra, **lab))
            assert g["status"] == (0 if label == 0.0 else -6), (det, g["err"])
            if label != 0.0:
                assert "sampled segments (0.0 outside them)" in g["err"]
        # with audio the reference label is the call's; segments alone have the levels 1.0 and 0.0
        assert _plan(**_base(detector=det, **lab))["ref_label"] == pytest.approx(label, abs=1e-7)
        assert _plan(**_base(detector=det, **only, **lab))["ref_label"] == 0.0


def _mixed(V, kinds, **kw):
    """V videos of kinds ("seg", "audio") by index, 2 tracks each, 30 s of audio; segment videos a 30 s full decode
    with two 10 s segments at 0 and 15 s."""
    pcm, sv, st, lo, hi = [0], [], [], [], []
    for v in range(V):
        pcm.append(pcm[-1] + 30 * FR)
        if kinds[v % len(kinds)] == "seg":
            sv.append(v)
            st += [0, 15]
            lo += [0, 15 * FR]
            hi += [10 * FR, 25 * FR]
    T = 2 * V
    req = dict(pcm_off=pcm, track_video=np.repeat(np.arange(V), 2), cue_start=np.tile([1.0, 5.0], T),
               cue_end=np.tile([2.0, 9.0], T), cue_off=np.arange(0, 2 * T + 1, 2), ratios=[1.0, 25 / 24.0],
               seg_video=sv, seg_total=[30.0] * len(sv), seg_off=np.arange(0, 2 * len(sv) + 1, 2), seg_start=st,
               seg_lo=lo, seg_hi=hi)
    req.update(kw)
    return req


@pytest.mark.parametrize("kinds", [("seg",), ("seg", "audio"), ("audio", "seg", "seg")])
@pytest.mark.parametrize("det,label,subs,packed_env", [
    (0, 0.0, "3", None), (0, 0.3, "3", None), (1, 0.0, "2", None), (0, 0.0, "3", "0"), (0, 0.0, "1", None)])
def test_packed_flag_per_sub_batch(built, kinds, det, label, subs, packed_env):
    from test_sig_ref_cpu import _chain_runs
    extra = dict(detector=det, lane=1, subbatches=subs)
    extra.update(dict(label=label) if det == 0 else dict(auditok_label=label))
    if packed_env is not None:
        extra["ref_packed"] = packed_env
    req = _mixed(12, kinds, **extra)
    p = _plan(**req)
    assert p["status"] == 0, p["err"]
    is_seg = set(p["seg_video"])
    for i in range(len(p["cut"]) - 1):
        v0, v1 = p["cut"][i], p["cut"][i + 1]
        videos_ok = all(v in is_seg or det == 0 for v in range(v0, v1))
        want = videos_ok and packed_env != "0" and p["two_level"] and _chain_runs(req, p, i)
        assert p["ref_packed"][i] == int(bool(want)), (kinds, det, label, i)
    if label != 0.0:
        assert p["ref_packed"] == [0] * len(p["ref_packed"])


def test_lane_eligibility_is_per_segment(built):
    # "lane 2": the real 8-sample alignment test; a segment starting off a multiple of 8 keeps the call unpipelined
    req = _mixed(120, ("seg", "audio"), lane=2)
    assert _plan(**req)["n_sub"] == [3]
    req["seg_lo"] = list(req["seg_lo"])
    req["seg_lo"][1] += 3
    assert _plan(**req)["n_sub"] == [1]
    # the segment videos' whole ranges do not count: misaligned video starts between segments do not matter
    req = _mixed(120, ("seg",), lane=2, pcm_off=np.arange(121) * (30 * FR + 8))
    assert _plan(**req)["n_sub"] == [3]


def _variant_tables():
    from test_gpu_vad_exact import VARIANTS
    if not _TABLES:
        from test_gpu_seg_exact import auditok_layout, energy_layout
        for fr, geo, _, cpl in VARIANTS.values():
            if (fr, geo, cpl) not in _TABLES:
                _TABLES[(fr, geo, cpl)] = (energy_layout(fr, geo, cpl), auditok_layout(fr, geo))
    return _TABLES


_TABLES = {}


def test_segment_launch_kernel_per_variant(built):
    """Each row of tests/test_gpu_seg_exact.py's kernel table reaches that kernel: the planner, with the library's own
    lane test, on that module's tables (energy and auditok), names the segment launch's kernel (vad_layout.h)."""
    from test_gpu_seg_exact import KERNEL
    from test_gpu_vad_exact import VARIANTS
    tables = _variant_tables()
    seen = set()
    for variant, (fr, geo, env, cpl) in VARIANTS.items():
        for det, c in enumerate(tables[(fr, geo, cpl)]):
            req = dict(pcm_off=c["pcm_off"], track_video=c["track_video"], cue_start=c["cue_start"],
                       cue_end=c["cue_end"], cue_off=c["cue_off"], ratios=[1.0], frame_rate=fr, detector=det,
                       chunk_samples=c.get("chunk", 0), lane=3, **c["seg"])
            layout = {"B2_VAD_LAYOUT": env["B2_VAD_LAYOUT"]} if "B2_VAD_LAYOUT" in env else {"B2_VAD_LAYOUT": ""}
            p = _plan(env=layout, **req)
            assert p["status"] == 0, (variant, p["err"])
            kernel, g, got_cpl = p["seg_kernel"]
            assert kernel == KERNEL[variant], (variant, det, p["seg_kernel"])
            if kernel == 1:   # the lane-group vector path at the chunks per lane of test_gpu_vad_exact's table
                assert got_cpl == cpl and c["fpw"] // 8 == g * cpl, (variant, det, p["seg_kernel"])
            seen.add(kernel)
    assert seen == {0, 1, 2}
    # the decision looks at starts only: a lane table stays lane-eligible with ragged ends, and one start off a
    # multiple of 8 moves it to the 16-bit path
    c = tables[(16000, "aligned", 5)][0]
    assert any(int(h) % 8 for h in c["seg"]["seg_hi"])
    req = dict(pcm_off=c["pcm_off"], track_video=c["track_video"], cue_start=c["cue_start"], cue_end=c["cue_end"],
               cue_off=c["cue_off"], ratios=[1.0], frame_rate=16000, lane=3, **dict(c["seg"]))
    req["seg_lo"] = np.array(req["seg_lo"])
    req["seg_lo"][3] += 1
    assert _plan(env={"B2_VAD_LAYOUT": ""}, **req)["seg_kernel"][0] == 2


# ---------------------------------------------------------------- seg_ref_kernel on the CPU

def _emul_kernel(L, run_lo, run_src, scratch, packed):
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.bin"), os.path.join(d, "out.bin")
        with open(src, "wb") as f:
            f.write(np.array([L, len(run_lo), len(scratch)], dtype=np.int64).tobytes() + np.int32(packed).tobytes())
            f.write(np.asarray(run_lo, dtype=np.int64).tobytes() + np.asarray(run_src, dtype=np.int64).tobytes())
            f.write(np.asarray(scratch, dtype=np.float32).tobytes())
        subprocess.check_call([EMUL, "kernel", src, dst])
        raw = np.fromfile(dst, dtype=np.uint8)
        return int(raw[:8].view(np.int64)[0]), raw[8:].view(np.uint32 if packed else np.float32)


def _runs_from(L, segs):
    """Owned-frame runs and scratch of segments [(begin, values)] written in order, frame by frame."""
    owner = np.full(L, -1, dtype=np.int64)
    want = np.zeros(L, dtype=np.float32)
    scratch, base = [], 0
    for b, vals in segs:
        e = min(b + len(vals), L)
        if e > b:
            owner[b:e] = base + np.arange(e - b)
            want[b:e] = vals[: e - b]
        scratch.append(np.asarray(vals, dtype=np.float32))
        base += len(vals)
    lo, src = [], []
    for f in range(L):
        same = f > 0 and ((owner[f] < 0 and owner[f - 1] < 0) or (owner[f - 1] >= 0 and owner[f] == owner[f - 1] + 1))
        if not same:
            lo.append(f)
            src.append(int(owner[f]))
    return lo, src, (np.concatenate(scratch) if scratch else np.zeros(0, np.float32)), want


@pytest.mark.parametrize("L", [0, 1, 31, 32, 33, 257, 8191, 8192, 8193, 20000])
def test_emulated_kernel(built, L):
    from oracle import sig_oracle
    rng = np.random.RandomState(L)
    segs = []
    for b in sorted(rng.randint(0, max(L, 1), 4)):
        segs.append((int(b), rng.choice(np.float32([1.0, 0.0, 0.3, -0.5]), rng.randint(1, 3000))))
    lo, src, scr, want = _runs_from(L, segs)
    for packed in (0, 1):
        first, body = _emul_kernel(L, lo, src, scr, packed)
        pos = np.flatnonzero(want > 0)
        assert first == (int(pos[0]) if len(pos) else -1), (L, packed)
        if packed:
            assert np.array_equal(body, sig_oracle.packed_words(want)) and len(body) == (L + 31) // 32
        else:
            assert np.array_equal(body, want), L


def test_emulated_kernel_without_speech(built):
    first, body = _emul_kernel(5000, [0, 100, 200], [-1, 0, -1], np.full(100, -0.5, np.float32), 0)
    assert first == -1 and body[100:200].tolist() == [-0.5] * 100 and not body[:100].any() and not body[200:].any()
