#!/usr/bin/env python
"""Generate the golden fixtures in this directory by running the REAL reference.

Run where a checkout of the reference is available (FFSUBSYNC_REFERENCE names it; the tests only
read the fixtures this writes):   FFSUBSYNC_REFERENCE=<checkout> python tests/golden/make_golden.py

The reference package cannot be imported normally here (ffmpeg-python, srt, pysubs2, tqdm
wheels are absent), so the hot-path modules are imported by path behind stub modules for the
missing third-party packages (SURVEY.md section 8c).  Nothing is copied: the reference's own
code computes every expected value written below.
"""
import importlib
import json
import os
import sys
import types
from datetime import timedelta

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402

REF = os.environ.get("FFSUBSYNC_REFERENCE", "ffsubsync-reference")  # checkout of smacke/ffsubsync v0.5.0


def load_reference():
    pkg = types.ModuleType("ffsubsync")
    pkg.__path__ = [os.path.join(REF, "ffsubsync")]
    sys.modules["ffsubsync"] = pkg
    ffmpeg = types.ModuleType("ffmpeg")
    ffmpeg.probe = lambda *a, **k: {"format": {"duration": "0"}}
    sys.modules["ffmpeg"] = ffmpeg
    srt = types.ModuleType("srt")

    class Subtitle:  # the only attribute the hot path reads is .content
        def __init__(self, index=0, start=None, end=None, content=""):
            self.index, self.start, self.end, self.content = index, start, end, content

    srt.Subtitle = Subtitle
    sys.modules["srt"] = srt
    pysubs2 = types.ModuleType("pysubs2")
    for name in ("SSAEvent", "SSAFile", "SSAStyle"):
        setattr(pysubs2, name, type(name, (), {}))
    sys.modules["pysubs2"] = pysubs2
    if "tqdm" not in sys.modules:
        try:
            import tqdm  # noqa: F401
        except ImportError:
            sys.modules["tqdm"] = types.ModuleType("tqdm")
    for missing in ("chardet", "charset_normalizer", "cchardet", "faust_cchardet"):
        try:
            importlib.import_module(missing)
        except ImportError:
            sys.modules[missing] = types.ModuleType(missing)
    mods = {}
    for name in ("aligners", "golden_section_search", "sklearn_shim", "constants",
                 "generic_subtitles", "subtitle_transformers", "speech_transformers"):
        mods[name] = importlib.import_module("ffsubsync." + name)
    return mods, srt


def jf(x):
    """JSON-safe float (keeps -inf / nan as strings)."""
    x = float(x)
    if np.isfinite(x):
        return x
    return repr(x)


def gen_alignment(mods, out):
    al = mods["aligners"]
    kats = []
    # tests/test_alignment.py:7-14 (note the test passes (s2, s1) as (ref, sub))
    for sub, ref, off in [("111001", "11001", -1), ("1001", "1001", 0), ("10010", "01001", 1)]:
        got = al.FFTAligner().fit_transform(ref, sub)
        assert got == off
        score, off2 = al.FFTAligner().fit_transform(ref, sub, get_score=True)
        kats.append({"ref": ref, "sub": sub, "mos": None, "offset": int(off2), "score": jf(score)})
    # SURVEY.md section 8c extra goldens
    extra = [([0, 1, 1, 0, 1], [0, 0.96, 0.96, 0], None), ([1, 1, 1, 1], [0, 0, 0], None)]
    for ref, sub, mos in extra:
        score, off = al.FFTAligner(mos).fit_transform(ref, sub, get_score=True)
        kats.append({"ref": ref, "sub": sub, "mos": mos, "offset": int(off), "score": jf(score)})
    rng = np.random.RandomState(7)
    ref, sub = rng.rand(50), rng.rand(40)
    for mos in (0, 1, 5, 20, 45, 80, 87, 88, 127, 200, 100000):
        score, off = al.FFTAligner(mos).fit_transform(ref, sub, get_score=True)
        kats.append({"ref": list(map(float, ref)), "sub": list(map(float, sub)), "mos": mos,
                     "offset": int(off), "score": jf(score)})
    out["kats"] = kats

    small = []
    for seed in range(240):
        ref, sub, mos = cases.small_align_case(seed)
        score, off = al.FFTAligner(mos).fit_transform(ref, sub, get_score=True)
        small.append({"seed": seed, "mos": mos, "offset": int(off), "score": jf(score)})
    out["small"] = small

    shifted = []
    for n in (6000, 60000, 360000, 720000, 1440000):
        ref, sub = cases.shifted_pair(n)
        for mos in (6000, None) + ((100000,) if n >= 360000 else ()):
            score, off = al.FFTAligner(mos).fit_transform(ref, sub, get_score=True)
            shifted.append({"n": n, "mos": mos, "offset": int(off), "score": jf(score)})
    out["shifted"] = shifted

    # wide-window cases (FFTAligner's default max_offset_samples=None and masks wider than a few
    # overlap-save tiles): lopsided lengths, non-binary levels, lengths that straddle a power of two
    wide = []
    for c in cases.WIDE_CASES:
        ref, sub = cases.wide_pair(**c)
        for mos in c["mos_list"]:
            score, off = al.FFTAligner(mos).fit_transform(ref, sub, get_score=True)
            wide.append({"case": c, "mos": mos, "offset": int(off), "score": jf(score)})
    out["wide"] = wide

    empties = []
    for ref, sub in (([], [1, 0, 1]), ([1, 0, 1], []), ([], [])):
        try:
            al.FFTAligner().fit(np.array(ref), np.array(sub))
            empties.append({"ref": ref, "sub": sub, "raises": None})
        except al.FailedToFindAlignmentException as e:
            empties.append({"ref": ref, "sub": sub, "raises": str(e)})
    out["empty"] = empties


def gen_multi_segment(mods, out, arrays):
    al, st = mods["aligners"], mods["speech_transformers"]
    sr = 100
    res = []
    for ci, (scale, shift) in enumerate([(1.0, 5.0), (1.0, -8.0), (25.0 / 24.0, 3.0), (24.0 / 25.0, -2.0)]):
        ref_full, sub = cases.multi_segment_case(scale, shift, sr)
        st.ffmpeg.probe = lambda *a, **k: {"format": {"duration": str(len(ref_full) / sr)}}
        t = st.MultiSegmentVideoSpeechTransformer(
            vad="webrtc", sample_rate=sr, frame_rate=48000, non_speech_label=0.0,
            segment_count=8, segment_duration=60)
        t._extract_segment_speech = lambda fname, start: (
            start, ref_full[start * sr:(start + t.segment_duration) * sr])
        t.fit("ref.mkv")
        sparse = t.transform()
        arrays["ms_sparse_%d" % ci] = np.packbits(sparse.astype(np.uint8))
        arrays["ms_sparse_len_%d" % ci] = np.array(len(sparse))
        per_ratio = []
        for sf in cases.ratio_grid():
            a = al.FFTAligner(max_offset_samples=60 * sr)
            a.fit(sparse, cases.scaled_signal(sub, sf), get_score=True)
            score, off = a.transform()
            per_ratio.append({"ratio": float(sf), "score": jf(score), "offset": int(off)})
        (bscore, boff), bidx_pipe = al.MaxScoreAligner(al.FFTAligner, None, sr, 60).fit_transform(
            sparse, [cases.scaled_signal(sub, sf) for sf in cases.ratio_grid()])
        bidx = [i for i, sf in enumerate(cases.ratio_grid())
                if cases.scaled_signal(sub, sf) is not None and
                np.array_equal(cases.scaled_signal(sub, sf), bidx_pipe)][0]
        res.append({"scale": scale, "shift": shift, "per_ratio": per_ratio,
                    "best": {"score": jf(bscore), "offset": int(boff), "index": bidx}})
    out["multi_segment"] = res


def gen_raster(mods, out, srt):
    st, stx, gs = mods["speech_transformers"], mods["subtitle_transformers"], mods["generic_subtitles"]

    class Subs(list):  # stands in for GenericSubtitlesFile: SubtitleScaler only iterates + clones props
        def clone_props_for_subs(self, new_subs):
            return Subs(new_subs)

    def make(starts, ends, contents):
        return Subs(
            gs.GenericSubtitle(timedelta(seconds=float(s)), timedelta(seconds=float(e)),
                               srt.Subtitle(content=c))
            for s, e, c in zip(starts, ends, contents))

    res = []
    # (seed, duration) synthetic cue lists through scaler + rasteriser for the 7-ratio grid
    for seed, dur in ((13, 600.0), (14, 1800.0), (15, 7200.0)):
        starts, ends = cases.synthetic_cues(seed, dur)
        subs = make(starts, ends, ["hello"] * len(starts))
        for ratio in cases.ratio_grid() + [0.9, 1.1, 0.976393, 2.0]:
            for start_seconds in ((0, 7) if seed == 13 else (0,)):
                scaled = stx.SubtitleScaler(ratio).fit(subs).transform()
                tr = st.SubtitleSpeechTransformer(sample_rate=100, start_seconds=start_seconds,
                                                  framerate_ratio=ratio).fit(scaled)
                x = tr.transform()
                levels, rs, re_ = cases.run_lengths(x)
                res.append({"seed": seed, "duration": dur, "ratio": float(ratio),
                            "start_seconds": start_seconds, "length": int(len(x)),
                            "levels": levels, "run_starts": rs, "run_stops": re_,
                            "max_time": jf(tr.max_time_),
                            # quirk: the mixin's __init__ never runs (MRO stops at the Protocol
                            # class), so these attributes only exist once a frame > 0.5 was seen
                            "start_frame": getattr(tr, "start_frame_", None),
                            "end_frame": getattr(tr, "end_frame_", None)})
    out["raster"] = res

    # tests/test_subtitles.py fake_srt timings + tests/test_metadata.py style contents
    starts = [0.178, 2.828, 4.653]
    ends = [2.416, 4.549, 6.062]
    contents = ['<i>Previously on "Your favorite TV show..."</i>', "Oh hi, Mark.",
                "You are tearing me apart, Lisa!"]
    kat = []
    for sr in (10, 20, 100, 300):
        for ss in (0, 2, 4, 6):
            keep = [i for i in range(3) if starts[i] >= ss]
            subs = make([starts[i] for i in keep], [ends[i] for i in keep], [contents[i] for i in keep])
            if not len(subs):
                continue
            tr = st.SubtitleSpeechTransformer(sample_rate=sr, start_seconds=ss).fit(subs)
            levels, rs, re_ = cases.run_lengths(tr.transform())
            kat.append({"sample_rate": sr, "start_seconds": ss, "cue_idx": keep,
                        "length": int(len(tr.transform())), "levels": levels,
                        "run_starts": rs, "run_stops": re_, "max_time": jf(tr.max_time_),
                        "start_frame": getattr(tr, "start_frame_", None),
                        "end_frame": getattr(tr, "end_frame_", None)})
    out["raster_kat"] = {"starts": starts, "ends": ends, "contents": contents, "cases": kat}

    meta_strings = ["[music]", "(door slams)", "<i>[music]</i>", "<i>Hello?</i>", "♪ ♫", "", "   ",
                    "English subtitles", "Tom - Jerry", "plain line", "{\\an8}", "（笑）", "【音乐】x",
                    "<font color='red'>♪</font>", "- Hi. - Hello."]
    out["metadata"] = [{"content": c, "edge": e, "is_metadata": bool(st._is_metadata(c, e))}
                       for c in meta_strings for e in (False, True)]

    # scaler rounding: timedelta(seconds=t*r).total_seconds() for awkward products
    rng = np.random.RandomState(5)
    ts = np.round(rng.uniform(0, 8000, 400), 3)
    rs = rng.choice(cases.ratio_grid() + [0.9, 1.1, 0.976393, 1.0236067977], 400)
    out["scale_roundtrip"] = [
        {"t": float(t), "r": float(r), "scaled": timedelta(seconds=float(t) * float(r)).total_seconds()}
        for t, r in zip(ts, rs)]


def gen_gss(mods, out):
    g, al = mods["golden_section_search"], mods["aligners"]
    calls = []

    def f(x, last):
        calls.append((float(x), bool(last)))
        return (x - 1.0417) ** 2

    interval = g.gss(f, al.MIN_FRAMERATE_RATIO, al.MAX_FRAMERATE_RATIO)
    out["gss_quadratic"] = {"calls": calls, "interval": [float(interval[0]), float(interval[1])]}

    # fit_gss on real (small) data: subpipe_maker(ratio) -> object with fit_transform(srtin)
    ref_full, sub = cases.multi_segment_case(25.0 / 24.0, 3.0)
    evals = []

    class Pipe:
        def __init__(self, ratio):
            self.ratio = ratio

        def fit_transform(self, _):
            return cases.scaled_signal(sub, self.ratio)

    def maker(ratio):
        evals.append(float(ratio))
        return Pipe(ratio)

    m = al.MaxScoreAligner(al.FFTAligner, None, 100, 60)
    m.fit(ref_full, [maker])
    (score, off), pipe = m.transform()
    out["gss_fit"] = {"evals": evals, "score": jf(score), "offset": int(off),
                      "ratio": float(pipe.ratio)}


def gen_maxscore(mods, out):
    al = mods["aligners"]
    res = []
    grid = cases.ratio_grid()
    for seed in range(6):
        rng = np.random.RandomState(300 + seed)
        n = 30000
        true_k = int(rng.randint(0, len(grid)))
        shift = int(rng.randint(-3000, 3001))
        base = (rng.rand(n) > 0.55).astype(float)
        sub0 = base.copy()
        # reference = sub warped by grid[true_k] then shifted, with 10 % flips
        ref = cases.scaled_signal(sub0, grid[true_k])
        ref = np.roll(ref, shift)
        flip = rng.rand(len(ref)) < 0.10
        ref = np.where(flip, 1.0 - ref, ref)
        subs = [cases.scaled_signal(sub0, r) * min(1.0 / r, 1.0) for r in grid]
        m = al.MaxScoreAligner(al.FFTAligner, None, 100, 60).fit(ref, subs)
        per = [{"score": jf(s[0][0]), "offset": int(s[0][1])} for s in m._scores]
        (bs, bo), bp = m.transform()
        bidx = [i for i, s in enumerate(subs) if s is bp][0]
        res.append({"seed": seed, "true_k": true_k, "shift": shift, "per_ratio": per,
                    "best": {"score": jf(bs), "offset": int(bo), "index": bidx}})
    out["maxscore"] = res
    # failure: nothing within max offset -> exception text
    m = al.MaxScoreAligner(al.FFTAligner(max_offset_samples=None), None, 100, 0.01)
    ref, sub = cases.shifted_pair(2000, 300)
    m.fit(ref, [sub])
    try:
        m.transform()
        out["maxscore_fail"] = None
    except al.FailedToFindAlignmentException as e:
        out["maxscore_fail"] = str(e)


def gen_segment_starts(mods, out):
    """MultiSegmentVideoSpeechTransformer._segment_starts (speech_transformers.py:812-830) and the
    sparse-signal assembly of .fit (:855-895) with a stubbed per-segment extractor."""
    st = mods["speech_transformers"]
    rows = []
    for total in (40.0, 60.0, 61.0, 119.5, 120.0, 600.0, 900.0, 3600.25, 7200.0, 95.0, 150.0):
        for count in (1, 3, 6, 8):
            for dur in (10, 60):
                for skip in (False, True):
                    t = st.MultiSegmentVideoSpeechTransformer(
                        vad="webrtc", sample_rate=100, frame_rate=48000, non_speech_label=0.0,
                        segment_count=count, segment_duration=dur, skip_intro_outro=skip)
                    rows.append({"total": total, "count": count, "duration": dur, "skip": skip,
                                 "starts": [int(v) for v in t._segment_starts(total)]})
    out["segment_starts"] = rows
    # assembly: segment s returns the constant (s % 7 + 1) / 8 for dur seconds (last one clipped by
    # the array end), one segment fails
    asm = []
    for total, count, dur in ((120.0, 3, 10), (325.37, 5, 30), (59.0, 4, 60)):
        st.ffmpeg.probe = lambda *a, **k: {"format": {"duration": str(total)}}
        t = st.MultiSegmentVideoSpeechTransformer(
            vad="subs_then_webrtc", sample_rate=100, frame_rate=48000, non_speech_label=0.0,
            segment_count=count, segment_duration=dur)
        starts = t._segment_starts(total)
        failing = starts[1] if len(starts) > 1 else None

        def extract(fname, start, _dur=dur, _failing=failing):
            if start == _failing:
                raise RuntimeError("boom")
            return start, np.full(_dur * 100, (start % 7 + 1) / 8.0)

        t._extract_segment_speech = extract
        t.fit("ref.mkv")
        x = t.transform()
        levels, rs, re = cases.run_lengths(x)
        asm.append({"total": total, "count": count, "duration": dur, "vad": t.vad, "len": int(len(x)),
                    "failing": failing, "runs": [[int(a), int(b), float(x[a])] for a, b in zip(rs, re)]})
    out["segment_assembly"] = asm


def gen_misc(mods, out):
    st = mods["speech_transformers"]
    mix = st.ComputeSpeechFrameBoundariesMixin()
    rows = []
    for arr in ([0, 0, 1, 1, 0, 1, 0], [0, 0, 0], [0.5, 0.5], [0.96, 0, 0.96], [1.0]):
        m = st.ComputeSpeechFrameBoundariesMixin()
        m.fit_boundaries(np.array(arr, dtype=float))
        rows.append({"x": arr, "start": m.start_frame_, "end": m.end_frame_, "num_frames": m.num_frames})
    out["boundaries"] = rows
    del mix


def main():
    mods, srt = load_reference()
    out, arrays = {}, {}
    gen_alignment(mods, out)
    gen_multi_segment(mods, out, arrays)
    gen_raster(mods, out, srt)
    gen_gss(mods, out)
    gen_maxscore(mods, out)
    gen_segment_starts(mods, out)
    gen_misc(mods, out)
    out["_meta"] = {"reference": "smacke/ffsubsync (v0.5.0)",
                    "numpy": np.__version__, "python": sys.version.split()[0],
                    "generator": "tests/golden/make_golden.py"}
    with open(os.path.join(HERE, "golden.json"), "w") as fh:
        json.dump(out, fh, indent=0, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, "golden_arrays.npz"), **arrays)
    print("wrote golden.json (%d top-level keys) and golden_arrays.npz (%d arrays)"
          % (len(out), len(arrays)))


if __name__ == "__main__":
    main()
