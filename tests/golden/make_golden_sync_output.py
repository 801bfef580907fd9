#!/usr/bin/env python
"""Generate tests/golden/sync_output.json by running the REAL reference's try_sync on prepared aligner answers.

Run where a checkout of the reference is available (FFSUBSYNC_REFERENCE names it; the tests only
read the fixture this writes):   FFSUBSYNC_REFERENCE=<checkout> python tests/golden/make_golden_sync_output.py

The reference is imported the way make_golden.py imports it, plus ffsubsync.ffsubsync itself (its version
module stubbed).  Per scenario: get_srt_pipe_maker builds (parse, scale) pipelines over in-memory cues,
get_framerate_ratios_to_try returns the scenario's list, MaxScoreAligner is a fake returning the scenario's
(score, offset, candidate) the way the reference's tests/test_quality_gate.py fakes it (or raising
FailedToFindAlignmentException), and GenericSubtitlesFile.write_file, SubtitleShifter and
assess_alignment_quality are wrapped to record what is written, what the shift produced and the gate's reasons.
Nothing is copied: the reference's own code computes every expected value written below.
"""
import argparse
import importlib
import json
import os
import sys
import types
from datetime import timedelta

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import jf, load_reference  # noqa: E402

US = timedelta(microseconds=1)
GRID = [24.0 / 23.976, 25.0 / 23.976, 25.0 / 24.0, 23.976 / 24.0, 23.976 / 25.0, 24.0 / 25.0]

# cue times as a parser hands them over (seconds; the pipeline parses them through timedelta)
BASIC = [(10.0, 11.0), (20.0, 21.0)]
MIXED = [(0.0, 0.5), (1.234567, 2.000001), (59.999999, 61.0), (3599.5, 3600.25), (14399.999999, 14400.0),
         (0.000001, 0.000003), (7.0000005, 8.0000015)]
HALF = [(0.000001, 0.000003), (0.000005, 0.000007), (1.000001, 2.000003), (0.5, 1.5), (2.5, 3.5), (4.000001, 4.5)]
FOUR_H = [(14400.0, 14401.5), (14399.123456, 14405.654321), (3.0, 4.0)]
DEFAULTS = dict(min_score=0.0, quality_max_offset_seconds=30.0, max_framerate_deviation=0.1)


def sc(name, cues, ratios, score, offset, k, gss_ratio=None, fail=False, gate=False, apply=0.0, suppress=None,
       **thresholds):
    """One try_sync run: ratios is the framerate list of get_framerate_ratios_to_try (None = the search), the
    candidate list is [1.0] + the grid; k indexes it (len = the search's point gss_ratio)."""
    th = dict(DEFAULTS)
    th.update(thresholds)
    return dict(name=name, cues=cues, ratios=ratios, score=score, offset=offset, k=k, gss_ratio=gss_ratio, fail=fail,
                gate=gate, apply_offset_seconds=apply, suppress=suppress, **th)


SCENARIOS = [
    # tests/test_quality_gate.py's three try_sync scenarios (offset in samples at 100 Hz)
    sc("qg_low_quality_written_original", BASIC, [], 500.0, 30000, 0, gate=True),
    sc("qg_applied_when_acceptable", BASIC, [], 500.0, 500, 0, gate=True),
    sc("qg_ignored_without_flag", BASIC, [], 500.0, 30000, 0, gate=False),
    # threshold edges
    sc("score_equals_min", BASIC, [], 0.0, 100, 0, gate=True),
    sc("score_below_min", BASIC, [], -1e-300, 100, 0, gate=True),
    sc("score_min_100", MIXED, [], 99.9, 100, 0, gate=True, min_score=100.0),
    sc("offset_equals_max", BASIC, [], 5.0, 3000, 0, gate=True),
    sc("offset_equals_max_negative", BASIC, [], 5.0, -3000, 0, gate=True),
    sc("offset_just_over_max", BASIC, [], 5.0, 3001, 0, gate=True),
    sc("offset_apply_over_max", BASIC, [], 5.0, 2990, 0, gate=True, apply=0.2),
    sc("scale_1.1", MIXED, [1.1, 0.9], 5.0, 0, 1, gate=True),
    sc("scale_0.9", MIXED, [1.1, 0.9], 5.0, 0, 2, gate=True),
    sc("scale_25_23.976_default", MIXED, GRID, 5.0, -250, 2, gate=True),
    sc("scale_25_23.976_tight", MIXED, GRID, 5.0, -250, 2, gate=True, max_framerate_deviation=0.01),
    sc("scale_24_25_tight", MIXED, GRID, 5.0, 250, 6, gate=True, max_framerate_deviation=0.04),
    sc("all_three_reasons", MIXED, [1.5], -5.0, 9900, 1, gate=True),
    sc("nan_thresholds", BASIC, [], 5.0, 100, 0, gate=True, min_score=float("nan"),
       quality_max_offset_seconds=float("nan"), max_framerate_deviation=float("nan")),
    # negative score: not successful, still written
    sc("negative_score_written", MIXED, GRID, -3.5, 1234, 3),
    sc("negative_score_gated", MIXED, GRID, -3.5, 1234, 3, gate=True),
    # suppression
    sc("suppress_none", BASIC, [], 5.0, -500, 0, suppress=None),
    sc("suppress_zero", BASIC, [], 5.0, -500, 0, suppress=0.0),
    sc("suppress_negative_zero", BASIC, [], 5.0, -500, 0, suppress=-0.0),
    sc("suppress_positive_held", BASIC, [], 5.0, 100, 0, suppress=2.0),
    sc("suppress_positive_equal", BASIC, [], 5.0, 200, 0, suppress=2.0),
    sc("suppress_negative_passes", BASIC, [], 5.0, -100, 0, suppress=-2.0),
    sc("suppress_negative_held", BASIC, [], 5.0, -300, 0, suppress=-2.0),
    sc("suppress_nan", BASIC, [], 5.0, 100, 0, suppress=float("nan")),
    sc("suppress_negative_score", BASIC, [], -5.0, 100, 0, suppress=2.0),
    sc("gated_before_suppression", BASIC, [], -5.0, 100, 0, gate=True, suppress=2.0),
    # negative and zero-crossing shifts, apply_offset_seconds
    sc("shift_negative", MIXED, [], 5.0, -1500, 0),
    sc("shift_zero_crossing", MIXED, GRID, 5.0, -123, 4),
    sc("apply_offset", MIXED, GRID, 5.0, 77, 1, apply=0.1),
    sc("apply_offset_negative", MIXED, GRID, 5.0, -77, 5, apply=-2.345678),
    sc("apply_offset_half_us", HALF, [], 5.0, 3, 0, apply=0.0000005),
    sc("apply_offset_third", HALF, [], 5.0, -1, 0, apply=1.0 / 3.0),
    # half-microsecond products, 4-hour times
    sc("half_us_products", HALF, [0.5, 1.5, 2.5], 5.0, 0, 1),
    sc("half_us_products_odd", HALF, [0.5, 1.5, 2.5], 5.0, 1, 3),
    sc("four_hours", FOUR_H, GRID, 5.0, 6000, 2),
    sc("four_hours_gss", FOUR_H, GRID + [None], 5.0, -4321, 7, gss_ratio=1.0416666666666667),
    # the search's point wins
    sc("gss", MIXED, GRID + [None], 5.0, 42, 7, gss_ratio=0.9591036734526315),
    sc("gss_gated", MIXED, GRID + [None], 5.0, 42, 7, gss_ratio=1.0816, gate=True, max_framerate_deviation=0.05),
    # a failed alignment
    sc("failed", MIXED, GRID, 0.0, 0, 0, fail=True),
    sc("failed_gated", MIXED, GRID, 0.0, 0, 0, fail=True, gate=True),
]

# tests/test_quality_gate.py's assess_alignment_quality cases, plus the exact edges
ASSESS = [
    (500.0, 3.0, 1.0, 0.0, 30.0, 0.1), (-1.0, 3.0, 1.0, 0.0, 30.0, 0.1), (500.0, 45.0, 1.0, 0.0, 30.0, 0.1),
    (500.0, 3.0, 25.0 / 24.0, 0.0, 30.0, 0.1), (500.0, 3.0, 25.0 / 23.976, 0.0, 30.0, 0.1),
    (500.0, 3.0, 24.0 / 25.0, 0.0, 30.0, 0.1), (500.0, 3.0, 1.05, 0.0, 30.0, 0.1), (500.0, 3.0, 0.95, 0.0, 30.0, 0.1),
    (500.0, 3.0, 25.0 / 24.0, 0.0, 30.0, 0.01), (-5.0, 99.0, 1.5, 0.0, 30.0, 0.1),
    (0.0, 30.0, 1.1, 0.0, 30.0, 0.1), (0.0, -30.0, 0.9, 0.0, 30.0, 0.1), (-0.04, -30.05, 1.1000001, 0.0, 30.0, 0.1),
    (100.0, 1.0, 1.0, 100.0, 30.0, 0.1), (99.95, 1.0, 1.0, 100.0, 30.0, 0.1),
]


def load_try_sync():
    mods, _ = load_reference()
    version = types.ModuleType("ffsubsync.version")
    version.get_version = lambda: "0"
    version.make_version_tuple = lambda *a, **k: (0,)
    sys.modules["ffsubsync.version"] = version
    return mods, importlib.import_module("ffsubsync.ffsubsync")


def run_scenario(mods, fs, s):
    gs = mods["generic_subtitles"]
    st = mods["subtitle_transformers"]
    shim = mods["sklearn_shim"]
    subs_in = [gs.GenericSubtitle(timedelta(seconds=a), timedelta(seconds=b), "x") for a, b in s["cues"]]

    class Parse(shim.TransformerMixin):
        def fit(self, *_):
            self.subs_ = gs.GenericSubtitlesFile(list(subs_in), sub_format="srt", encoding="utf-8")
            return self

        def transform(self, *_):
            return self.subs_

    def maker(scale_factor):
        if scale_factor is None:   # the search's entry: a callable, as the reference's maker returns
            return lambda r: maker(r)
        return shim.Pipeline([("parse", Parse()), ("scale", st.SubtitleScaler(scale_factor))])

    rec = {"written": None, "shifted": None, "reasons": None}

    class Fake:
        def __init__(self, *a, **k):
            pass

        def fit_transform(self, refstring, subpipes):
            if s["fail"]:
                raise mods["aligners"].FailedToFindAlignmentException("no alignment")
            pipe = subpipes[s["k"]]
            if callable(pipe):
                pipe = pipe(s["gss_ratio"]).fit(None)
            return (s["score"], s["offset"]), pipe

    class Shifter(st.SubtitleShifter):
        def fit(self, subs, *a):
            super().fit(subs, *a)
            rec["shifted"] = [[(c.start // US), (c.end // US)] for c in self.subs_]
            return self

    real_assess = fs.assess_alignment_quality

    def assess(*a, **k):
        rec["reasons"] = real_assess(*a, **k)
        return rec["reasons"]

    def write_file(self, fname):
        rec["written"] = [[(c.start // US), (c.end // US)] for c in self.subs_]

    saved = (fs.get_srt_pipe_maker, fs.get_framerate_ratios_to_try, fs.MaxScoreAligner, fs.SubtitleShifter,
             fs.assess_alignment_quality, gs.GenericSubtitlesFile.write_file)
    fs.get_srt_pipe_maker = lambda args, srtin: maker
    fs.get_framerate_ratios_to_try = lambda args: list(s["ratios"])
    fs.MaxScoreAligner = Fake
    fs.SubtitleShifter = Shifter
    fs.assess_alignment_quality = assess
    gs.GenericSubtitlesFile.write_file = write_file
    try:
        args = argparse.Namespace(
            srtin=["in.srt"], srtout="out.srt", skip_sync=False, skip_infer_framerate_ratio=True, reference="ref.mkv",
            max_offset_seconds=600, apply_offset_seconds=s["apply_offset_seconds"],
            skip_sync_on_low_quality=s["gate"], min_score=s["min_score"],
            quality_max_offset_seconds=s["quality_max_offset_seconds"],
            max_framerate_deviation=s["max_framerate_deviation"], merge_with_reference=False, output_encoding="same",
            suppress_output_if_offset_less_than=s["suppress"], overwrite_input=False, gss=False)
        result = {"retval": 0}
        ok = fs.try_sync(args, types.SimpleNamespace(transform=lambda _: None), result)
    finally:
        (fs.get_srt_pipe_maker, fs.get_framerate_ratios_to_try, fs.MaxScoreAligner, fs.SubtitleShifter,
         fs.assess_alignment_quality, gs.GenericSubtitlesFile.write_file) = saved
    # the cue times as the batched calls receive them: the parsed timedeltas' total_seconds()
    starts = [c.start.total_seconds() for c in subs_in]
    ends = [c.end.total_seconds() for c in subs_in]
    return dict(
        name=s["name"], cue_start=starts, cue_end=ends, ratios=[1.0] + [r for r in s["ratios"] if r is not None],
        gss=any(r is None for r in s["ratios"]), best_score=jf(s["score"]), best_offset=s["offset"],
        best_k=-1 if s["fail"] else s["k"], gss_ratio=jf(s["gss_ratio"]) if s["gss_ratio"] is not None else None,
        gate=s["gate"], apply_offset_seconds=s["apply_offset_seconds"], min_score=jf(s["min_score"]),
        quality_max_offset_seconds=jf(s["quality_max_offset_seconds"]),
        max_framerate_deviation=jf(s["max_framerate_deviation"]),
        suppress=None if s["suppress"] is None else jf(s["suppress"]),
        sync_was_successful=bool(ok), written=rec["written"], shifted=rec["shifted"], reasons=rec["reasons"],
        offset_seconds=jf(result["offset_seconds"]) if "offset_seconds" in result else None,
        framerate_scale_factor=jf(result["framerate_scale_factor"]) if "framerate_scale_factor" in result else None)


def main():
    mods, fs = load_try_sync()
    out = {"scenarios": [run_scenario(mods, fs, s) for s in SCENARIOS], "assess": []}
    for score, off, scale, ms, mo, md in ASSESS:
        out["assess"].append(dict(args=[score, off, scale, ms, mo, md],
                                  reasons=fs.assess_alignment_quality(score, off, scale, min_score=ms,
                                                                      max_offset_seconds=mo,
                                                                      max_framerate_deviation=md)))
    path = os.path.join(HERE, "sync_output.json")
    with open(path, "w") as fh:
        json.dump(out, fh, indent=1)
    print("wrote %s: %d scenarios, %d assessments" % (path, len(out["scenarios"]), len(out["assess"])))


if __name__ == "__main__":
    main()
