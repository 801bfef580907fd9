#!/usr/bin/env python
"""Generate tests/golden/pgs.json by running the REAL reference's PGS reference path (--pgs-ref-stream).

Run where a checkout of the reference is available (FFSUBSYNC_REFERENCE names it; the tests only
read the fixture this writes):   FFSUBSYNC_REFERENCE=<checkout> python tests/golden/make_golden_pgs.py

The reference is imported the way make_golden.py imports it; its ffprobe call (ffmpeg.probe and
ffmpeg_bin_path) is stubbed to return prepared packet / stream dicts.  Nothing is copied: the
reference's own code computes every expected value written below.
"""
import json
import os
import sys
from datetime import timedelta

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
from make_golden import jf, load_reference  # noqa: E402


def packet(pts, dur, size):
    return {"pts_time": str(pts), "duration_time": "N/A" if dur is None else str(dur), "size": str(size)}


# the reference's tests/test_pgs.py packet lists, plus unparsable values and the size boundary
PACKET_CASES = [
    ("basic", [packet(1.0, 2.5, 1000), packet(5.0, 1.0, 800)]),
    ("clear_event", [packet(1.0, 2.0, 1000), packet(3.0, 0.001, 30)]),
    ("na_duration", [packet(1.0, None, 1000), packet(5.0, 2.0, 900)]),
    ("nothing_usable", [packet(1.0, None, 1000), packet(2.0, 1.0, 20)]),
    ("empty", []),
    ("missing_fields", [{"pts_time": "1.0", "duration_time": "2.0"}, {"pts_time": "3.0", "size": "500"},
                        {"duration_time": "1.0", "size": "500"}, packet(10.0, 1.0, 200)]),
    ("unparsable", [{"pts_time": "x", "duration_time": "1.0", "size": "100"},
                    {"pts_time": "1.0", "duration_time": "1.0", "size": "1.5"}, packet(2.0, 0.5, 51),
                    packet(3.0, 0.5, 50)]),
    ("negative_duration", [packet(4.0, -1.0, 60), packet(0.5, 0.25, 60)]),
]

STREAM_CASES = [
    ("first_pgs", {"streams": [{"codec_type": "video", "index": 0}, {"codec_type": "audio", "index": 1},
                               {"codec_type": "subtitle", "codec_name": "hdmv_pgs_subtitle", "index": 2}]}),
    ("after_text", {"streams": [{"codec_type": "subtitle", "codec_name": "subrip", "index": 2},
                                {"codec_type": "subtitle", "codec_name": "ass", "index": 3},
                                {"codec_type": "subtitle", "codec_name": "hdmv_pgs_subtitle", "index": 4},
                                {"codec_type": "subtitle", "codec_name": "hdmv_pgs_subtitle", "index": 5}]}),
    ("none", {"streams": [{"codec_type": "subtitle", "codec_name": "subrip", "index": 2}]}),
    ("no_streams", {}),
]


def signal_cases():
    rng = np.random.RandomState(31)
    two_h = []
    t = 3.0
    while len(two_h) < 1500:
        d = float(rng.uniform(0.5, 6.0))
        two_h.append((round(t, 3), round(t + d, 3)))
        t += d + float(rng.exponential(1.4))
    return [
        ("edges", [(0.125, 0.285), (7200.0, 7200.125), (-0.015, 0.125), (1234.565, 1240.0)]),
        ("negative_zero_overlap_unsorted", [(30.0, 31.5), (10.0, 12.0), (11.0, 13.25), (20.0, 20.0),
                                            (25.0, 24.0), (-3.0, 2.005), (40.0, 40.004), (40.006, 40.01)]),
        ("end_clamp", [(1.0, 2.0), (5.0, 9.995)]),
        ("max_end_negative", [(-5.0, -0.015)]),
        ("max_end_tiny_negative", [(-1.0, -0.005)]),
        ("max_end_exact_negative", [(-2.0, -0.02)]),
        ("negative_length", [(-1.0, -0.05), (-0.5, -0.3)]),
        ("single", [(0.0, 0.0)]),
        ("two_hours", [(a, min(b, 7200.0)) for a, b in two_h if a < 7190.0]),
    ]


class _Pipe:
    """A subtitle pipeline at one ratio: SubtitleScaler + SubtitleSpeechTransformer, as try_sync builds it."""
    def __init__(self, st, stx, r):
        self.st, self.stx, self.r = st, stx, r

    def transform(self, subs, *_):
        return self.fit_transform(subs)

    def fit_transform(self, subs, *_):
        scaled = self.stx.SubtitleScaler(self.r).fit(subs).transform()
        return self.st.SubtitleSpeechTransformer(100, 0, self.r).fit(scaled).transform()


def gen_pgs(mods, out, srt):
    st, stx, gs, al = (mods["speech_transformers"], mods["subtitle_transformers"], mods["generic_subtitles"],
                       mods["aligners"])
    probe_result = {}
    st.ffmpeg_bin_path = lambda *a, **k: "ffprobe"
    st.ffmpeg.probe = lambda *a, **k: probe_result["value"]

    rows = []
    for name, pk in PACKET_CASES:
        probe_result["value"] = {"packets": pk}
        got = st._get_pgs_timings_via_ffprobe("x.mkv", "0:s:0")
        rows.append({"name": name, "packets": pk, "timings": None if got is None else [list(t) for t in got]})
    out["pgs_packets"] = rows

    rows = []
    for name, probe in STREAM_CASES:
        probe_result["value"] = probe
        rows.append({"name": name, "probe": probe, "stream": st.find_pgs_stream("x.mkv")})
    out["pgs_streams"] = rows

    # PGSSpeechTransformer.fit, its packet-timing step answering with the exact intervals (the packet parsing is
    # pinned above)
    saved_timings = st._get_pgs_timings_via_ffprobe

    def fit(intervals, ss):
        st._get_pgs_timings_via_ffprobe = lambda *a, **k: list(intervals)
        t = st.PGSSpeechTransformer(sample_rate=100, start_seconds=ss, ref_stream="s:0")
        try:
            t.fit("x.mkv")
        except ValueError as e:
            return None, str(e)
        return np.asarray(t.transform(), dtype=float), None

    rows = []
    sig_2h = None
    for name, iv in signal_cases():
        timings = [(float(a), float(b)) for a, b in iv]
        for ss in (0, 3, -2):
            x, err = fit(iv, ss)
            row = {"name": name, "start_seconds": ss, "starts": [a for a, _ in timings],
                   "ends": [b for _, b in timings], "error": err}
            if x is not None:
                levels, rs, re_ = cases.run_lengths(x)
                row.update(length=int(len(x)), levels=levels, run_starts=rs, run_stops=re_)
                if name == "two_hours" and ss == 0:
                    sig_2h = x
            rows.append(row)
    out["pgs_signals"] = rows
    st._get_pgs_timings_via_ffprobe = saved_timings

    # an input track against the 2 h PGS reference: its intervals scaled by 25/24 and delayed by 3.5 s
    two_h = [r for r in rows if r["name"] == "two_hours" and r["start_seconds"] == 0][0]
    true_r = 25.0 / 24.0
    in_starts = [round(a / true_r + 3.5, 3) for a in two_h["starts"]]
    in_ends = [round(b / true_r + 3.5, 3) for b in two_h["ends"]]
    class Subs(list):
        def clone_props_for_subs(self, new_subs):
            return Subs(new_subs)

    subs = Subs(gs.GenericSubtitle(timedelta(seconds=a), timedelta(seconds=b), srt.Subtitle(content="s"))
                for a, b in zip(in_starts, in_ends))
    grid = cases.ratio_grid()
    m = al.MaxScoreAligner(al.FFTAligner, subs, 100, 60).fit(sig_2h, [_Pipe(st, stx, r) for r in grid])
    per = [{"score": jf(sc[0][0]), "offset": int(sc[0][1])} for sc in m._scores]
    (bs, bo), bp = m.transform()
    out["pgs_maxscore"] = {"in_starts": in_starts, "in_ends": in_ends, "max_offset_seconds": 60, "per_ratio": per,
                           "best": {"score": jf(bs), "offset": int(bo),
                                    "index": [i for i, (_, p) in enumerate(m._scores) if p is bp][0]}}
    # --gss: the grid plus the golden-section search (try_sync's list with the maker last)
    g = al.MaxScoreAligner(al.FFTAligner, subs, 100, 60)
    g.fit(sig_2h, [_Pipe(st, stx, r) for r in grid] + [lambda r: _Pipe(st, stx, r)])
    (gs_, go), gp = g.transform()
    out["pgs_gss"] = {"per_candidate": [{"score": jf(sc[0][0]), "offset": int(sc[0][1])} for sc in g._scores],
                      "gss_ratio": float(g._scores[-1][1].r),
                      "best": {"score": jf(gs_), "offset": int(go),
                               "index": [i for i, (_, p) in enumerate(g._scores) if p is gp][0]}}


def main():
    mods, srt = load_reference()
    out = {}
    gen_pgs(mods, out, srt)
    out["_meta"] = {"reference": "smacke/ffsubsync (PGS reference path)", "numpy": np.__version__,
                    "python": sys.version.split()[0], "generator": "tests/golden/make_golden_pgs.py"}
    with open(os.path.join(HERE, "pgs.json"), "w") as fh:
        json.dump(out, fh, indent=0, sort_keys=True)
    print("wrote pgs.json")


if __name__ == "__main__":
    main()
