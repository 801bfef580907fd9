#!/usr/bin/env python
"""Generate tests/golden/subs_ref.json by running the REAL reference's embedded-subtitle path.

Run where a checkout of the reference is available (FFSUBSYNC_REFERENCE names it; the tests only
read the fixture this writes):   FFSUBSYNC_REFERENCE=<checkout> python tests/golden/make_golden_subs_ref.py

The reference is imported the way make_golden.py imports it (behind stub modules for the missing
third-party packages).  Nothing is copied: the reference's own code computes every expected value
written below.
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


def gen_subs_ref(mods, out, srt):
    """VideoSpeechTransformer(vad="subs_then_webrtc").fit on a video whose text subtitle streams are prepared cue
    lists (speech_transformers.py:479-523,609-619): stream enumeration and extraction are stubbed to hand the lists
    over, and the parse step of make_subtitle_speech_pipeline passes them through.  Records, per video, the stream
    the reference chose and its signal (as runs), and MaxScoreAligner over the 7-ratio grid of an input track
    against the 2 h case's signal."""
    st, stx, gs, al = (mods["speech_transformers"], mods["subtitle_transformers"], mods["generic_subtitles"],
                       mods["aligners"])

    class Subs(list):
        def clone_props_for_subs(self, new_subs):
            return Subs(new_subs)

    def make(starts, ends, contents):
        return Subs(gs.GenericSubtitle(timedelta(seconds=float(a)), timedelta(seconds=float(b)),
                                       srt.Subtitle(content=c)) for a, b, c in zip(starts, ends, contents))

    class PassParser:   # the parse step: the "buffer" already is the parsed cue list
        def __init__(self, **kw):
            self.__dict__.update(kw)

        def fit(self, subs, *_):
            self.subs_ = subs
            return self

        def transform(self, *_):
            return self.subs_

        def fit_transform(self, subs, *_):
            return self.fit(subs).transform()

    saved_parser = st.make_subtitle_parser
    st.make_subtitle_parser = lambda fmt, encoding=None, caching=False, max_subtitle_seconds=None, start_seconds=0, \
        **kw: PassParser(encoding=encoding, max_subtitle_seconds=max_subtitle_seconds, start_seconds=start_seconds)

    def fit_video(streams, start_seconds):
        t = st.VideoSpeechTransformer(vad="subs_then_webrtc", sample_rate=100, frame_rate=48000,
                                      non_speech_label=0.0, start_seconds=start_seconds)
        lists = [make(*s) for s in streams]
        t._probe_embedded_subtitle_streams = lambda fname: ["0:s:%d" % i for i in range(len(lists))]
        t._extract_embedded_subs_single_pass = lambda fname, names: list(lists)
        t._extract_embedded_subs_per_stream = lambda fname, names: list(lists)

        def no_audio(fname):
            raise AssertionError("the embedded-subtitle path fell back to audio")

        t._fit_using_audio = no_audio
        t.fit("ref.mkv")
        x = np.asarray(t.transform(), dtype=float)
        # which stream: the signal each stream gives on its own (ties are built from different cue lists)
        own = [st.SubtitleSpeechTransformer(100, start_seconds, 1.0).fit(stx.SubtitleScaler(1.0).fit(
            make(*s)).transform()) for s in streams]
        chosen = [i for i, o in enumerate(own) if np.array_equal(o.transform(), x)][0]
        return x, chosen, [float(o.max_time_) for o in own]

    syn = cases.synthetic_cues(21, 7200.0)
    syn_short = cases.synthetic_cues(22, 5400.0)
    meta_contents = ["[music]", "Hello there.", "How are you?", "(door slams)", "Fine.", "English subtitles"]
    videos = [
        # tied max_time_: the first of the two streams ending at 100.0 s wins
        ("tie", 0, [([1.0, 20.0, 40.0], [5.0, 30.0, 100.0], ["a", "b", "c"]),
                    ([2.0, 50.0], [9.0, 100.0], ["d", "e"]),
                    ([3.0], [60.0], ["f"])]),
        # start_seconds above the first cues: negative slice starts wrap
        ("start_seconds", 7, [([2.0, 5.0, 10.0, 30.5], [4.0, 9.25, 12.0, 33.0], ["a", "b", "c", "d"])]),
        # metadata first / last cues (kept out) and one in the middle (edge rule)
        ("metadata", 0, [([0.5, 3.0, 6.0, 9.0, 12.0, 15.0], [2.5, 5.5, 8.0, 11.0, 14.0, 18.0], meta_contents),
                         ([1.0], [10.0], ["x"])]),
        # an empty stream counts; a one-cue stream is longer
        ("one_and_empty", 0, [([], [], []), ([4.25], [6.5], ["only"])]),
        ("empty_only", 0, [([], [], [])]),
        ("empty_only_start", 3, [([], [], [])]),
        # a 2 h stream against a 1.5 h one
        ("two_hours", 0, [(list(syn_short[0]), list(syn_short[1]), ["s"] * len(syn_short[0])),
                          (list(syn[0]), list(syn[1]), ["s"] * len(syn[0]))]),
    ]
    rows = []
    sig_2h = None
    for name, ss, streams in videos:
        x, chosen, times = fit_video(streams, ss)
        levels, rs, re_ = cases.run_lengths(x)
        rows.append({"name": name, "start_seconds": ss,
                     "streams": [{"starts": [float(a) for a in s[0]], "ends": [float(b) for b in s[1]],
                                  "contents": list(s[2])} for s in streams],
                     "max_time": times, "chosen": chosen, "length": int(len(x)), "levels": levels,
                     "run_starts": rs, "run_stops": re_})
        if name == "two_hours":
            sig_2h = x
    st.make_subtitle_parser = saved_parser
    out["subs_ref"] = rows

    # the input track: the 2 h stream's cues scaled by 25/24 and delayed by 3.5 s, through try_sync's grid
    starts, ends = syn
    true_r = 25.0 / 24.0
    in_starts = [round(a / true_r + 3.5, 3) for a in starts]
    in_ends = [round(b / true_r + 3.5, 3) for b in ends]
    subs = make(in_starts, in_ends, ["s"] * len(in_starts))
    sigs = []
    for r in cases.ratio_grid():
        scaled = stx.SubtitleScaler(r).fit(subs).transform()
        sigs.append(st.SubtitleSpeechTransformer(sample_rate=100, start_seconds=0, framerate_ratio=r).fit(scaled)
                    .transform())
    m = al.MaxScoreAligner(al.FFTAligner, None, 100, 60).fit(sig_2h, sigs)
    per = [{"score": jf(sc[0][0]), "offset": int(sc[0][1])} for sc in m._scores]
    (bs, bo), bp = m.transform()
    bidx = [i for i, sg in enumerate(sigs) if sg is bp][0]
    out["subs_ref_maxscore"] = {"video": "two_hours", "in_starts": in_starts, "in_ends": in_ends,
                                "max_offset_seconds": 60, "per_ratio": per,
                                "best": {"score": jf(bs), "offset": int(bo), "index": bidx}}


def main():
    mods, srt = load_reference()
    out = {}
    gen_subs_ref(mods, out, srt)
    out["_meta"] = {"reference": "smacke/ffsubsync (v0.5.0)", "numpy": np.__version__,
                    "python": sys.version.split()[0], "generator": "tests/golden/make_golden_subs_ref.py"}
    with open(os.path.join(HERE, "subs_ref.json"), "w") as fh:
        json.dump(out, fh, indent=0, sort_keys=True)
    print("wrote subs_ref.json")


if __name__ == "__main__":
    main()
