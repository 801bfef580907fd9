#!/usr/bin/env python
"""Generate tests/golden/signal_ref.json by running the REAL reference's serialized-speech path
(``ffs ref.npz -i in.srt``: DeserializeSpeechTransformer, then MaxScoreAligner over the ratio grid and with --gss).

Run where a checkout of the reference is available (FFSUBSYNC_REFERENCE names it; the tests only
read the fixture this writes):   FFSUBSYNC_REFERENCE=<checkout> python tests/golden/make_golden_signal_ref.py

Each stored signal is written as a real ``.npz`` (key "speech") and ``.npy`` file to a temporary directory and read
back by the reference's DeserializeSpeechTransformer.fit; the two reads must agree, and each label's output is
recorded once.  Nothing is copied: the reference's own code computes every expected value written below.  Signals are
recorded as run lengths (levels, run starts) with their exact float64 values: "stored" once per signal, "signals"
once per (signal, label).  One JSON row per line.
"""
import json
import os
import sys
import tempfile
from datetime import timedelta

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import cases  # noqa: E402
from make_golden import jf, load_reference  # noqa: E402
from make_golden_pgs import _Pipe  # noqa: E402

LABELS = (0.0, 0.5, -0.5)
EDGE = [1.0 - 2.0 ** -53, 1.0 - 2.0 ** -25, 1.0, 0.0, -0.5, -np.inf, 0.999, 1.0, 1.0 - 2.0 ** -24, 0.5, 1.0, 1.0]


def _runs_signal(n, rng, gap_values, speech=1.0, mean_run=180.0, mean_gap=140.0):
    """n frames of speech runs (value `speech`) and gaps, each gap one value drawn from gap_values."""
    x = np.empty(n, dtype=np.float64)
    i, on = 0, False
    while i < n:
        d = max(1, int(rng.exponential(mean_run if on else mean_gap)))
        x[i: i + d] = speech if on else gap_values[rng.randint(len(gap_values))]
        i += d
        on = not on
    return x


def stored_signals():
    """(name, stored float64 values) of every case."""
    rng = np.random.RandomState(41)
    palette = [0.0, 1.0 - 2.0 ** -53, -np.inf, 0.3, 1.0 - 2.0 ** -25, -0.5]
    # a sparse three-level signal shaped like a multi-segment reference: silence, speech and a half level
    three = np.zeros(5000)
    for s in range(100, 5000, 700):
        three[s: s + 120] = 1.0
        three[s + 300: s + 380] = 0.5
    return [
        ("edges", np.array(EDGE)),
        ("r32", _runs_signal(32, rng, palette, mean_run=3, mean_gap=3)),
        ("r33", _runs_signal(33, rng, palette, mean_run=3, mean_gap=3)),
        ("r63", _runs_signal(63, rng, palette, mean_run=4, mean_gap=4)),
        ("r96", _runs_signal(96, rng, palette, mean_run=5, mean_gap=5)),
        ("r7", np.array([1.0, 0.25, 1.0, 1.0, 1.0 - 2.0 ** -25, -np.inf, 1.0])),
        ("empty", np.zeros(0)),
        ("three_level", three),
        ("two_hours", _runs_signal(720000, rng, palette, mean_run=1500.0, mean_gap=1100.0)),
    ]


def rle(x):
    """(levels, starts) of x, levels exact (jf for -inf)."""
    x = np.asarray(x, dtype=np.float64)
    if len(x) == 0:
        return [], []
    change = np.flatnonzero(x[1:] != x[:-1]) + 1
    starts = np.concatenate([[0], change])
    return [jf(v) for v in x[starts]], [int(s) for s in starts]


def gen(mods, out, srt):
    st, stx, gs, al = (mods["speech_transformers"], mods["subtitle_transformers"], mods["generic_subtitles"],
                       mods["aligners"])
    stored, rows = [], []
    sig_2h = None
    with tempfile.TemporaryDirectory() as tmp:
        for name, x in stored_signals():
            npz, npy = os.path.join(tmp, name + ".npz"), os.path.join(tmp, name + ".npy")
            np.savez(npz, speech=x)
            np.save(npy, x)
            levels, starts = rle(x)
            stored.append({"name": name, "length": int(len(x)), "levels": levels, "starts": starts})
            for label in LABELS:
                y = st.DeserializeSpeechTransformer(label).fit(npz).transform()
                y_npy = st.DeserializeSpeechTransformer(label).fit(npy).transform()
                assert y.dtype == y_npy.dtype == np.float64 and np.array_equal(y, y_npy)
                ol, os_ = rle(y)
                rows.append({"name": name, "label": label, "formats": ["npz", "npy"], "length": int(len(x)),
                             "out_levels": ol, "out_starts": os_})
                if name == "two_hours" and label == 0.0:
                    sig_2h = np.asarray(y, dtype=float)
    out["stored"] = stored
    out["signals"] = rows

    # an input track against the 2 h reference: its speech runs as cues, scaled by 25/24 and delayed by 3.5 s
    on = np.concatenate([[0], (sig_2h == 1.0).astype(np.int8), [0]])
    d = np.diff(on)
    starts, stops = np.flatnonzero(d == 1), np.flatnonzero(d == -1)
    true_r = 25.0 / 24.0
    in_starts = [round(a / 100.0 / true_r + 3.5, 3) for a in starts]
    in_ends = [round(b / 100.0 / true_r + 3.5, 3) for b in stops]

    class Subs(list):
        def clone_props_for_subs(self, new_subs):
            return Subs(new_subs)

    subs = Subs(gs.GenericSubtitle(timedelta(seconds=a), timedelta(seconds=b), srt.Subtitle(content="s"))
                for a, b in zip(in_starts, in_ends))
    grid = cases.ratio_grid()
    m = al.MaxScoreAligner(al.FFTAligner, subs, 100, 60).fit(sig_2h, [_Pipe(st, stx, r) for r in grid])
    per = [{"score": jf(sc[0][0]), "offset": int(sc[0][1])} for sc in m._scores]
    (bs, bo), bp = m.transform()
    out["maxscore"] = {"in_starts": in_starts, "in_ends": in_ends, "max_offset_seconds": 60, "per_ratio": per,
                       "best": {"score": jf(bs), "offset": int(bo),
                                "index": [i for i, (_, p) in enumerate(m._scores) if p is bp][0]}}
    g = al.MaxScoreAligner(al.FFTAligner, subs, 100, 60)
    g.fit(sig_2h, [_Pipe(st, stx, r) for r in grid] + [lambda r: _Pipe(st, stx, r)])
    (gs_, go), gp = g.transform()
    out["gss"] = {"per_candidate": [{"score": jf(sc[0][0]), "offset": int(sc[0][1])} for sc in g._scores],
                  "gss_ratio": float(g._scores[-1][1].r),
                  "best": {"score": jf(gs_), "offset": int(go),
                           "index": [i for i, (_, p) in enumerate(g._scores) if p is gp][0]}}


def main():
    mods, srt = load_reference()
    out = {}
    gen(mods, out, srt)
    out["_meta"] = {"reference": "smacke/ffsubsync (serialized speech reference, DeserializeSpeechTransformer)",
                    "numpy": np.__version__, "python": sys.version.split()[0],
                    "generator": "tests/golden/make_golden_signal_ref.py"}
    # one row per line: a readable diff at a few tens of KB
    lines = []
    for key in sorted(out):
        val = out[key]
        if isinstance(val, list):
            body = "[\n" + ",\n".join(json.dumps(r, sort_keys=True) for r in val) + "\n]"
        else:
            body = json.dumps(val, sort_keys=True)
        lines.append("%s: %s" % (json.dumps(key), body))
    with open(os.path.join(HERE, "signal_ref.json"), "w") as fh:
        fh.write("{\n" + ",\n".join(lines) + "\n}\n")
    print("wrote signal_ref.json")


if __name__ == "__main__":
    main()
