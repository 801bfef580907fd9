#!/usr/bin/env python
"""Reference-signal traffic of one bench step on the run path, float reference against packed bits.

COMPUTED FROM SHAPES, NOT MEASURED: bytes each kernel has to move for the reference of every video, at the
bench shape by default (256 two-hour pairs at 16 kHz, 100 windows per second).  The run path's own table
((R >> 5) + 3 entries of 8 bytes per video, written by ref_bits_kernel or ref_words_scan_kernel and read by
run_corr_kernel) is the same in both formats and left out.

    python tools/ref_traffic.py [--pairs 256] [--seconds 7200] [--cands 1]

--cands: re-scored candidates per pair (winner-only calls re-score the nominations of the ratios that can still
win; on the bench corpus that is about one per pair).  Each re-scored candidate reads the reference over the whole
overlap (about R frames for the bench's +-60 s windows).
"""
import argparse


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--cands", type=float, default=1.0)
    a = ap.parse_args()
    R = int(a.seconds * 100)                 # reference windows per video
    words = (R + 31) // 32
    rows = [
        ("VAD writes the reference", 4 * R, 4 * words),
        ("reference table reads it (ref_bits / ref_words_scan)", 4 * R, 4 * words),
        ("rescore_kernel reads it, per re-scored candidate x %g" % a.cands, 4 * R * a.cands, 4 * words * a.cands),
    ]
    print("computed from shapes (not measured): %d pairs x %g s, R = %d windows per video" % (a.pairs, a.seconds, R))
    print("%-58s %14s %14s" % ("per pair", "float (MB)", "packed (MB)"))
    tf = tp = 0.0
    for name, f, p in rows:
        print("%-58s %14.3f %14.3f" % (name, f / 1e6, p / 1e6))
        tf += f
        tp += p
    print("%-58s %14.3f %14.3f" % ("total per pair", tf / 1e6, tp / 1e6))
    print("%-58s %14.3f %14.3f" % ("total per step (GB)", tf * a.pairs / 1e9, tp * a.pairs / 1e9))
    print("saved per step: %.3f GB = %.2f ms at 2.9 TB/s (the step's measured HBM rate)"
          % ((tf - tp) * a.pairs / 1e9, (tf - tp) * a.pairs / 2.9e12 * 1e3))


if __name__ == "__main__":
    main()
