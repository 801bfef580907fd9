"""Restatement of the reference's PGS (bitmap subtitle) reference path (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/ffsubsync/speech_transformers.py:
  * :1012-1044  find_pgs_stream            (first hdmv_pgs_subtitle stream -> "0:s:N")
  * :1047-1100  _get_pgs_timings_via_ffprobe (show packets -> (pts, pts + duration))
  * :1186-1198  PGSSpeechTransformer.fit    (intervals -> 100 Hz signal, float64)
Pinned against the reference by tests/golden/make_golden_pgs.py (tests/golden/pgs.json).
"""
from typing import List, Optional, Sequence, Tuple

import numpy as np


def find_pgs_stream(probe: dict) -> Optional[str]:
    """Specifier "0:s:N" of the first PGS stream, N counting subtitle streams only; None without one."""
    n_sub = 0
    for s in probe.get("streams", []):
        if s.get("codec_type") != "subtitle":
            continue
        if s.get("codec_name") == "hdmv_pgs_subtitle":
            return "0:s:%d" % n_sub
        n_sub += 1
    return None


def pgs_timings(packets: Sequence[dict]) -> Optional[List[Tuple[float, float]]]:
    """Show packets' (start, end): every field present and parsable, duration not "N/A", size above 50 bytes."""
    out = []
    for p in packets:
        fields = [p.get(k) for k in ("pts_time", "duration_time", "size")]
        if any(f is None for f in fields) or fields[1] == "N/A":
            continue
        try:
            t0, d, size = float(fields[0]), float(fields[1]), int(fields[2])
        except ValueError:
            continue
        if size > 50:
            out.append((t0, t0 + d))
    return out or None


def pgs_frame(t: float, start_seconds: float, sample_rate: int) -> int:
    """int(round((t - start_seconds) * sample_rate)): float64 product, round half to even."""
    return int(round((float(t) - start_seconds) * sample_rate))


def pgs_length(max_end: float, sample_rate: int) -> int:
    """int(max_end * sample_rate) + 2: truncation toward zero, may be 1, 0 or negative."""
    return int(float(max_end) * sample_rate) + 2


def pgs_signal(intervals: Sequence[Tuple[float, float]], sample_rate: int = 100,
               start_seconds: float = 0.0) -> np.ndarray:
    """The float64 signal: 1.0 over [max(s0, 0), min(s1, n)) of every interval where that is not empty."""
    if not intervals:
        raise ValueError("empty interval list")
    n = pgs_length(max(e for _, e in intervals), sample_rate)
    x = np.zeros(n, dtype=float)   # raises for n < 0, as the reference does
    for s, e in intervals:
        a = max(pgs_frame(s, start_seconds, sample_rate), 0)
        b = min(pgs_frame(e, start_seconds, sample_rate), n)
        if a < b:
            x[a:b] = 1.0
    return x
