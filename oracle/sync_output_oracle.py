"""try_sync's epilogue (ffsubsync/ffsubsync.py:236-299) restated in plain Python over a batched call's results:
the winning scale, offset_seconds, the --skip-sync-on-low-quality gate, --suppress-output-if-offset-less-than,
sync_was_successful, and the output times through datetime.timedelta exactly as SubtitleScaler and
SubtitleShifter compute them.  The yardstick of b2_apply_sync (tests/test_sync_output_cpu.py checks it against
the reference's own try_sync, tests/golden/sync_output.json).  Status bits as in include/ffsubsync_b200.h."""
import math
from datetime import timedelta

import numpy as np

WRITTEN, APPLIED, SUCCESSFUL, FAILED, SUPPRESSED, LOW_SCORE, LOW_OFFSET, LOW_FRAMERATE = (1 << i for i in range(8))
US = timedelta(microseconds=1)


def td_us(seconds: float) -> int:
    return timedelta(seconds=float(seconds)) // US


def decide(best_score, best_offset, best_k, ratios, gss_ratio, sample_rate, apply_offset_seconds=0.0, gate=False,
           min_score=0.0, quality_max_offset_seconds=30.0, max_framerate_deviation=0.1, suppress=None):
    """(status, scale, offset_seconds) of one track; gss_ratio None when no search ran."""
    K = len(ratios)
    best_k = int(best_k)
    if 0 <= best_k < K:
        scale = float(ratios[best_k])
    elif gss_ratio is not None and best_k == K and 0.9 <= float(gss_ratio) <= 1.1:
        scale = float(gss_ratio)
    else:
        return FAILED, math.nan, math.nan
    best_score = float(best_score)
    offset_seconds = int(best_offset) / float(sample_rate) + float(apply_offset_seconds)
    status = SUCCESSFUL if not best_score < 0 else 0
    if gate:
        low = 0
        if best_score < min_score:
            low |= LOW_SCORE
        if abs(offset_seconds) > quality_max_offset_seconds:
            low |= LOW_OFFSET
        if abs(scale - 1.0) > max_framerate_deviation:
            low |= LOW_FRAMERATE
        if low:
            return low | WRITTEN, scale, offset_seconds
    status |= APPLIED
    status |= WRITTEN if offset_seconds >= (suppress or float("-inf")) else SUPPRESSED
    return status, scale, offset_seconds


def apply_sync(best_score, best_offset, best_k, gss_ratio, cue_start, cue_end, cue_off, ratios, sample_rate, **rule):
    """b2_apply_sync over T tracks: returns (synced_start_us, synced_end_us, offset_seconds, scale, status), numpy
    arrays; the cue arrays cover cue_off[0] .. cue_off[T] at their absolute indices."""
    T = len(cue_off) - 1
    n = int(cue_off[-1]) if T >= 0 else 0
    su = np.zeros(n, np.int64)
    eu = np.zeros(n, np.int64)
    off = np.full(T, np.nan)
    sc = np.full(T, np.nan)
    st = np.zeros(T, np.int32)
    for t in range(T):
        g = None if gss_ratio is None else gss_ratio[t]
        st[t], sc[t], off[t] = decide(best_score[t], best_offset[t], best_k[t], ratios, g, sample_rate, **rule)
        for i in range(int(cue_off[t]), int(cue_off[t + 1])):
            for src, dst in ((cue_start, su), (cue_end, eu)):
                x = float(src[i])
                if st[t] & APPLIED:
                    # SubtitleScaler: timedelta(seconds=total_seconds * scale); SubtitleShifter: + timedelta(offset)
                    dst[i] = td_us(x * sc[t]) + td_us(off[t])
                else:
                    dst[i] = td_us(x)
    return su, eu, off, sc, st
