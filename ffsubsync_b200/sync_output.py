"""What try_sync does with the aligner's answer (ffsubsync/ffsubsync.py:236-299), for the batched calls.

``BatchSynchronizer.apply_sync`` / ``apply_sync_host`` run b2_apply_sync: per track the scale and offset, the
``--skip-sync-on-low-quality`` gate, ``--suppress-output-if-offset-less-than`` and ``sync_was_successful`` as
status bits, and per cue the output time in microseconds.  This module holds the bits, the reference's
``assess_alignment_quality`` and ``reasons``, which rebuilds its reason strings from a track's bits.
"""
from typing import List

from .constants import DEFAULT_MAX_FRAMERATE_DEVIATION, DEFAULT_MIN_SCORE, DEFAULT_QUALITY_MAX_OFFSET_SECONDS

# status bits of b2_apply_sync (include/ffsubsync_b200.h B2_SYNC_*)
WRITTEN = 1          # the reference writes this track's output
APPLIED = 2          # the synced times are scaled and shifted (else the parsed originals)
SUCCESSFUL = 4       # the track keeps try_sync's sync_was_successful true
FAILED = 8           # no alignment: nothing is written
SUPPRESSED = 16      # --suppress-output-if-offset-less-than held the output back
LOW_SCORE = 32       # the gate's reasons, in the reference's order
LOW_OFFSET = 64
LOW_FRAMERATE = 128
LOW_QUALITY = LOW_SCORE | LOW_OFFSET | LOW_FRAMERATE


def assess_alignment_quality(best_score: float, offset_seconds: float, scale_factor: float, *, min_score: float,
                             max_offset_seconds: float, max_framerate_deviation: float) -> List[str]:
    """The reference's gate (ffsubsync/ffsubsync.py:145-174): the reasons an alignment looks too low-quality to
    trust, empty to trust it."""
    reasons: List[str] = []
    if best_score < min_score:
        reasons.append("score %.1f < %.1f" % (best_score, min_score))
    if abs(offset_seconds) > max_offset_seconds:
        reasons.append("|offset| %.1fs > %.1fs" % (abs(offset_seconds), max_offset_seconds))
    framerate_deviation = abs(scale_factor - 1.0)
    if framerate_deviation > max_framerate_deviation:
        reasons.append("framerate deviation %.3f > %.3f" % (framerate_deviation, max_framerate_deviation))
    return reasons


def reasons(status: int, best_score: float, offset_seconds: float, scale: float, *,
            min_score: float = DEFAULT_MIN_SCORE, max_offset_seconds: float = DEFAULT_QUALITY_MAX_OFFSET_SECONDS,
            max_framerate_deviation: float = DEFAULT_MAX_FRAMERATE_DEVIATION) -> List[str]:
    """The reason strings the reference logs for a gated track, from its status bits and apply_sync's
    offset_seconds / scale (pass the thresholds of the apply_sync call).  Empty for a track the gate let through."""
    status = int(status)
    out: List[str] = []
    if status & LOW_SCORE:
        out.append("score %.1f < %.1f" % (best_score, min_score))
    if status & LOW_OFFSET:
        out.append("|offset| %.1fs > %.1fs" % (abs(offset_seconds), max_offset_seconds))
    if status & LOW_FRAMERATE:
        out.append("framerate deviation %.3f > %.3f" % (abs(scale - 1.0), max_framerate_deviation))
    return out
