// Bit-exact restatement of what the reference's try_sync does with an aligner's answer
// (ffsubsync/ffsubsync.py:236-299): the winning scale and the offset in seconds, the
// --skip-sync-on-low-quality gate (assess_alignment_quality, :145-174), --suppress-output-if-offset-less-than,
// sync_was_successful, and the output times SubtitleScaler + SubtitleShifter write
// (ffsubsync/subtitle_transformers.py:13-50, generic_subtitles.py:128-132).  Shared by sync_output.cu
// (apply_sync_kernel), b2_apply_sync's host checks (api.cu) and the CPU emulator
// tests/host_emul/sync_output_emul.cu.  The host half must be compiled without FMA contraction.
#pragma once
#include "../../include/ffsubsync_b200.h"
#include "job_plan.cuh"   // b2_rm_add, the search's interval B2_GSS_LO / B2_GSS_HI
#include "raster_math.cuh"

// The thresholds of one b2_apply_sync call.  suppress_below: -inf when there is no suppression threshold
// (the reference's `thresh or float("-inf")`: None and 0.0 both mean none).
struct B2SyncRule {
  int sample_rate;
  double apply_offset_seconds;
  int gate;                        // --skip-sync-on-low-quality
  double min_score, max_offset_seconds, max_framerate_deviation;
  double suppress_below;
};

inline B2SyncRule b2_sync_rule(int sample_rate, double apply_offset_seconds, int gate_enabled, double min_score,
                               double max_offset_seconds, double max_framerate_deviation, int has_suppress,
                               double suppress_output_if_offset_less_than) {
  return B2SyncRule{sample_rate, apply_offset_seconds, gate_enabled ? 1 : 0, min_score, max_offset_seconds,
                    max_framerate_deviation,
                    (has_suppress && suppress_output_if_offset_less_than != 0.0) ? suppress_output_if_offset_less_than
                                                                                 : -INFINITY};
}

// The per-track decision.  scale / offset_seconds are NaN for a failed track; shift_us is the shift the
// output times get (0 unless B2_SYNC_APPLIED).  ratios: the K grid ratios; gss_ratio: the track's search
// point (read only when has_gss and best_k == K).  A search point outside [0.9, 1.1] (not one the search can
// produce, NaN included) counts as a failed alignment, so no output time leaves the range the arithmetic
// is exact on.
struct B2SyncTrack {
  int status;
  double scale, offset_seconds;
  long long shift_us;
};

RASTER_HD B2SyncTrack b2_sync_decide(double best_score, int best_offset, int best_k, const double* ratios, int K,
                                     bool has_gss, double gss_ratio, const B2SyncRule& r) {
  B2SyncTrack o{B2_SYNC_FAILED, NAN, NAN, 0};
  double scale;
  if (best_k >= 0 && best_k < K) {
    scale = ratios[best_k];
  } else if (has_gss && best_k == K && gss_ratio >= B2_GSS_LO && gss_ratio <= B2_GSS_HI) {
    scale = gss_ratio;
  } else {
    return o;   // MaxScoreAligner raised: nothing is written, result is left unset
  }
  // offset_samples / float(SAMPLE_RATE) + apply_offset_seconds: two correctly rounded operations
  const double off = b2_rm_add(b2_rm_div((double)best_offset, (double)r.sample_rate), r.apply_offset_seconds);
  o.scale = scale;
  o.offset_seconds = off;
  int st = B2_SYNC_SUCCESSFUL;
  if (best_score < 0) st = 0;   // the output is still written
  if (r.gate) {
    int low = 0;
    if (best_score < r.min_score) low |= B2_SYNC_LOW_SCORE;
    if (fabs(off) > r.max_offset_seconds) low |= B2_SYNC_LOW_OFFSET;
    if (fabs(b2_rm_sub(scale, 1.0)) > r.max_framerate_deviation) low |= B2_SYNC_LOW_FRAMERATE;
    if (low) {   // the original cues are written; the track is not successful
      o.status = low | B2_SYNC_WRITTEN;
      return o;
    }
  }
  st |= B2_SYNC_APPLIED;
  if (off >= r.suppress_below) st |= B2_SYNC_WRITTEN;
  else st |= B2_SYNC_SUPPRESSED;
  o.status = st;
  o.shift_us = b2_timedelta_us(off);
  return o;
}

// One output time: timedelta(seconds=t * scale) + timedelta(seconds=offset) for applied tracks, the parsed
// original timedelta(seconds=t) otherwise.
RASTER_HD long long b2_synced_us(double t, const B2SyncTrack& d) {
  return (d.status & B2_SYNC_APPLIED) ? b2_scaled_us(t, d.scale) + d.shift_us : b2_scaled_us(t, 1.0);
}
