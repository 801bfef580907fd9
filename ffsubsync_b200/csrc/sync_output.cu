// try_sync's epilogue over a finished batched sync call (b2_apply_sync): per track the decision of
// sync_output.cuh (scale, offset, gate, suppression, status), per cue the time the reference writes.
// One CTA per track: every thread derives the track's decision from the call's outputs (a few loads of
// the same words and a dozen flops, cheaper than a shared-memory round trip) and writes a slice of its cues.
#include <algorithm>

#include "common.cuh"
#include "sync_output.cuh"

struct ApplySyncParams {
  const double* bs;
  const int32_t* bo;
  const int32_t* bk;
  const double* gss;          // null: no search ran
  const double* start_s;      // absolute cue indices
  const double* end_s;
  const long long* cue_off;   // [T + 1]
  const double* ratios;       // [K]
  int T, K;
  B2SyncRule rule;
  long long* start_us;        // absolute cue indices
  long long* end_us;
  double* offset_seconds;     // [T]
  double* scale;
  int* status;
};

__global__ void __launch_bounds__(256) apply_sync_kernel(ApplySyncParams p) {
  for (int t = blockIdx.x; t < p.T; t += gridDim.x) {
    const bool has_gss = p.gss != nullptr;
    const int k = p.bk[t];
    const B2SyncTrack d = b2_sync_decide(p.bs[t], p.bo[t], k, p.ratios, p.K, has_gss,
                                         has_gss && k == p.K ? p.gss[t] : 0.0, p.rule);
    if (threadIdx.x == 0) {
      p.offset_seconds[t] = d.offset_seconds;
      p.scale[t] = d.scale;
      p.status[t] = d.status;
    }
    for (long long i = p.cue_off[t] + threadIdx.x; i < p.cue_off[t + 1]; i += blockDim.x) {
      p.start_us[i] = b2_synced_us(p.start_s[i], d);
      p.end_us[i] = b2_synced_us(p.end_s[i], d);
    }
  }
}

int b2i_apply_sync_launch(b2_ctx* h, const double* d_bs, const int32_t* d_bo, const int32_t* d_bk,
                          const double* d_gss, int T, const double* cue_start, const double* cue_end,
                          const int64_t* cue_off, double t_max, const double* ratios, int K, const B2SyncRule& rule,
                          int64_t* d_start_us, int64_t* d_end_us, double* d_offset_seconds, double* d_scale,
                          int32_t* d_status) {
  B2Range range("b2:apply_sync");
  // cue times and tables are host metadata: only [cue_off[0], cue_off[T]) is uploaded (pointers rebased)
  const size_t c0 = (size_t)cue_off[0], ncue = (size_t)cue_off[T] - c0;
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, ncue * 16 + (size_t)(T + 1) * 8 + (size_t)K * 8 + 256));
  ApplySyncParams p;
  void *hs, *he;
  p.start_s = (const double*)b2i_meta_reserve(&a, ncue * 8, &hs) - c0;
  p.end_s = (const double*)b2i_meta_reserve(&a, ncue * 8, &he) - c0;
  p.cue_off = (const long long*)b2i_meta_put(&a, cue_off, (size_t)(T + 1) * 8);
  p.ratios = K ? (const double*)b2i_meta_put(&a, ratios, (size_t)K * 8) : nullptr;
  // the cue times are checked in the pass that copies them into the pinned arena (one read of each; NaN fails the
  // comparison): a separate check pass would cost as much as the copy
  const double *s = cue_start + c0, *e = cue_end + c0;
  double *ds = (double*)hs, *de = (double*)he;
  int ok = 1;
  for (size_t i = 0; i < ncue; ++i) {
    ds[i] = s[i];
    de[i] = e[i];
    ok &= (fabs(s[i]) < t_max) & (fabs(e[i]) < t_max);
  }
  B2_TRY(b2i_meta_commit(&a));   // committed either way: the ring's reuse rule counts on every arena's event
  if (!ok)
    for (size_t i = 0; i < ncue; ++i)
      for (const double v : {s[i], e[i]}) {
        if (!isfinite(v)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: cue %zu: time %g is not finite", c0 + i, v);
        if (!(fabs(v) < t_max))
          B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: cue %zu: time %g, scaled by the largest ratio and shifted by the "
                  "largest offset, reaches B2_MAX_CUE_SECONDS (|t| must stay below %.17g)", c0 + i, v, t_max);
      }
  p.bs = d_bs;
  p.bo = d_bo;
  p.bk = d_bk;
  p.gss = d_gss;
  p.T = T;
  p.K = K;
  p.rule = rule;
  p.start_us = (long long*)d_start_us;
  p.end_us = (long long*)d_end_us;
  p.offset_seconds = d_offset_seconds;
  p.scale = d_scale;
  p.status = d_status;
  apply_sync_kernel<<<(unsigned)std::min(T, 65535), 256, 0, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "apply_sync_kernel");
  return B2_OK;
}

// b2_apply_split: the same output arithmetic with each cue's own offset.  Track t's decision at offset o is
// b2_sync_decide's for the candidate (ratio[t], o) with the gate and suppression off, so a cue's time is what
// try_sync's SubtitleScaler + SubtitleShifter write when that cue's segment is shifted by o.  A track without
// segments (n_segments <= 0: skipped, or its reference has a third level) is FAILED and keeps its original times.
struct ApplySplitParams {
  const double* ratio;        // [T]
  const int32_t* n_seg;       // [T]
  const int32_t* cue_offset;  // absolute cue indices
  const double* start_s;
  const double* end_s;
  const long long* cue_off;   // [T + 1]
  int T;
  B2SyncRule rule;            // gate off, no suppression
  long long* start_us;
  long long* end_us;
  int* status;
};

__global__ void __launch_bounds__(256) apply_split_kernel(ApplySplitParams p) {
  for (int t = blockIdx.x; t < p.T; t += gridDim.x) {
    const bool live = p.n_seg[t] > 0;
    if (threadIdx.x == 0) p.status[t] = live ? (B2_SYNC_WRITTEN | B2_SYNC_APPLIED) : B2_SYNC_FAILED;
    for (long long i = p.cue_off[t] + threadIdx.x; i < p.cue_off[t + 1]; i += blockDim.x) {
      const B2SyncTrack d = b2_sync_decide(0.0, live ? p.cue_offset[i] : 0, live ? 0 : -1, p.ratio + t, 1, false, 0.0,
                                           p.rule);
      p.start_us[i] = b2_synced_us(p.start_s[i], d);
      p.end_us[i] = b2_synced_us(p.end_s[i], d);
    }
  }
}

int b2i_apply_split_launch(b2_ctx* h, const double* ratio, const int32_t* d_n_segments, const int32_t* d_cue_offset,
                           int T, const double* cue_start, const double* cue_end, const int64_t* cue_off, double t_max,
                           const B2SyncRule& rule, int64_t* d_start_us, int64_t* d_end_us, int32_t* d_status) {
  B2Range range("b2:apply_split");
  const size_t c0 = (size_t)cue_off[0], ncue = (size_t)cue_off[T] - c0;
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, ncue * 16 + (size_t)(T + 1) * 8 + (size_t)T * 8 + 256));
  ApplySplitParams p;
  void *hs, *he;
  p.start_s = (const double*)b2i_meta_reserve(&a, ncue * 8, &hs) - c0;
  p.end_s = (const double*)b2i_meta_reserve(&a, ncue * 8, &he) - c0;
  p.cue_off = (const long long*)b2i_meta_put(&a, cue_off, (size_t)(T + 1) * 8);
  p.ratio = (const double*)b2i_meta_put(&a, ratio, (size_t)T * 8);
  const double *s = cue_start + c0, *e = cue_end + c0;
  double *ds = (double*)hs, *de = (double*)he;
  int ok = 1;
  for (size_t i = 0; i < ncue; ++i) {
    ds[i] = s[i];
    de[i] = e[i];
    ok &= (fabs(s[i]) < t_max) & (fabs(e[i]) < t_max);
  }
  B2_TRY(b2i_meta_commit(&a));
  if (!ok)
    for (size_t i = 0; i < ncue; ++i)
      for (const double v : {s[i], e[i]}) {
        if (!isfinite(v)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: cue %zu: time %g is not finite", c0 + i, v);
        if (!(fabs(v) < t_max))
          B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: cue %zu: time %g, scaled by the largest ratio and shifted by the "
                  "largest offset, reaches B2_MAX_CUE_SECONDS (|t| must stay below %.17g)", c0 + i, v, t_max);
      }
  p.n_seg = d_n_segments;
  p.cue_offset = d_cue_offset;
  p.T = T;
  p.rule = rule;
  p.start_us = (long long*)d_start_us;
  p.end_us = (long long*)d_end_us;
  p.status = d_status;
  apply_split_kernel<<<(unsigned)std::min(T, 65535), 256, 0, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "apply_split_kernel");
  return B2_OK;
}
