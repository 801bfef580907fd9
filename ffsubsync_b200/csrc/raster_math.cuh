// Bit-exact restatement of the reference's cue arithmetic (and, at the end, of its PGS interval arithmetic),
// shared by both rasterisers (raster.cu:
// raster_cues_kernel, raster_bits_kernel), by b2_rasterize_lengths on the host (api.cu) and by the
// CPU emulator tests/host_emul/raster_emul.cu.  Reference: SubtitleScaler.fit
// (ffsubsync/subtitle_transformers.py:35-47) + SubtitleSpeechTransformer.fit
// (ffsubsync/speech_transformers.py:957-980).
//
// Valid for finite times with |t * ratio| < B2_MAX_CUE_SECONDS and |start_seconds| below it too: there
// every microsecond count is an exact double, so (double)us / 1e6 is the correctly rounded quotient
// Python's int / int gives.  Callers reject everything else (api.cu) - the reference raises in
// timedelta for non-finite times, and beyond 2^63 us the integer product below overflows.
// On the host the intrinsics are the plain IEEE operations; the host half must be compiled without
// FMA contraction (-ffp-contract=off).
#pragma once
#include <math.h>

#include <cuda_runtime.h>

// 2^53 microseconds (about 285 years) in seconds
#define B2_MAX_CUE_SECONDS 9007199254.740992

#ifdef __CUDACC__
#define RASTER_HD __host__ __device__ __forceinline__
#else
#define RASTER_HD inline
#endif

RASTER_HD double b2_rm_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

RASTER_HD double b2_rm_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}

RASTER_HD double b2_rm_div(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

RASTER_HD long long b2_rm_rint(double x) {  // half-to-even (the host's default rounding mode)
#ifdef __CUDA_ARCH__
  return __double2ll_rn(x);
#else
  return llrint(x);
#endif
}

// timedelta(seconds=x) in integer microseconds: whole seconds exact, fractional part * 1e6 rounded
// half-to-even (CPython's delta_new; the whole part is a multiple of 1e6, so its parity is even).
RASTER_HD long long b2_timedelta_us(double x) {
  double whole;
  const double frac = modf(x, &whole);
  return (long long)whole * 1000000LL + b2_rm_rint(b2_rm_mul(frac, 1e6));
}

// timedelta(seconds=t*ratio) in microseconds (SubtitleScaler.fit, one correctly rounded product)
RASTER_HD long long b2_scaled_us(double t, double ratio) { return b2_timedelta_us(b2_rm_mul(t, ratio)); }

// timedelta(seconds=t*ratio).total_seconds(): the microseconds above, then one correctly rounded
// division (no FMA contraction).
RASTER_HD double b2_scaled_seconds(double t, double ratio) { return b2_rm_div((double)b2_scaled_us(t, ratio), 1e6); }

// Signal length int(max_time * sample_rate) + 2 (speech_transformers.py:958-962), max_time the largest
// scaled cue end and at least 0.  max_end: the largest unscaled cue end (0 for a track without cues).
// The max over cues of the scaled end is the scaled max end because the product, the microsecond
// rounding and the division are all monotone non-decreasing for ratio > 0.
RASTER_HD long long b2_signal_length(double max_end, double ratio, int sample_rate) {
  double max_time = 0.0;
  const double e = b2_scaled_seconds(max_end, ratio);
  if (e > max_time) max_time = e;
  return (long long)b2_rm_mul(max_time, (double)sample_rate) + 2;
}

// samples[first:last] of a length-n array with Python slice semantics (negative index wraps once).
RASTER_HD void b2_cue_bounds(double start_s, double end_s, double ratio, double start_seconds,
                             int sample_rate, long long n, long long& first, long long& last) {
  const double st = b2_scaled_seconds(start_s, ratio);
  const double en = b2_scaled_seconds(end_s, ratio);
  first = b2_rm_rint(b2_rm_mul(b2_rm_sub(st, start_seconds), (double)sample_rate));
  last = first + b2_rm_rint(b2_rm_mul(b2_rm_sub(en, st), (double)sample_rate));
  if (first < 0) { first += n; if (first < 0) first = 0; } else if (first > n) first = n;
  if (last < 0) { last += n; if (last < 0) last = 0; } else if (last > n) last = n;
}

// ---- PGS references (PGSSpeechTransformer.fit, ffsubsync/speech_transformers.py:1186-1198) ----------------------
// The bitmap-subtitle rule differs from the text one above: raw float64 times (no microsecond rounding), each end
// rounded on its own, and a length that is truncated toward zero with no max(0, .).  Valid for finite times and
// start_seconds with magnitude below B2_MAX_CUE_SECONDS and sample_rate <= B2_PGS_MAX_SAMPLE_RATE: every frame index
// then fits an int64 (2 * 2^33 s * 2^28 Hz < 2^62).  Callers reject everything else (sync_plan.h pgs_list_check).
#define B2_PGS_MAX_SAMPLE_RATE (1 << 28)

// int(max_end * sample_rate) + 2: may be 1, 0 or negative for max_end < 0 (np.zeros raises on negative)
RASTER_HD long long b2_pgs_length(double max_end, int sample_rate) {
  return (long long)b2_rm_mul(max_end, (double)sample_rate) + 2;
}

// The interval's frames [first, last) in a length-n signal: int(round((t - start_seconds) * sample_rate)) per end
// (Python round: half to even), then first = max(first, 0), last = min(last, n).  Empty when first >= last
// (intervals may overlap, be unsorted or have a negative duration).
RASTER_HD void b2_pgs_bounds(double start_s, double end_s, double start_seconds, int sample_rate, long long n,
                             long long& first, long long& last) {
  first = b2_rm_rint(b2_rm_mul(b2_rm_sub(start_s, start_seconds), (double)sample_rate));
  last = b2_rm_rint(b2_rm_mul(b2_rm_sub(end_s, start_seconds), (double)sample_rate));
  if (first < 0) first = 0;
  if (last > n) last = n;
}
