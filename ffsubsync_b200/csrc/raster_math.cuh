// Bit-exact restatement of the reference's cue arithmetic, shared by both rasterisers (raster.cu:
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

// timedelta(seconds=t*ratio).total_seconds(): whole seconds exact, fractional part * 1e6 rounded
// half-to-even to integer microseconds, then one correctly rounded division (no FMA contraction).
RASTER_HD double b2_scaled_seconds(double t, double ratio) {
  const double x = b2_rm_mul(t, ratio);
  double whole;
  const double frac = modf(x, &whole);
  const long long us = (long long)whole * 1000000LL + b2_rm_rint(b2_rm_mul(frac, 1e6));
  return b2_rm_div((double)us, 1e6);
}

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
