// Per-job alignment plan and the golden-section step, shared by the host planner (corr.cu:
// b2i_align_launch), the device-driven GSS rounds (gss.cu: gss_step_kernel) and the CPU emulator
// tests/host_emul/gss_emul.cu.  Plain __host__ __device__ arithmetic: no CUDA runtime calls.
//
// Reference: FFTAligner.fit (ffsubsync/aligners.py:31-48: padded length, mask slice, offset of a
// conv[] index) and golden_section_search.gss (ffsubsync/golden_section_search.py:15-74).  The host
// half must be compiled without FMA contraction (-ffp-contract=off), like raster_math.cuh.
#pragma once
#include <stdint.h>

#include "../../include/ffsubsync_b200.h"
#include "raster_math.cuh"

// ---- FFTAligner's window --------------------------------------------------------------------
// int(2 ** math.ceil(math.log(n, 2))), aligners.py:67-68; quirk_mask bit k set: CPython's
// ceil(math.log(2**k, 2)) == k + 1 (see b2_create).
RASTER_HD long long b2_padded_length(long long n, uint64_t quirk_mask) {
  int k = 0;
  while ((1LL << k) < n) ++k;
  if ((1LL << k) == n && (quirk_mask >> k) & 1ULL) ++k;
  return 1LL << k;
}

struct B2JobPlan {
  int kind;            // 0 window left, 1 empty input (aligners.py:58-66), 2 everything masked
  long long N;         // padded length (kind != 1)
  long long lo, hi;    // surviving conv[] index range [lo, hi) (kind 0)
  long long o_lo, o_hi;  // its offsets, o = N - 1 - S - index (aligners.py:47), inclusive (kind 0)
  int masked_offset;   // offset reported when kind == 2
};

// One (reference length R, subtitle length S) job.  max_offset_samples: B2_MAX_OFFSET_NONE or any
// int64 width, which goes through the reference's slice arithmetic (aligners.py:31-43) literally; widths
// are clamped to +-2^40 first (beyond every padded length, so the result is unchanged).
RASTER_HD B2JobPlan b2_plan_job(long long R, long long S, long long max_offset_samples, uint64_t quirk_mask) {
  B2JobPlan p;
  p.kind = 1;
  p.N = 0;
  p.lo = p.hi = 0;
  p.o_lo = 0;
  p.o_hi = -1;
  p.masked_offset = 0;
  if (R == 0 || S == 0) return p;
  const long long N = b2_padded_length(R + S, quirk_mask);
  p.N = N;
  long long lo = 0, hi = N;
  if (max_offset_samples != B2_MAX_OFFSET_NONE) {
    const long long lim = 1LL << 40;
    const long long mo = max_offset_samples < -lim ? -lim : (max_offset_samples > lim ? lim : max_offset_samples);
    const long long a = N - 1 - mo - S;
    const long long bb = N - 1 + mo - S;
    lo = a >= 0 ? (a < N ? a : N) : (a + N > 0 ? a + N : 0);
    hi = bb >= 0 ? (bb < N ? bb : N) : (bb + N > 0 ? bb + N : 0);
  }
  if (lo >= hi) {
    p.kind = 2;
    p.masked_offset = (int)(N - 1 - S);
    return p;
  }
  p.kind = 0;
  p.lo = lo;
  p.hi = hi;
  p.o_lo = N - S - hi;
  p.o_hi = N - 1 - S - lo;
  return p;
}

// ---- golden-section search over the framerate ratio ------------------------------------------
// MaxScoreAligner.fit_gss (aligners.py:111-129): gss(-score, MIN_FRAMERATE_RATIO, MAX_FRAMERATE_RATIO,
// tol=1e-4) evaluates 17 points; the 17th is the candidate.  The interval and tolerance are fixed.
#define B2_GSS_LO 0.9
#define B2_GSS_HI 1.1
constexpr int kGssEvals = 17;   // n + 1 with n = ceil(log(1e-4 / 0.2) / log(invphi)) = 16

// (sqrt(5) - 1) / 2 and (3 - sqrt(5)) / 2 as Python evaluates them (both subtractions are exact)
constexpr double kGssInvPhi = 0.6180339887498949;
constexpr double kGssInvPhi2 = 0.3819660112501051;

RASTER_HD double b2_rm_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

struct B2GssLane {
  double a, b, c, d, yc, yd, h;
  int left;            // the previous round evaluated c (1) or d (0)
};

// Round r (0 .. n) of a search with n >= 1 iterations: takes y_prev, the objective (the negated
// score) at the point of round r - 1 (unused at r = 0), and returns the point of round r.  Rounds 0 and
// 1 are gss's c and d; round r >= 2 is loop iteration k = r - 2.  Every operation is the reference's
// float64 operation in its order, and the comparisons are IEEE (an all-masked window scores -inf, so
// its objective is +inf).
RASTER_HD double b2_gss_step(B2GssLane& s, int r, double y_prev, double lo, double hi) {
  if (r == 0) {
    s.a = lo < hi ? lo : hi;
    s.b = lo < hi ? hi : lo;
    s.h = b2_rm_sub(s.b, s.a);
    s.c = b2_rm_add(s.a, b2_rm_mul(kGssInvPhi2, s.h));
    s.d = b2_rm_add(s.a, b2_rm_mul(kGssInvPhi, s.h));
    s.yc = s.yd = 0.0;
    s.left = 1;
    return s.c;
  }
  if (r == 1) {
    s.yc = y_prev;
    s.left = 0;
    return s.d;
  }
  if (s.left) s.yc = y_prev;
  else s.yd = y_prev;
  s.h = b2_rm_mul(kGssInvPhi, s.h);
  if (s.yc < s.yd) {
    s.b = s.d;
    s.d = s.c;
    s.yd = s.yc;
    s.c = b2_rm_add(s.a, b2_rm_mul(kGssInvPhi2, s.h));
    s.left = 1;
    return s.c;
  }
  s.a = s.c;
  s.c = s.d;
  s.yc = s.yd;
  s.d = b2_rm_add(s.a, b2_rm_mul(kGssInvPhi, s.h));
  s.left = 0;
  return s.d;
}

// gss's return value after the last round's objective y_last: (a, d) if yc < yd else (c, b).
RASTER_HD void b2_gss_finish(B2GssLane& s, double y_last, double& lo, double& hi) {
  if (s.left) s.yc = y_last;
  else s.yd = y_last;
  if (s.yc < s.yd) {
    lo = s.a;
    hi = s.d;
  } else {
    lo = s.c;
    hi = s.b;
  }
}
