// Run-length correlation of a subtitle bit mask against a two-level reference (csrc/runcorr.cu), the
// arithmetic shared by the kernel and its CPU emulation (tests/host_emul/runcorr_emul.cu).
//
// On the b2_sync_batch / b2_sync_tracks path the reference is this call's own VAD output, so every value
// is 1.0 or the non-speech label, and the subtitle signal is a bit mask made of cue runs.  With
//     s' = hi  inside a run, -1 outside          (hi = 2*(double)level - 1, what rescore_kernel uses)
//     r' = 1   where m = (r == 1.0f), alpha else  (alpha = 2*(double)label - 1)
// the score at offset o (sum over the overlap j in [max(0,-o), min(S, R-o)) of s'[j]*r'[j+o]) is
//     score = hi*c11 - c01 + (hi*alpha)*c10 - alpha*c00
// where c_um counts the overlap frames with subtitle bit u and reference bit m.  All four counts follow
// from n_ov (overlap length), Uov (subtitle bits in the overlap), Mwin (reference bits under it) and
//     UM(o) = sum over runs [a, b) of ( M(b + o) - M(a + o) ),   M(p) = reference bits below p, p clamped to [0, R]
// UM is the heavy term: (2 x runs) x (offsets).  A thread owns 32 consecutive offsets o0 .. o0+31.  For an
// endpoint e it loads the 32 reference bits starting at e + o0 (one funnel shift of two words) and
// M(e + o0) (per-word prefix + popcount), so that M(e + o0 + i) = M(e + o0) + (bits t < i of the window):
// the per-bit sums over all endpoints are kept in 4-bit counters, eight to a register (SWAR), and the
// 32 offsets' UM values are their prefix sums.
#pragma once
#include <math.h>
#include <stdint.h>

#include <cuda_runtime.h>

#ifdef __CUDACC__
#define RC_HD __host__ __device__ __forceinline__
#else
#define RC_HD inline
#endif

namespace runcorr {

constexpr int kOffsetsPerThread = 32;
constexpr int kMaxThreads = 1024;
constexpr int kMaxWindow = kOffsetsPerThread * kMaxThreads;  // widest window one CTA covers
// 4-bit counters gain at most 2 per run (the end's bit and the start's complemented bit): 7 runs fit
constexpr int kRunsPerFlush = 7;

RC_HD uint32_t rc_funnel_r(uint32_t lo, uint32_t hi, int s) {  // bits s .. s+31 of (hi:lo), 0 <= s < 32
#ifdef __CUDA_ARCH__
  return __funnelshift_r(lo, hi, (unsigned)s);
#else
  return s == 0 ? lo : (lo >> s) | (hi << (32 - s));
#endif
}

RC_HD int rc_popc(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}

RC_HD uint2 rc_load(const uint2* p) {
#ifdef __CUDA_ARCH__
  return __ldg(p);
#else
  return *p;
#endif
}

// Packed reference of one video: q[w + 1] = (bits of word w, reference bits below word w) for
// w = -1 .. (R >> 5) + 1, i.e. (R >> 5) + 3 entries; bit t of word w is m[32 w + t] (0 outside [0, R)).
RC_HD long long rc_ref_entries(int R) { return (long long)(R >> 5) + 3; }

// The 32 reference bits at p .. p+31 (bit t = m[p + t], zero outside [0, R)) and M(p), for any p.
// p is clamped to [-32, R] before any load: below -32 the window is all zero and M = 0 (as at -32),
// above R the window is all zero and M = M(R) (as at R).  So q[0] .. q[(R >> 5) + 2] are the only
// entries ever read.
RC_HD void rc_ref_window(const uint2* q, int R, int p, uint32_t& win, int& pre) {
  p = p < -32 ? -32 : (p > R ? R : p);
  const int w = p >> 5, s = p & 31;  // arithmetic shift: w >= -1
  const uint2 a = rc_load(q + w + 1), b = rc_load(q + w + 2);
  win = rc_funnel_r(a.x, b.x, s);
  pre = (int)a.y + rc_popc(a.x & ((1u << s) - 1u));
}

RC_HD int rc_ref_prefix(const uint2* q, int R, int p) {
  uint32_t w;
  int pre;
  rc_ref_window(q, R, p, w, pre);
  return pre;
}

// Per-thread accumulation of UM over the runs [ra[r], rb[r]) for the offsets o0 .. o0+31:
// UM(o0 + i) = base + sum_{t < i} cnt[t] - i * nr on return.
RC_HD void rc_flush(uint32_t (&nib)[4], int (&cnt)[32]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int i = 0; i < 8; ++i) cnt[4 * i + k] += (int)((nib[k] >> (4 * i)) & 15u);
    nib[k] = 0;
  }
}

RC_HD void rc_thread_counts(const uint2* q, int R, const int* ra, const int* rb, int nr, int o0, int (&cnt)[32],
                            int& base) {
#pragma unroll
  for (int t = 0; t < 32; ++t) cnt[t] = 0;
  uint32_t nib[4] = {0u, 0u, 0u, 0u};
  base = 0;
  int r = 0;
  while (r < nr) {
    const int r_end = nr - r < kRunsPerFlush ? nr : r + kRunsPerFlush;
    for (; r < r_end; ++r) {
      const int a = ra[r], b = rb[r];
      uint32_t wa, wb;
      int pa, pb;
      rc_ref_window(q, R, a + o0, wa, pa);
      rc_ref_window(q, R, b + o0, wb, pb);
      base += pb - pa;
      wa = ~wa;  // the start counts -bit = (1 - bit) - 1; the -1s are taken out as i * nr below
#pragma unroll
      for (int k = 0; k < 4; ++k) nib[k] += ((wb >> k) & 0x11111111u) + ((wa >> k) & 0x11111111u);
    }
    rc_flush(nib, cnt);
  }
}

// U(x): subtitle bits below frame x (runs sorted, rc[r] = total length of the runs before r).
RC_HD int rc_sub_prefix(const int* ra, const int* rb, const int* rc, int nr, int x) {
  int lo = 0, hi = nr;  // first run with ra >= x
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ra[mid] < x) lo = mid + 1;
    else hi = mid;
  }
  if (lo == 0) return 0;
  const int e = rb[lo - 1] < x ? rb[lo - 1] : x;
  return rc[lo - 1] + e - ra[lo - 1];
}

struct RcLevels {
  double hi, alpha, hia;  // 2*level - 1, 2*label - 1, hi*alpha
};

RC_HD RcLevels rc_levels(float sub_level, float ref_label) {
  RcLevels l;
  l.hi = 2.0 * (double)sub_level - 1.0;
  l.alpha = 2.0 * (double)ref_label - 1.0;
  l.hia = l.hi * l.alpha;
  return l;
}

// The score at offset o from UM(o); the other three counts from prefix sums.
RC_HD double rc_score(const uint2* q, int R, int S, const int* ra, const int* rb, const int* rc, int nr, int o,
                      int um, const RcLevels& l) {
  const int j_lo = o < 0 ? -o : 0;
  const int j_hi = S < R - o ? S : R - o;
  if (j_hi <= j_lo) return 0.0;
  const int n_ov = j_hi - j_lo;
  const int mw = rc_ref_prefix(q, R, j_hi + o) - rc_ref_prefix(q, R, j_lo + o);
  const int uo = rc_sub_prefix(ra, rb, rc, nr, j_hi) - rc_sub_prefix(ra, rb, rc, nr, j_lo);
  const double c11 = um, c01 = mw - um, c10 = uo - um, c00 = n_ov - mw - uo + um;
  return (l.hi * c11 - c01) + (l.hia * c10 - l.alpha * c00);
}

// Nomination margin epsilon of a job whose overlaps have at most n frames (n = min(R, S)).  With
// c = max|s'| * max|r'| and u = 2^-53:
//   rescore_kernel's float64 sum (fma per term, exact products, summation depth <= n + 25 including the
//   256-lane tree and pick_kernel's 16 partials) is within gamma_{n+32} * n * c of the exact sum;
//   rc_score is within 6u * n * c of it (four products, one rounded hi*alpha, three additions) and its
//   result and the cut max - eps each round by at most 2u * n * c.
// An offset that attains the re-scored maximum is therefore at most 2 * (gamma + 8u) * n * c below the
// largest rc_score, the factor 2 because the maximum's own offset carries the same errors.  Padded by 1 %.
RC_HD double rc_eps(double n, const RcLevels& l) {
  const double u = 1.1102230246251565e-16;
  const double ah = fabs(l.hi), aa = fabs(l.alpha);
  const double c = (ah > 1.0 ? ah : 1.0) * (aa > 1.0 ? aa : 1.0);
  const double k = n + 32.0;
  const double gamma = k * u / (1.0 - k * u);
  return 2.02 * (gamma + 8.0 * u) * n * c;
}

}  // namespace runcorr
