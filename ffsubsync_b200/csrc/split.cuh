// Per-segment offsets with a split penalty (csrc/split.cu, DESIGN.md section 4 "K9s"): the arithmetic shared by
// the kernels and their CPU emulations (tests/host_emul/split_emul.cu, split_cluster_emul.cu, split_capped_emul.cu,
// split_directed_emul.cu, split_breaks_emul.cu).
//
// A track's subtitle mask (S frames, runs [a_k, b_k) of 1s) is cut into units: unit j is the gap before run j
// and run j, [start_j, end_j) with start_0 = 0, start_j = b_{j-1}, end_j = b_j, except that the last unit ends at
// S (a mask without runs is one unit [0, S)).  At offset o (subtitle frame f meets reference frame f + o) unit j
// contributes the run path's four-count score over its frames of the overlap [max(0, -o), min(S, R - o)):
//     u_j(o) = (hi*c11 - c01) + (hia*c10 - alpha*c00)
// with hi = 2*(double)level - 1, alpha = 2*beta - 1, hia = hi*alpha (runcorr.cuh's rc_levels).  With M(p) the
// reference bits below p, p clamped to [0, R] (rc_ref_window):
//     n_ov = |[start, end) n [-o, R - o)|,  mw = M(end + o) - M(start + o),
//     uo   = |[a, b) n [-o, R - o)|,        um = M(b + o) - M(a + o)
// (frames outside [0, R) have no reference bit), c11 = um, c01 = mw - um, c10 = uo - um,
// c00 = n_ov - mw - uo + um.  The units' contributions add up to the whole track's score at o.
// The programme over units j = 0 .. n-1 (lambda = split_penalty >= 0):
//     V_0(o) = u_0(o),   V_j(o) = u_j(o) + max(V_{j-1}(o), M_{j-1} - lambda),   M_j = max_o V_j(o)
// in float64 with every operation rounded on its own (no contraction): c = M_{j-1} - lambda, then the
// switch decision c > V_{j-1}(o) (staying wins a tie), then u_j(o) + (switch ? c : V_{j-1}(o)).  The argmax of
// each unit is its largest offset attaining M_j.  With +-1 signals (level 1, label 0) every value is an integer
// below 2^53, so every cell is exact.
#pragma once
#include "runcorr.cuh"

#ifdef __CUDACC__
#define SP_HD __host__ __device__ __forceinline__
#else
#define SP_HD inline
#endif

namespace split {

using runcorr::kOffsetsPerThread;
constexpr int kMaxWindow = runcorr::kMaxWindow;  // b2_split_tracks' envelope
constexpr int kMaxRuns = 16384;                  // runs of one track (shared memory of the run table)
// A track is one thread-block cluster of C CTAs of at most kCtaThreads threads (32 float64 V each stay in registers
// at 128 registers a thread); cluster thread g = rank * blockDim + tid owns the offsets o_lo + 32 g .. + 31.
constexpr int kCtaThreads = 512;
constexpr int kCtaWindow = kOffsetsPerThread * kCtaThreads;  // offsets of one CTA: C = ceil(W / kCtaWindow)
constexpr int kMaxCluster = 16;                              // non-portable past 8
// b2_split_tracks_capped: at most kMaxSegments layers, one cluster of N x C CTAs per track (N x C <= the widest
// cluster of split_capped_dp_kernel the device co-schedules)
constexpr int kMaxSegments = 16;

SP_HD double sp_add(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
SP_HD double sp_sub(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
SP_HD double sp_mul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

struct SpLevels {
  double hi, alpha, hia;
};

// level: the track's subtitle level (float)min(1/x, 1); beta: the reference's level other than 1.0
SP_HD SpLevels sp_levels(float level, double beta) {
  SpLevels l;
  l.hi = sp_sub(sp_mul(2.0, (double)level), 1.0);
  l.alpha = sp_sub(sp_mul(2.0, beta), 1.0);
  l.hia = sp_mul(l.hi, l.alpha);
  return l;
}

// Unit j of nr runs: [start, end) holding the run [a, b) (a = b = 0 for the one unit of a mask without runs)
struct SpUnit {
  int start, a, b, end;
};

SP_HD SpUnit sp_unit(const int* ra, const int* rb, int nr, int S, int j) {
  SpUnit u;
  if (nr == 0) {
    u.start = 0;
    u.a = 0;
    u.b = 0;
    u.end = S;
    return u;
  }
  u.start = j == 0 ? 0 : rb[j - 1];
  u.a = ra[j];
  u.b = rb[j];
  u.end = j == nr - 1 ? S : rb[j];
  return u;
}

SP_HD int sp_overlap(int lo, int hi, int o, int R) {  // |[lo, hi) n [-o, R - o)|
  const int x = lo > -o ? lo : -o;
  const int y = hi < R - o ? hi : R - o;
  return y > x ? y - x : 0;
}

// u_j(o) from the unit and the four reference prefixes M(start + o), M(a + o), M(b + o), M(end + o)
SP_HD double sp_score(const SpUnit& u, int o, int R, int m_start, int m_a, int m_b, int m_end, const SpLevels& l) {
  const int n_ov = sp_overlap(u.start, u.end, o, R);
  if (n_ov == 0) return 0.0;
  const int mw = m_end - m_start, um = m_b - m_a, uo = sp_overlap(u.a, u.b, o, R);
  const double c11 = um, c01 = mw - um, c10 = uo - um, c00 = n_ov - mw - uo + um;
  return sp_add(sp_sub(sp_mul(l.hi, c11), c01), sp_sub(sp_mul(l.hia, c10), sp_mul(l.alpha, c00)));
}

// u_j(o) at one offset (the backtrack's re-score of the chosen path)
SP_HD double sp_unit_score(const uint2* q, int R, const SpUnit& u, int o, const SpLevels& l) {
  using runcorr::rc_ref_prefix;
  return sp_score(u, o, R, rc_ref_prefix(q, R, u.start + o), rc_ref_prefix(q, R, u.a + o),
                  rc_ref_prefix(q, R, u.b + o), rc_ref_prefix(q, R, u.end + o), l);
}

// One thread's step of the programme over its offsets o0 .. o0 + n_mine - 1 (n_mine <= 32) for one unit:
// the four prefixes of all 32 offsets come from one funnel-shifted window and one word prefix per endpoint.
// first: unit 0 (V = u).  Otherwise c = M_{j-1} - lambda and bit i of the returned word is set when offset
// o0 + i switched.  v[i] becomes V_j(o0 + i); best / barg: the thread's maximum and its largest offset.
SP_HD uint32_t sp_thread_step(const uint2* q, int R, const SpUnit& u, int o0, int n_mine, bool first, double c,
                              const SpLevels& l, double (&v)[32], double& best, int& barg) {
  uint32_t w_s, w_a, w_b, w_e;
  int p_s, p_a, p_b, p_e;
  runcorr::rc_ref_window(q, R, u.start + o0, w_s, p_s);
  runcorr::rc_ref_window(q, R, u.a + o0, w_a, p_a);
  runcorr::rc_ref_window(q, R, u.b + o0, w_b, p_b);
  runcorr::rc_ref_window(q, R, u.end + o0, w_e, p_e);
  uint32_t dec = 0;
  best = -INFINITY;
  barg = -2147483647 - 1;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    if (i < n_mine) {
      const uint32_t below = (1u << i) - 1u;
      const double s = sp_score(u, o0 + i, R, p_s + runcorr::rc_popc(w_s & below), p_a + runcorr::rc_popc(w_a & below),
                                p_b + runcorr::rc_popc(w_b & below), p_e + runcorr::rc_popc(w_e & below), l);
      double x;
      if (first) {
        x = s;
      } else {
        const bool sw = c > v[i];
        dec |= (uint32_t)sw << i;
        x = sp_add(s, sw ? c : v[i]);
      }
      v[i] = x;
      if (x >= best) {  // increasing offsets: ties go to the largest
        best = x;
        barg = o0 + i;
      }
    }
  }
  return dec;
}

// The directed programme (b2_split_tracks_directed, direction kDir = +1 or -1): a switch at o may only come from an
// offset on the kDir side behind it,
//     P_{j-1}(o) = max { V_{j-1}(o') : o' < o }  (kDir = +1; o' > o for kDir = -1, -inf when empty)
//     c = P_{j-1}(o) - lambda,   switch = c > V_{j-1}(o),   V_j(o) = u_j(o) + (switch ? c : V_{j-1}(o))
// with the rounding of sp_thread_step.  p: the exclusive prefix (kDir = -1: suffix) maximum of V_{j-1} over the
// offsets before o0 (after o0 + n_mine - 1); the thread walks its offsets in the direction's order with a running
// maximum of the old values.  Bit i of rec is set when V_{j-1}(o0 + i) is a record: >= everything before it
// (kDir = +1), > everything after it (kDir = -1); a switch's source is the nearest record behind it.  Bit i of the
// returned word is set when o0 + i switched; best / barg as sp_thread_step.
template <int kDir>
SP_HD uint32_t sp_thread_step_dir(const uint2* q, int R, const SpUnit& u, int o0, int n_mine, bool first, double p,
                                  double penalty, const SpLevels& l, double (&v)[32], double& best, int& barg,
                                  uint32_t& rec) {
  uint32_t w_s, w_a, w_b, w_e;
  int p_s, p_a, p_b, p_e;
  runcorr::rc_ref_window(q, R, u.start + o0, w_s, p_s);
  runcorr::rc_ref_window(q, R, u.a + o0, w_a, p_a);
  runcorr::rc_ref_window(q, R, u.b + o0, w_b, p_b);
  runcorr::rc_ref_window(q, R, u.end + o0, w_e, p_e);
  uint32_t dec = 0, rb = 0;
  best = -INFINITY;
  barg = -2147483647 - 1;
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const int i = kDir > 0 ? k : 31 - k;
    if (i < n_mine) {
      const uint32_t below = (1u << i) - 1u;
      const double s = sp_score(u, o0 + i, R, p_s + runcorr::rc_popc(w_s & below), p_a + runcorr::rc_popc(w_a & below),
                                p_b + runcorr::rc_popc(w_b & below), p_e + runcorr::rc_popc(w_e & below), l);
      double x;
      if (first) {
        x = s;
      } else {
        const double old = v[i];
        rb |= (uint32_t)(kDir > 0 ? old >= p : old > p) << i;
        const double c = sp_sub(p, penalty);
        const bool sw = c > old;
        dec |= (uint32_t)sw << i;
        x = sp_add(s, sw ? c : old);
        p = old > p ? old : p;
      }
      v[i] = x;
      if (kDir > 0 ? x >= best : x > best) {  // ties go to the largest offset in either walk
        best = x;
        barg = o0 + i;
      }
    }
  }
  rec = rb;
  return dec;
}

// The programme along stated breaks (b2_split_tracks_breaks, breaks d_1 .. d_n, each +1 or -1, 1 <= n <= kMaxBreaks):
// layer m holds the paths with exactly m breaks, the i-th break moving the offset strictly up (d_i = +1) or down (-1),
//     V_{0,0} = u_0,  V_{0,m} = -inf (m >= 1);  V_{j,0} = u_j + V_{j-1,0}  (layer 0 never switches)
//     c = P^{d_m}_{j-1,m-1}(o) - lambda,   V_{j,m}(o) = u_j(o) + (c > V_{j-1,m}(o) ? c : V_{j-1,m}(o))  (m >= 1)
// with P^{+1} the exclusive prefix maximum over o' < o, P^{-1} the exclusive suffix maximum over o' > o (-inf when
// empty), each operation rounded on its own as in sp_thread_step_dir.  A break's source is the nearest record of
// V_{j-1,m-1} on the d_m side (sp_thread_step_dir's record rule), so no row is stored.
constexpr int kMaxBreaks = 15;

// One cell of a layer m >= 1 in the walk of its break (kUp: d_m = +1): old = V_{j-1,m-1}(o), cur = V_{j-1,m}(o) becomes
// V_{j,m}(o); pm, the maximum of V_{j-1,m-1} behind o, takes old in.  bit: the cell's bit in the switch and record words.
template <bool kUp>
SP_HD void sp_break_cell(double s, double old, double& cur, double& pm, double penalty, int bit, uint32_t& d,
                         uint32_t& r) {
  r |= (uint32_t)(kUp ? old >= pm : old > pm) << bit;
  const double c = sp_sub(pm, penalty);
  const bool sw = c > cur;
  d |= (uint32_t)sw << bit;
  cur = sp_add(s, sw ? c : cur);
  pm = old > pm ? old : pm;
}

// One thread's step over its kM offsets o0 .. o0 + n_mine - 1 for all layers 0 .. nb (nb + 1 <= kL, kL x kM <= 32) of
// one unit: u_j is scored once per offset, then the layers are updated from the top down (layer m reads the old values
// of layer m - 1), each walking the offsets in its break's order; layer 0 (which never switches, and whose old values
// only layer 1 reads) is updated inside layer 1's walk.  With two layers that walk is the only one and scores u_j
// itself.  up: bit m set when d_m = +1.  p[m] (m >= 1): the maximum of V_{j-1,m-1} over the offsets on the d_m side
// behind this thread's.  first: unit 0.  v[m][i] = V_{j,m}(o0 + i); offsets past n_mine and layers past nb keep -inf.
// Bit m * kM + i of sw is set when o0 + i switched into layer m, of rec when V_{j-1,m-1}(o0 + i) is a record on the d_m
// side (>= all before it for +1, > all after it for -1).
template <int kL, int kM>
SP_HD void sp_thread_step_breaks(const uint2* q, int R, const SpUnit& u, int o0, int n_mine, bool first, int nb,
                                 uint32_t up, const double (&p)[kL], double penalty, const SpLevels& l,
                                 double (&v)[kL][kM], uint32_t& sw, uint32_t& rec) {
  static_assert(kL * kM <= 32, "one bit per layer and offset");
  constexpr bool kStore = kL > 2;  // more than one walk reads u_j
  uint32_t w_s, w_a, w_b, w_e;
  int p_s, p_a, p_b, p_e;
  runcorr::rc_ref_window(q, R, u.start + o0, w_s, p_s);
  runcorr::rc_ref_window(q, R, u.a + o0, w_a, p_a);
  runcorr::rc_ref_window(q, R, u.b + o0, w_b, p_b);
  runcorr::rc_ref_window(q, R, u.end + o0, w_e, p_e);
  auto score = [&](int i) {
    const uint32_t below = (1u << i) - 1u;
    return sp_score(u, o0 + i, R, p_s + runcorr::rc_popc(w_s & below), p_a + runcorr::rc_popc(w_a & below),
                    p_b + runcorr::rc_popc(w_b & below), p_e + runcorr::rc_popc(w_e & below), l);
  };
  double s[kStore ? kM : 1];
  if constexpr (kStore) {
#pragma unroll
    for (int i = 0; i < kM; ++i) s[i] = i < n_mine ? score(i) : 0.0;
  }
  uint32_t d = 0, r = 0;
  if (first) {
#pragma unroll
    for (int i = 0; i < kM; ++i) {
      if (i < n_mine) {
        if constexpr (kStore) v[0][i] = s[i];
        else v[0][i] = score(i);
      }
    }
    sw = 0;
    rec = 0;
    return;
  }
  if constexpr (kStore) {
#pragma unroll
    for (int m = kL - 1; m >= 2; --m) {
      if (m > nb) continue;
      double pm = p[m];
      if ((up >> m) & 1u) {  // both walks unrolled, so every register index is a constant
#pragma unroll
        for (int i = 0; i < kM; ++i)
          if (i < n_mine) sp_break_cell<true>(s[i], v[m - 1][i], v[m][i], pm, penalty, m * kM + i, d, r);
      } else {
#pragma unroll
        for (int i = kM - 1; i >= 0; --i)
          if (i < n_mine) sp_break_cell<false>(s[i], v[m - 1][i], v[m][i], pm, penalty, m * kM + i, d, r);
      }
    }
  }
  double pm = p[1];  // layer 1 (nb >= 1), then layer 0 at each offset once layer 1 has read its old value
  if (up & 2u) {
#pragma unroll
    for (int i = 0; i < kM; ++i) {
      if (i < n_mine) {
        double si;
        if constexpr (kStore) si = s[i];
        else si = score(i);
        sp_break_cell<true>(si, v[0][i], v[1][i], pm, penalty, kM + i, d, r);
        v[0][i] = sp_add(si, v[0][i]);
      }
    }
  } else {
#pragma unroll
    for (int i = kM - 1; i >= 0; --i) {
      if (i < n_mine) {
        double si;
        if constexpr (kStore) si = s[i];
        else si = score(i);
        sp_break_cell<false>(si, v[0][i], v[1][i], pm, penalty, kM + i, d, r);
        v[0][i] = sp_add(si, v[0][i]);
      }
    }
  }
  sw = d;
  rec = r;
}

// One step of the unit maximum over candidates (warp lanes, a CTA's warps, a cluster's CTAs): the larger value, and
// among equal values the larger offset, so the merge gives np.argmax over the reversed window in any order.
SP_HD void sp_merge(double& best, int& barg, double ob, int oa) {
  if (ob > best || (ob == best && oa > barg)) {
    best = ob;
    barg = oa;
  }
}

}  // namespace split
