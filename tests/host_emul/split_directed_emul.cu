// CPU emulation of split_directed_dp_kernel, one track on a thread-block cluster of C CTAs (the directed split,
// ffsubsync_b200/csrc/split.cu and split.cuh): the same __host__ __device__ functions run for every thread of every
// CTA, one after the other, between the kernel's barriers, and the kernel's exclusive scan of the thread maxima is
// restated level by level (lanes, then the warps' slots after the CTA barrier, then the CTAs' slots after the cluster
// barrier).  Test infrastructure; tests/test_split_directed_cpu.py drives it.
//
// usage: split_directed_emul in.bin out.bin direction C cta_threads [dead]
// in.bin : int32 R, S, o_lo, W ; float32 level ; float64 beta, penalty ; uint8 m[R] (0/1) ; uint8 sub[S] (0/1)
// out.bin: int32 n_units ; per unit: float64 max (the scan's total) ; int32 argmax of the last unit ;
//          per unit j >= 1: uint8 switch[W], uint8 record[W] (the records of V_{j-1}) ; int32 C ;
//          per CTA: int32 CTA barriers, int32 cluster barriers, as the kernel's control flow runs them
// Cluster thread g = rank * cta_threads + tid owns the offsets o_lo + 32 g .. (CTAs past the window own none).  C = 1
// is the kernel's plain launch (no cluster barrier).  dead: the track the kernel skips: n_units 0 and no barrier in
// any CTA.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "../../ffsubsync_b200/csrc/split.cuh"

using namespace split;

struct CtaCount {  // barriers one CTA ran
  int cta = 0, cluster = 0;
};

// rc_decode_runs' barriers for an S-frame mask in a CTA of n threads (three per pass over the words)
static int decode_barriers(int S, int n) { return 3 * ((S >> 5) / n + 1); }

static double dmax(double a, double b) { return b > a ? b : a; }

template <int kDir>
static void run(const uint2* q, int R, int S, int o_lo, int W, float level, double beta, double pen, int C, int nt,
                const std::vector<int>& ra, const std::vector<int>& rb, std::vector<CtaCount>& cnt,
                std::vector<double>& mxs, int& last_arg, std::vector<unsigned char>& sw,
                std::vector<unsigned char>& rc, int& nu) {
  const int nr = (int)ra.size(), nw = nt / 32, G = C * nt;
  nu = nr > 0 ? nr : 1;
  for (int r = 0; r < C; ++r) cnt[r].cta += decode_barriers(S, nt) + 1;
  const SpLevels l = sp_levels(level, beta);
  std::vector<double> v((size_t)G * 32), p(G, -INFINITY), tb(G), lane_ex(G), warp_tot((size_t)C * nw),
      cta_tot(C);
  std::vector<int> targ(G), warp_arg((size_t)C * nw), cta_arg(C);
  mxs.assign(nu, 0.0);
  sw.assign((size_t)nu * W, 0);
  rc.assign((size_t)nu * W, 0);
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra.data(), rb.data(), nr, S, j);
    const bool last = j == nu - 1;
    for (int g = 0; g < G; ++g) {  // every thread's step
      const int n_mine = std::max(0, std::min(kOffsetsPerThread, W - kOffsetsPerThread * g));
      double best = -INFINITY;
      int barg = -2147483647 - 1;
      if (n_mine > 0) {
        uint32_t rec = 0;
        double (&vt)[32] = *reinterpret_cast<double(*)[32]>(&v[(size_t)g * 32]);
        const uint32_t d = sp_thread_step_dir<kDir>(q, R, u, o_lo + kOffsetsPerThread * g, n_mine, j == 0, p[g], pen,
                                                    l, vt, best, barg, rec);
        for (int i = 0; i < n_mine; ++i) {
          sw[(size_t)j * W + kOffsetsPerThread * g + i] = (d >> i) & 1u;
          rc[(size_t)j * W + kOffsetsPerThread * g + i] = (rec >> i) & 1u;
        }
      }
      tb[g] = best;
      targ[g] = barg;
    }
    for (int r = 0; r < C; ++r) {  // each CTA up to its CTA barrier: the lanes' scan and the warps' slots
      for (int w = 0; w < nw; ++w) {
        const int g0 = r * nt + 32 * w;
        double tot = -INFINITY, wb = -INFINITY;
        int am = -2147483647 - 1;
        for (int k = 0; k < 32; ++k) {  // lanes in the direction's order
          const int lane = kDir > 0 ? k : 31 - k;
          lane_ex[g0 + lane] = tot;
          tot = dmax(tot, tb[g0 + lane]);
          sp_merge(wb, am, tb[g0 + lane], targ[g0 + lane]);  // the warp's argmax (the kernel: at the last unit)
        }
        warp_tot[(size_t)r * nw + w] = tot;
        warp_arg[(size_t)r * nw + w] = am;
      }
      ++cnt[r].cta;
      double mx = -INFINITY;
      int am = -2147483647 - 1;
      for (int w = 0; w < nw; ++w) sp_merge(mx, am, warp_tot[(size_t)r * nw + w], warp_arg[(size_t)r * nw + w]);
      cta_tot[r] = mx;
      cta_arg[r] = am;
      if (C > 1) ++cnt[r].cluster;
    }
    double mx = -INFINITY;
    int am = -2147483647 - 1;
    for (int r = 0; r < C; ++r) sp_merge(mx, am, cta_tot[r], cta_arg[r]);
    mxs[j] = mx;
    if (last) last_arg = am;
    for (int g = 0; g < G; ++g) {  // after the barriers: the warps and the CTAs on the kDir side behind
      const int r = g / nt, w = (g % nt) / 32;
      double ex = lane_ex[g];
      for (int x = kDir > 0 ? 0 : w + 1; x < (kDir > 0 ? w : nw); ++x) ex = dmax(ex, warp_tot[(size_t)r * nw + x]);
      for (int x = kDir > 0 ? 0 : r + 1; x < (kDir > 0 ? r : C); ++x) ex = dmax(ex, cta_tot[x]);
      p[g] = ex;
    }
  }
  if (C > 1)
    for (int r = 0; r < C; ++r) ++cnt[r].cluster;  // the final barrier before any CTA exits
}

int main(int argc, char** argv) {
  if (argc != 6 && argc != 7) return 2;
  const int dir = atoi(argv[3]), C = atoi(argv[4]), nt = atoi(argv[5]);
  const bool dead = argc == 7 && atoi(argv[6]) != 0;
  if ((dir != 1 && dir != -1) || C < 1 || C > kMaxCluster || nt < 32 || nt > kCtaThreads || nt % 32) return 5;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  int hdr[4];
  float level;
  double bp[2];
  if (fread(hdr, 4, 4, f) != 4 || fread(&level, 4, 1, f) != 1 || fread(bp, 8, 2, f) != 2) return 4;
  const int R = hdr[0], S = hdr[1], o_lo = hdr[2], W = hdr[3];
  std::vector<unsigned char> m(R), sub(S);
  if (fread(m.data(), 1, R, f) != (size_t)R || fread(sub.data(), 1, S, f) != (size_t)S) return 4;
  fclose(f);
  if (W < 1 || W > C * nt * kOffsetsPerThread) return 5;
  // packed reference as split_ref_kernel writes it, between poison entries (every bit set, a huge prefix)
  constexpr int kPoison = 64;
  const long long n_q = runcorr::rc_ref_entries(R);
  std::vector<uint2> q_guarded(n_q + 2 * kPoison, make_uint2(0xffffffffu, 0x40000000u));
  uint2* q = q_guarded.data() + kPoison;
  q[0] = make_uint2(0u, 0u);
  int below = 0;
  for (int w = 0; w <= (R >> 5) + 1; ++w) {
    uint32_t bits = 0;
    for (int t = 0; t < 32; ++t) {
      const long long i = 32LL * w + t;
      if (i < R && m[i]) bits |= 1u << t;
    }
    q[w + 1] = make_uint2(bits, (uint32_t)below);
    below += __builtin_popcount(bits);
  }
  std::vector<int> ra, rb;
  for (int j = 0; j < S;) {
    if (!sub[j]) {
      ++j;
      continue;
    }
    int e = j;
    while (e < S && sub[e]) ++e;
    ra.push_back(j);
    rb.push_back(e);
    j = e;
  }
  std::vector<CtaCount> cnt(C);
  std::vector<double> mxs;
  std::vector<unsigned char> sw, rc;
  int nu = 0, last_arg = 0;
  if (!dead) {  // the early exit is the track's: every CTA takes it, before any barrier
    if (dir > 0)
      run<1>(q, R, S, o_lo, W, level, bp[0], bp[1], C, nt, ra, rb, cnt, mxs, last_arg, sw, rc, nu);
    else
      run<-1>(q, R, S, o_lo, W, level, bp[0], bp[1], C, nt, ra, rb, cnt, mxs, last_arg, sw, rc, nu);
  }
  f = fopen(argv[2], "wb");
  fwrite(&nu, 4, 1, f);
  if (nu > 0) fwrite(mxs.data(), 8, nu, f);
  fwrite(&last_arg, 4, 1, f);
  for (int j = 1; j < nu; ++j) {
    fwrite(sw.data() + (size_t)j * W, 1, W, f);
    fwrite(rc.data() + (size_t)j * W, 1, W, f);
  }
  fwrite(&C, 4, 1, f);
  for (int r = 0; r < C; ++r) {
    fwrite(&cnt[r].cta, 4, 1, f);
    fwrite(&cnt[r].cluster, 4, 1, f);
  }
  fclose(f);
  return 0;
}
