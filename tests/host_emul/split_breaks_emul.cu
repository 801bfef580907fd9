// CPU emulation of split_breaks_dp_kernel<kM>, one track on a thread-block cluster of C CTAs (the split along stated
// breaks, ffsubsync_b200/csrc/split.cu and split.cuh): sp_thread_step_breaks runs for every thread of every CTA, one
// after the other, between the kernel's barriers, and the kernel's per-layer exclusive scans of the thread maxima are
// restated level by level (lanes, then the warps' slots after the CTA barrier, then the CTAs' slots after the cluster
// barrier), as is the last unit's per-layer maximum and argmax.  Test infrastructure; tests/test_split_breaks_cpu.py
// drives it.
//
// usage: split_breaks_emul in.bin out.bin C cta_threads [dead]
// in.bin : int32 R, S, o_lo, W, nb ; int32 breaks[nb] ; float32 level ; float64 beta, penalty ; uint8 m[R] (0/1) ;
//          uint8 sub[S] (0/1)
// out.bin: int32 n_units, int32 kM ; float64 profile[nb + 1] ; int32 argmax[nb + 1] (the last unit's) ;
//          per unit j >= 1 and layer m = 1 .. nb: uint8 switch[W], uint8 record[W] ; int32 C ;
//          per CTA: int32 CTA barriers, int32 cluster barriers, as the kernel's control flow runs them
// Cluster thread g = rank * cta_threads + tid owns the kM = 32 / (nb + 1) offsets o_lo + kM g .. (CTAs past the window
// own none).  Every launch is a cluster launch, so C = 1 runs cluster barriers too.  dead: the track the kernel skips:
// n_units 0 and no barrier in any CTA.
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

struct Out {
  int nu = 0;
  std::vector<double> profile;
  std::vector<int> arg;
  std::vector<unsigned char> sw, rc;  // [unit][layer][offset]
};

template <int kM>
static void run(const uint2* q, int R, int S, int o_lo, int W, int nb, uint32_t up, float level, double beta,
                double pen, int C, int nt, const std::vector<int>& ra, const std::vector<int>& rb,
                std::vector<CtaCount>& cnt, Out& out) {
  constexpr int kL = 32 / kM;
  const int nr = (int)ra.size(), nw = nt / 32, G = C * nt, L = nb + 1;
  const int nu = nr > 0 ? nr : 1;
  out.nu = nu;
  for (int r = 0; r < C; ++r) cnt[r].cta += decode_barriers(S, nt) + 1;
  const SpLevels l = sp_levels(level, beta);
  struct Thread {
    double v[kL][kM];
    double p[kL];
  };
  std::vector<Thread> th(G);
  for (auto& x : th)
    for (int m = 0; m < kL; ++m) {
      x.p[m] = -INFINITY;
      for (int i = 0; i < kM; ++i) x.v[m][i] = -INFINITY;
    }
  std::vector<double> tot(G), lane_ex(G), warp_tot((size_t)C * nw), cta_tot(C);
  out.sw.assign((size_t)nu * L * W, 0);
  out.rc.assign((size_t)nu * L * W, 0);
  out.profile.assign(L, 0.0);
  out.arg.assign(L, 0);
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra.data(), rb.data(), nr, S, j);
    for (int g = 0; g < G; ++g) {  // every thread's step
      const int n_mine = std::max(0, std::min(kM, W - kM * g));
      if (n_mine <= 0) continue;
      uint32_t d = 0, rec = 0;
      sp_thread_step_breaks<kL, kM>(q, R, u, o_lo + kM * g, n_mine, j == 0, nb, up, th[g].p, pen, l, th[g].v, d, rec);
      for (int m = 1; m < L; ++m)
        for (int i = 0; i < n_mine; ++i) {
          out.sw[((size_t)j * L + m) * W + kM * g + i] = (d >> (m * kM + i)) & 1u;
          out.rc[((size_t)j * L + m) * W + kM * g + i] = (rec >> (m * kM + i)) & 1u;
        }
    }
    for (int r = 0; r < C; ++r) ++cnt[r].cta;  // the unit's CTA barrier
    for (int m = 1; m < L; ++m) {  // layer m's scan of layer m - 1's thread maxima in d_m's order
      const bool fwd = (up >> m) & 1u;
      for (int g = 0; g < G; ++g) {
        double x = th[g].v[m - 1][0];
        for (int i = 1; i < kM; ++i) x = dmax(x, th[g].v[m - 1][i]);
        tot[g] = x;
      }
      for (int r = 0; r < C; ++r) {
        for (int w = 0; w < nw; ++w) {
          const int g0 = r * nt + 32 * w;
          double run = -INFINITY;
          for (int k = 0; k < 32; ++k) {  // lanes in the direction's order
            const int lane = fwd ? k : 31 - k;
            lane_ex[g0 + lane] = run;
            run = dmax(run, tot[g0 + lane]);
          }
          warp_tot[(size_t)r * nw + w] = run;
        }
        double mx = -INFINITY;
        for (int w = 0; w < nw; ++w) mx = dmax(mx, warp_tot[(size_t)r * nw + w]);
        cta_tot[r] = mx;
      }
      for (int g = 0; g < G; ++g) {  // after the barriers: the warps and the CTAs on the d_m side behind
        const int r = g / nt, w = (g % nt) / 32;
        double ex = lane_ex[g];
        for (int x = fwd ? 0 : w + 1; x < (fwd ? w : nw); ++x) ex = dmax(ex, warp_tot[(size_t)r * nw + x]);
        for (int x = fwd ? 0 : r + 1; x < (fwd ? r : C); ++x) ex = dmax(ex, cta_tot[x]);
        th[g].p[m] = ex;
      }
    }
    if (j == nu - 1)
      for (int m = 0; m < L; ++m) {  // each layer's maximum: threads, lanes, warps and CTAs in any order
        double mx = -INFINITY;
        int am = -2147483647 - 1;
        for (int g = 0; g < G; ++g) {
          const int n_mine = std::max(0, std::min(kM, W - kM * g));
          for (int i = 0; i < n_mine; ++i) sp_merge(mx, am, th[g].v[m][i], o_lo + kM * g + i);
        }
        out.profile[m] = mx;
        out.arg[m] = am;
      }
    for (int r = 0; r < C; ++r) ++cnt[r].cluster;  // the unit's cluster barrier
  }
  for (int r = 0; r < C; ++r) ++cnt[r].cluster;  // the final barrier before any CTA exits
}

int main(int argc, char** argv) {
  if (argc != 5 && argc != 6) return 2;
  const int C = atoi(argv[3]), nt = atoi(argv[4]);
  const bool dead = argc == 6 && atoi(argv[5]) != 0;
  if (C < 1 || C > kMaxCluster || nt < 32 || nt > kCtaThreads || nt % 32) return 5;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  int hdr[5];
  if (fread(hdr, 4, 5, f) != 5) return 4;
  const int R = hdr[0], S = hdr[1], o_lo = hdr[2], W = hdr[3], nb = hdr[4];
  if (nb < 1 || nb > kMaxBreaks) return 5;
  std::vector<int> brk(nb);
  float level;
  double bp[2];
  if (fread(brk.data(), 4, nb, f) != (size_t)nb || fread(&level, 4, 1, f) != 1 || fread(bp, 8, 2, f) != 2) return 4;
  std::vector<unsigned char> m(R), sub(S);
  if (fread(m.data(), 1, R, f) != (size_t)R || fread(sub.data(), 1, S, f) != (size_t)S) return 4;
  fclose(f);
  uint32_t up = 0;
  for (int i = 0; i < nb; ++i) up |= (uint32_t)(brk[i] > 0) << (i + 1);
  const int kM = 32 / (nb + 1);
  if (W < 1 || W > C * nt * kM) return 5;
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
  Out out;
  if (!dead) {  // the early exit is the track's: every CTA takes it, before any barrier
    switch (kM) {
      case 16: run<16>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      case 10: run<10>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      case 8: run<8>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      case 6: run<6>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      case 5: run<5>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      case 4: run<4>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      case 3: run<3>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
      default: run<2>(q, R, S, o_lo, W, nb, up, level, bp[0], bp[1], C, nt, ra, rb, cnt, out); break;
    }
  }
  const int L = nb + 1;
  f = fopen(argv[2], "wb");
  fwrite(&out.nu, 4, 1, f);
  fwrite(&kM, 4, 1, f);
  if (out.nu > 0) {
    fwrite(out.profile.data(), 8, L, f);
    fwrite(out.arg.data(), 4, L, f);
  }
  for (int j = 1; j < out.nu; ++j)
    for (int m = 1; m < L; ++m) {
      fwrite(out.sw.data() + ((size_t)j * L + m) * W, 1, W, f);
      fwrite(out.rc.data() + ((size_t)j * L + m) * W, 1, W, f);
    }
  fwrite(&C, 4, 1, f);
  for (int r = 0; r < C; ++r) {
    fwrite(&cnt[r].cta, 4, 1, f);
    fwrite(&cnt[r].cluster, 4, 1, f);
  }
  fclose(f);
  return 0;
}
