// CPU emulation of split_dp_kernel<true>, one track on a thread-block cluster (ffsubsync_b200/csrc/split.cuh): the
// same __host__ __device__ functions run for every thread of every CTA, one after the other, between the kernel's
// barriers.  Test infrastructure; tests/test_split_wide_cpu.py drives it.
//
// usage: split_cluster_emul in.bin out.bin C cta_threads [dead]
// in.bin : int32 R, S, o_lo, W ; float32 level ; float64 beta, penalty ; uint8 m[R] (0/1) ; uint8 sub[S] (0/1)
// out.bin: int32 n_units ; per unit: float64 max, int32 argmax ; per unit j >= 1: uint8 switch[W] ; int32 C ;
//          per CTA: int32 CTA barriers, int32 cluster barriers, as the kernel's control flow runs them
// A cluster of C CTAs of cta_threads threads: cluster thread g = rank * cta_threads + tid owns the offsets
// o_lo + 32 g .. (CTAs past the window own none); each CTA reduces its warps, publishes its maximum in its slot, and
// after the cluster barrier merges all C slots in rank order, as the kernel does.  dead: the track the kernel skips
// (NaN ratio, empty window, three-level reference): n_units 0 and no barrier in any CTA.
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

int main(int argc, char** argv) {
  if (argc != 5 && argc != 6) return 2;
  const int C = atoi(argv[3]), nt = atoi(argv[4]);
  const bool dead = argc == 6 && atoi(argv[5]) != 0;
  if (C < 1 || C > kMaxCluster || nt < 32 || nt > kCtaThreads || nt % 32) return 5;
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
  std::vector<int> args;
  std::vector<unsigned char> sw;
  int nu = 0;
  if (!dead) {  // the early exit is the track's: every CTA takes it, before any barrier
    const int nr = (int)ra.size();
    nu = nr > 0 ? nr : 1;
    for (int r = 0; r < C; ++r) cnt[r].cta += decode_barriers(S, nt) + 1;
    const SpLevels l = sp_levels(level, bp[0]);
    std::vector<double> v((size_t)C * nt * 32);
    mxs.resize(nu);
    args.resize(nu);
    sw.assign((size_t)nu * W, 0);
    std::vector<double> slot_mx(C);
    std::vector<int> slot_arg(C);
    double c = 0.0;
    for (int j = 0; j < nu; ++j) {
      const SpUnit u = sp_unit(ra.data(), rb.data(), nr, S, j);
      for (int r = 0; r < C; ++r) {  // each CTA up to its cluster barrier
        double cmx = -INFINITY;
        int carg = -2147483647 - 1;
        for (int w = 0; w < nt / 32; ++w) {
          double wmx = -INFINITY;
          int warg = -2147483647 - 1;
          for (int lane = 0; lane < 32; ++lane) {
            const int g = r * nt + 32 * w + lane;
            const int n_mine = std::max(0, std::min(kOffsetsPerThread, W - kOffsetsPerThread * g));
            double best = -INFINITY;
            int barg = -2147483647 - 1;
            if (n_mine > 0) {
              double (&vt)[32] = *reinterpret_cast<double(*)[32]>(&v[(size_t)g * 32]);
              const uint32_t d = sp_thread_step(q, R, u, o_lo + kOffsetsPerThread * g, n_mine, j == 0, c, l, vt,
                                                best, barg);
              for (int i = 0; i < n_mine; ++i) sw[(size_t)j * W + kOffsetsPerThread * g + i] = (d >> i) & 1u;
            }
            sp_merge(wmx, warg, best, barg);
          }
          sp_merge(cmx, carg, wmx, warg);
        }
        ++cnt[r].cta;
        slot_mx[r] = cmx;
        slot_arg[r] = carg;
        ++cnt[r].cluster;
      }
      // after the barrier every CTA merges the C slots in rank order; they all read the same slots
      double mx = slot_mx[0];
      int am = slot_arg[0];
      for (int r = 1; r < C; ++r) sp_merge(mx, am, slot_mx[r], slot_arg[r]);
      mxs[j] = mx;
      args[j] = am;
      c = sp_sub(mx, bp[1]);
    }
    for (int r = 0; r < C; ++r) ++cnt[r].cluster;  // the final barrier before any CTA exits
  }
  f = fopen(argv[2], "wb");
  fwrite(&nu, 4, 1, f);
  for (int j = 0; j < nu; ++j) {
    fwrite(&mxs[j], 8, 1, f);
    fwrite(&args[j], 4, 1, f);
  }
  if (nu > 1) fwrite(sw.data() + W, 1, (size_t)(nu - 1) * W, f);
  fwrite(&C, 4, 1, f);
  for (int r = 0; r < C; ++r) {
    fwrite(&cnt[r].cta, 4, 1, f);
    fwrite(&cnt[r].cluster, 4, 1, f);
  }
  fclose(f);
  return 0;
}
