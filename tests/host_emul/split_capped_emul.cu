// CPU emulation of split_capped_dp_kernel, one track on a thread-block cluster of N x C CTAs (the capped split,
// ffsubsync_b200/csrc/split.cu and split.cuh): the same __host__ __device__ functions run for every thread of every
// CTA, one after the other, between the kernel's barriers.  Test infrastructure; tests/test_split_capped_cpu.py
// drives it.
//
// usage: split_capped_emul in.bin out.bin N C cta_threads [dead]
// in.bin : int32 R, S, o_lo, W ; float32 level ; float64 beta, penalty ; uint8 m[R] (0/1) ; uint8 sub[S] (0/1)
// out.bin: int32 n_units ; per unit, per layer: float64 max, int32 argmax (what layer part 0 merges; the last unit's
//          maxima are the profile) ; per unit j >= 1, per layer: uint8 switch[W] ; int32 N x C ;
//          per CTA: int32 CTA barriers, int32 cluster barriers, as the kernel's control flow runs them
// CTA rank r runs layer r / C over window part r % C: part thread g = (r % C) * cta_threads + tid owns the offsets
// o_lo + 32 g .. (CTAs past the window own none).  Each CTA reduces its warps and publishes its maximum in its slot;
// after the cluster barrier each CTA merges its own layer's C slots and the layer below's C slots in rank order, the
// latter giving its next c (layer 0: c = -inf throughout).  dead: the track the kernel skips: n_units 0 and no barrier
// in any CTA.
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
  if (argc != 6 && argc != 7) return 2;
  const int N = atoi(argv[3]), C = atoi(argv[4]), nt = atoi(argv[5]);
  const bool dead = argc == 7 && atoi(argv[6]) != 0;
  const int NC = N * C;
  if (N < 1 || N > kMaxSegments || C < 1 || NC > kMaxCluster || nt < 32 || nt > kCtaThreads || nt % 32) return 5;
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
  std::vector<CtaCount> cnt(NC);
  std::vector<double> mxs;
  std::vector<int> args;
  std::vector<unsigned char> sw;
  int nu = 0;
  if (!dead) {  // the early exit is the track's: every CTA takes it, before any barrier
    const int nr = (int)ra.size();
    nu = nr > 0 ? nr : 1;
    for (int r = 0; r < NC; ++r) cnt[r].cta += decode_barriers(S, nt) + 1;
    const SpLevels l = sp_levels(level, bp[0]);
    std::vector<double> v((size_t)NC * nt * 32);  // per CTA, per thread
    std::vector<double> c(NC, -INFINITY);         // each CTA's c
    mxs.assign((size_t)nu * N, 0.0);
    args.assign((size_t)nu * N, 0);
    sw.assign((size_t)nu * N * W, 0);
    std::vector<double> slot_mx(NC);
    std::vector<int> slot_arg(NC);
    for (int j = 0; j < nu; ++j) {
      const SpUnit u = sp_unit(ra.data(), rb.data(), nr, S, j);
      for (int r = 0; r < NC; ++r) {  // each CTA up to its cluster barrier
        const int layer = r / C, part = r % C;
        double cmx = -INFINITY;
        int carg = -2147483647 - 1;
        for (int w = 0; w < nt / 32; ++w) {
          double wmx = -INFINITY;
          int warg = -2147483647 - 1;
          for (int lane = 0; lane < 32; ++lane) {
            const int g = part * nt + 32 * w + lane;
            const int n_mine = std::max(0, std::min(kOffsetsPerThread, W - kOffsetsPerThread * g));
            double best = -INFINITY;
            int barg = -2147483647 - 1;
            if (n_mine > 0) {
              double (&vt)[32] = *reinterpret_cast<double(*)[32]>(&v[((size_t)r * nt + 32 * w + lane) * 32]);
              const uint32_t d = sp_thread_step(q, R, u, o_lo + kOffsetsPerThread * g, n_mine, j == 0, c[r], l, vt,
                                                best, barg);
              for (int i = 0; i < n_mine; ++i)
                sw[((size_t)j * N + layer) * W + kOffsetsPerThread * g + i] = (d >> i) & 1u;
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
      // after the barrier: each CTA merges its own layer's slots (part 0 writes the argmax) and the layer below's
      for (int r = 0; r < NC; ++r) {
        const int layer = r / C, part = r % C, own = layer * C;
        if (part == 0) {
          double mx = slot_mx[own];
          int am = slot_arg[own];
          for (int p = 1; p < C; ++p) sp_merge(mx, am, slot_mx[own + p], slot_arg[own + p]);
          mxs[(size_t)j * N + layer] = mx;
          args[(size_t)j * N + layer] = am;
        }
        if (layer > 0) {
          double mx = slot_mx[own - C];
          int am = slot_arg[own - C];
          for (int p = 1; p < C; ++p) sp_merge(mx, am, slot_mx[own - C + p], slot_arg[own - C + p]);
          c[r] = sp_sub(mx, bp[1]);
        }
      }
    }
    for (int r = 0; r < NC; ++r) ++cnt[r].cluster;  // the final barrier before any CTA exits
  }
  f = fopen(argv[2], "wb");
  fwrite(&nu, 4, 1, f);
  for (size_t i = 0; i < (size_t)nu * N; ++i) {
    fwrite(&mxs[i], 8, 1, f);
    fwrite(&args[i], 4, 1, f);
  }
  if (nu > 1) fwrite(sw.data() + (size_t)N * W, 1, (size_t)(nu - 1) * N * W, f);
  fwrite(&NC, 4, 1, f);
  for (int r = 0; r < NC; ++r) {
    fwrite(&cnt[r].cta, 4, 1, f);
    fwrite(&cnt[r].cluster, 4, 1, f);
  }
  fclose(f);
  return 0;
}
