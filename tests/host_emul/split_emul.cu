// CPU emulation of split_dp_kernel's arithmetic (ffsubsync_b200/csrc/split.cuh): the same __host__ __device__
// functions run for every thread of the CTA, one after the other, with the CTA's max / argmax per unit.  Test
// infrastructure; tests/test_split_cpu.py drives it.
//
// usage: split_emul in.bin out.bin
// in.bin : int32 R, S, o_lo, W ; float32 level ; float64 beta, penalty ; uint8 m[R] (0/1) ; uint8 sub[S] (0/1)
// out.bin: int32 n_units ; per unit: float64 max, int32 argmax ; per unit j >= 1: uint8 switch[W]
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "../../ffsubsync_b200/csrc/split.cuh"

using namespace split;

int main(int argc, char** argv) {
  if (argc != 3) return 2;
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
  if (W < 1 || W > kMaxWindow) return 5;
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
  const int nr = (int)ra.size(), nu = nr > 0 ? nr : 1;
  const SpLevels l = sp_levels(level, bp[0]);
  const int n_thr = (W + kOffsetsPerThread - 1) / kOffsetsPerThread;
  std::vector<double> v((size_t)n_thr * 32);
  std::vector<double> mxs(nu);
  std::vector<int> args(nu);
  std::vector<unsigned char> sw((size_t)nu * W, 0);
  double c = 0.0;
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra.data(), rb.data(), nr, S, j);
    double mx = -INFINITY;
    int am = 0;
    for (int tid = 0; tid < n_thr; ++tid) {
      const int o0 = o_lo + kOffsetsPerThread * tid;
      const int n_mine = W - kOffsetsPerThread * tid < kOffsetsPerThread ? W - kOffsetsPerThread * tid : kOffsetsPerThread;
      double (&vt)[32] = *reinterpret_cast<double(*)[32]>(&v[(size_t)tid * 32]);
      double best;
      int barg;
      const uint32_t d = sp_thread_step(q, R, u, o0, n_mine, j == 0, c, l, vt, best, barg);
      for (int i = 0; i < n_mine; ++i) sw[(size_t)j * W + kOffsetsPerThread * tid + i] = (d >> i) & 1u;
      if (best > mx || (best == mx && barg > am)) {
        mx = best;
        am = barg;
      }
    }
    mxs[j] = mx;
    args[j] = am;
    c = sp_sub(mx, bp[1]);
  }
  f = fopen(argv[2], "wb");
  fwrite(&nu, 4, 1, f);
  for (int j = 0; j < nu; ++j) {
    fwrite(&mxs[j], 8, 1, f);
    fwrite(&args[j], 4, 1, f);
  }
  fwrite(sw.data() + W, 1, (size_t)(nu - 1) * W, f);
  fclose(f);
  return 0;
}
