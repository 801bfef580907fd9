// CPU emulation of run_corr_kernel's arithmetic (ffsubsync_b200/csrc/runcorr.cuh): the same
// __host__ __device__ functions run for every thread of the CTA, one after the other.  Test
// infrastructure (the build container has no GPU); tests/test_runcorr_cpu.py drives it.
//
// usage: runcorr_emul in.bin out.bin
// in.bin : int32 R, S, o_lo, W ; float32 level, label ; float32 ref[R] (1.0 or label) ; uint8 sub[S] (0/1)
// out.bin: float64 score[W] (offset o_lo + m) ; float64 eps ; int32 um[W] (UM of each offset)
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "../../ffsubsync_b200/csrc/runcorr.cuh"

using namespace runcorr;

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  int hdr[4];
  float lv[2];
  if (fread(hdr, 4, 4, f) != 4 || fread(lv, 4, 2, f) != 2) return 4;
  const int R = hdr[0], S = hdr[1], o_lo = hdr[2], W = hdr[3];
  std::vector<float> ref(R);
  std::vector<unsigned char> sub(S);
  if (fread(ref.data(), 4, R, f) != (size_t)R || fread(sub.data(), 1, S, f) != (size_t)S) return 4;
  fclose(f);
  if (W < 1 || W > kMaxWindow) return 5;

  // packed reference, laid out as ref_bits_kernel writes it, between kPoison poison entries on each side
  // (every bit set, a huge prefix): a read outside q[0] .. q[(R >> 5) + 2] changes a score or a UM count
  constexpr int kPoison = 64;
  const long long n_q = rc_ref_entries(R);
  std::vector<uint2> q_guarded(n_q + 2 * kPoison, make_uint2(0xffffffffu, 0x40000000u));
  uint2* q = q_guarded.data() + kPoison;
  q[0] = make_uint2(0u, 0u);
  int below = 0;
  for (int w = 0; w <= (R >> 5) + 1; ++w) {
    uint32_t bits = 0;
    for (int t = 0; t < 32; ++t) {
      const long long i = 32LL * w + t;
      if (i < R && ref[i] == 1.0f) bits |= 1u << t;
    }
    q[w + 1] = make_uint2(bits, (uint32_t)below);
    below += __builtin_popcount(bits);
  }
  // runs of the mask, and the total length of the runs before each
  std::vector<int> ra, rb, rl;
  for (int j = 0, len = 0; j < S;) {
    if (!sub[j]) {
      ++j;
      continue;
    }
    int e = j;
    while (e < S && sub[e]) ++e;
    ra.push_back(j);
    rb.push_back(e);
    rl.push_back(len);
    len += e - j;
    j = e;
  }
  const int nr = (int)ra.size();
  const RcLevels l = rc_levels(lv[0], lv[1]);
  const int n_thr = (W + kOffsetsPerThread - 1) / kOffsetsPerThread;
  std::vector<double> score(W);
  std::vector<int> um_out(W);
  for (int tid = 0; tid < n_thr; ++tid) {
    const int o0 = o_lo + kOffsetsPerThread * tid;
    const int n_mine = W - kOffsetsPerThread * tid < kOffsetsPerThread ? W - kOffsetsPerThread * tid : kOffsetsPerThread;
    int cnt[32], base;
    rc_thread_counts(q, R, ra.data(), rb.data(), nr, o0, cnt, base);
    int um = base;
    for (int i = 0; i < n_mine; ++i) {
      const int m = kOffsetsPerThread * tid + i;
      um_out[m] = um;
      score[m] = rc_score(q, R, S, ra.data(), rb.data(), rl.data(), nr, o0 + i, um, l);
      um += cnt[i] - nr;
    }
  }
  const double eps = rc_eps((double)(R < S ? R : S), l);
  f = fopen(argv[2], "wb");
  fwrite(score.data(), 8, W, f);
  fwrite(&eps, 8, 1, f);
  fwrite(um_out.data(), 4, W, f);
  fclose(f);
  return 0;
}
