// K1o: the speech output of the batched sync calls (b2_speech_output, `--serialize-speech`; DESIGN.md section 4).
// speech_out_kernel reads the call's reference-signal buffer once more, behind every chain, and writes the listed
// videos' frames as float64, back to back (speech_out.cuh).  Bandwidth-bound: 8 bytes written per frame, 4 (floats) or
// 1/8 (packed bits) read.
#include <algorithm>

#include "common.cuh"
#include "speech_out.cuh"

namespace {

// One CTA per tile of kSpeechTile output frames (grid-stride over the tiles); thread t writes frames t, t + 256, ...
// of the tile, so every warp store covers 256 contiguous bytes whatever the video boundaries.  A thread's video is
// found once per tile by bisection and then advanced.
__global__ void __launch_bounds__(kSpeechThreads) speech_out_kernel(const float* __restrict__ ref,
                                                                   const long long* __restrict__ off,
                                                                   const B2SpeechVideo* __restrict__ vids, int n,
                                                                   long long total, double* __restrict__ out) {
  const long long tiles = (total + kSpeechTile - 1) / kSpeechTile;
  for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
    long long f = t * kSpeechTile + threadIdx.x;
    if (f >= total) continue;
    int i = b2_speech_video(off, n, f);
#pragma unroll 4
    for (int k = 0; k < (int)(kSpeechTile / kSpeechThreads); ++k, f += kSpeechThreads) {
      if (f >= total) break;
      while (__ldg(off + i + 1) <= f) ++i;
      out[f] = b2_speech_frame(ref, vids[i], f - __ldg(off + i));
    }
  }
}

}  // namespace

int b2i_speech_out_launch(b2_ctx* h, const float* d_ref, const int64_t* off, const B2SpeechVideo* vids, int n,
                          double* d_out) {
  const long long total = n > 0 ? (long long)off[n] : 0;
  if (total == 0) return B2_OK;
  B2Range range("b2:speech_out");
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, (size_t)(n + 1) * 8 + (size_t)n * sizeof(B2SpeechVideo) + 256));
  const long long* d_off = (const long long*)b2i_meta_put(&a, off, (size_t)(n + 1) * 8);
  const B2SpeechVideo* d_vids = (const B2SpeechVideo*)b2i_meta_put(&a, vids, (size_t)n * sizeof(B2SpeechVideo));
  B2_TRY(b2i_meta_commit(&a));
  const long long tiles = (total + kSpeechTile - 1) / kSpeechTile;
  const unsigned grid = (unsigned)std::min<long long>(tiles, (long long)h->sm_count * 8);
  speech_out_kernel<<<grid, kSpeechThreads, 0, h->stream>>>(d_ref, d_off, d_vids, n, total, d_out);
  B2_CHECK_LAUNCH(h, "speech_out_kernel");
  return B2_OK;
}
