// The speech output of the batched sync calls (b2_speech_output, `--serialize-speech`): speech_out_kernel's frame rule,
// shared with its CPU emulator (tests/host_emul/speech_out_emul.cu).
//
// Listed video i's frames speech[off[i] .. off[i+1]) are its reference signal widened to float64, read from the call's
// reference buffer at src (absolute): float32 frames, or in a packed sub-batch ceil(R/32) uint32 words of the bits
// m = (r == 1.0f), frame f at bit f & 31 of word f >> 5; a clear bit is the video's low level (its label for detector and
// signal videos, 0.0 for text, PGS and segment videos).
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define SO_HD __host__ __device__ __forceinline__
#else
#define SO_HD inline
#endif

constexpr int kSpeechThreads = 256;
constexpr long long kSpeechTile = 4096;   // output frames per CTA and tile: 16 per thread

struct B2SpeechVideo {
  long long src;   // the video's first frame (or word) in the reference buffer
  float low;       // a clear bit's value (packed only)
  int packed;
};

// The listed video of output frame f < off[n]: the last i with off[i] <= f (never an empty one)
SO_HD int b2_speech_video(const long long* off, int n, long long f) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (off[mid] <= f) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// frame r of a listed video
SO_HD double b2_speech_frame(const float* ref, const B2SpeechVideo& v, long long r) {
  if (!v.packed) return (double)ref[v.src + r];
  const uint32_t w = reinterpret_cast<const uint32_t*>(ref)[v.src + (r >> 5)];
  return (w >> (r & 31)) & 1u ? 1.0 : (double)v.low;
}
