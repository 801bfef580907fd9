// The sampled-segment reference rule (MultiSegmentVideoSpeechTransformer.fit, ffsubsync/speech_transformers.py:
// 855-895) as seg_ref_kernel applies it, shared with its CPU emulator (tests/host_emul/seg_ref_emul.cu).
//
// The reference of a segment video has L = int(total * sample_rate) + 2 frames, 0.0 outside its segments.  The planner
// turns the segments into owned-frame runs (sync_plan.h plan_segments): run r covers frames run_lo[r] .. run_lo[r+1]-1
// and reads the segments' detector output from scratch index run_src[r] on, or is 0.0 (run_src[r] < 0).  The video
// has speech when a frame is > 0, as the reference's np.any(sparse > 0).
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define SG_HD __host__ __device__ __forceinline__
#else
#define SG_HD inline
#endif

constexpr int kSegUnits = 8;       // 32-frame units per warp per chunk
constexpr int kSegThreads = 256;
constexpr long long kSegChunkFrames = (long long)(kSegThreads / 32) * kSegUnits * 32;   // 8192 frames

// The run of frame f, starting the search at run r (f >= run_lo[r]): the last run whose first frame is <= f
SG_HD int b2_seg_run(const long long* run_lo, int r, int r_end, long long f) {
  while (r + 1 < r_end && run_lo[r + 1] <= f) ++r;
  return r;
}

// frame f of the run r: the owning segment's value, or 0.0
SG_HD float b2_seg_frame(const float* scratch, const long long* run_lo, const long long* run_src, int r, long long f) {
  return run_src[r] < 0 ? 0.0f : scratch[run_src[r] + (f - run_lo[r])];
}
