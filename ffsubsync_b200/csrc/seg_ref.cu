// K1m: sampled segments as references of the batched sync calls (b2_sync_tracks_seg, --multi-segment-sync; DESIGN.md
// section 4).  The detector step first runs the call's detector over the segments only (b2i_vad_launch with a table
// of PCM ranges with gaps, and auditok's tokenizer), compactly into a scratch area; seg_ref_kernel then writes every
// frame of each segment video's reference - the owning segment's frame or 0.0 (seg_ref.cuh) - as floats, or as the
// run path's packed bits, and flags the video's first frame > 0.  sentinel_kernel (sig_ref.cu) gives the tracks of a
// video without such a frame the B2_BEST_K_NO_SPEECH sentinel.
#include <algorithm>

#include "common.cuh"
#include "seg_ref.cuh"
#include "sig_ref.cuh"   // kSigNoBadFrame: the flags' unset value

namespace {

struct SegRefParams {
  const float* scratch;             // the segments' detector output
  float* out;                       // the reference-signal buffer (uint32 words when packed)
  unsigned long long* speech;       // [call's V]: first frame > 0 (atomicMin), kSigNoBadFrame: none
  const long long* out_off;         // [n]: video i's frames (or words) start at out + out_off[i]
  const long long* len;             // [n]: its frame count L
  const long long* chunk_off;       // [n+1]: its chunks of kSegChunkFrames frames
  const int* run_first;             // [n+1]: its runs
  const long long* run_lo;
  const long long* run_src;
  const int* vid;                   // [n]: its index in the call (speech)
  int n;
  int packed;
};

// One CTA per chunk of 8192 frames of one video (grid-stride over the chunks of every listed video); warp w of the
// CTA owns 8 units of 32 frames, lane l frame 32u + l of them.  The frames of a lane increase, so its run is found
// once by bisection and then advanced.  Scratch is read only where a segment owns the frame.
__global__ void __launch_bounds__(kSegThreads) seg_ref_kernel(SegRefParams p) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long total = p.chunk_off[p.n];
  for (long long c = blockIdx.x; c < total; c += gridDim.x) {
    int lo = 0, hi = p.n - 1;   // the video of chunk c: the last i with chunk_off[i] <= c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(p.chunk_off + mid) <= c) lo = mid;
      else hi = mid - 1;
    }
    const long long L = __ldg(p.len + lo);
    const long long f0 = (c - __ldg(p.chunk_off + lo)) * kSegChunkFrames + (long long)warp * (kSegUnits * 32);
    if (f0 >= L) continue;
    const int r0 = __ldg(p.run_first + lo), r1 = __ldg(p.run_first + lo + 1);
    int r = r0, rh = r1 - 1;   // the run of this lane's first frame
    while (r < rh) {
      const int mid = (r + rh + 1) >> 1;
      if (__ldg(p.run_lo + mid) <= f0 + lane) r = mid;
      else rh = mid - 1;
    }
    long long speech_at = -1;
#pragma unroll
    for (int u = 0; u < kSegUnits; ++u) {
      const long long f = f0 + u * 32 + lane;
      const bool in = f < L;
      float v = 0.0f;
      if (in) {
        r = b2_seg_run(p.run_lo, r, r1, f);
        v = b2_seg_frame(p.scratch, p.run_lo, p.run_src, r, f);
      }
      const unsigned pos = __ballot_sync(0xffffffffu, in && v > 0.0f);
      if (pos && speech_at < 0) speech_at = f0 + u * 32 + (__ffs(pos) - 1);
      if (p.packed) {
        const unsigned word = __ballot_sync(0xffffffffu, in && v == 1.0f);
        if (lane == 0 && f0 + u * 32 < L)
          reinterpret_cast<uint32_t*>(p.out)[__ldg(p.out_off + lo) + ((f0 >> 5) + u)] = word;
      } else if (in) {
        p.out[__ldg(p.out_off + lo) + f] = v;
      }
    }
    if (speech_at >= 0 && lane == 0) atomicMin(p.speech + __ldg(p.vid + lo), (unsigned long long)speech_at);
  }
}

}  // namespace

int b2i_seg_ref_launch(b2_ctx* h, const float* d_scratch, const int64_t* out_off, const int* videos, int n_seg,
                       const int* run_first, const int64_t* run_lo, const int64_t* run_src, bool packed,
                       float* d_out, unsigned long long* d_speech) {
  if (n_seg <= 0) return B2_OK;
  B2Range range("b2:seg_ref");
  std::vector<long long> oo(n_seg), len(n_seg), chunk_off(n_seg + 1, 0);
  std::vector<int> vid(n_seg), rf(n_seg + 1);
  const int rb = run_first[0];
  for (int i = 0; i < n_seg; ++i) {
    const int v = videos[i];
    oo[i] = out_off[v];
    len[i] = out_off[v + 1] - out_off[v];
    vid[i] = v;
    rf[i] = run_first[i] - rb;
    chunk_off[i + 1] = chunk_off[i] + (len[i] + kSegChunkFrames - 1) / kSegChunkFrames;
  }
  rf[n_seg] = run_first[n_seg] - rb;
  // the flags of the listed videos (and of the videos between them, which nothing reads)
  B2_CUDA(h, cudaMemsetAsync(d_speech + videos[0], 0xff, (size_t)(videos[n_seg - 1] - videos[0] + 1) * 8,
                             h->stream));
  const long long total = chunk_off[n_seg];
  if (total == 0) return B2_OK;
  MetaArena a;
  const size_t tbl = (size_t)n_seg * 8, runs = (size_t)rf[n_seg] * 8;
  B2_TRY(b2i_meta_begin(h, &a, 3 * tbl + 8 + 2 * runs + (size_t)(2 * n_seg + 1) * 4 + 512));
  SegRefParams p;
  p.out_off = (const long long*)b2i_meta_put(&a, oo.data(), tbl);
  p.len = (const long long*)b2i_meta_put(&a, len.data(), tbl);
  p.chunk_off = (const long long*)b2i_meta_put(&a, chunk_off.data(), tbl + 8);
  p.run_first = (const int*)b2i_meta_put(&a, rf.data(), (size_t)(n_seg + 1) * 4);
  p.run_lo = (const long long*)b2i_meta_put(&a, run_lo + rb, runs);
  p.run_src = (const long long*)b2i_meta_put(&a, run_src + rb, runs);
  p.vid = (const int*)b2i_meta_put(&a, vid.data(), (size_t)n_seg * 4);
  B2_TRY(b2i_meta_commit(&a));
  p.scratch = d_scratch;
  p.out = d_out;
  p.speech = d_speech;
  p.n = n_seg;
  p.packed = packed ? 1 : 0;
  long long grid = std::min<long long>(total, (long long)h->sm_count * 4);
  // b2_sync_batch's pipeline: a later sub-batch's detector step keeps to the SM partition
  if (h->vad_partition_sms > 0) grid = std::min<long long>(grid, h->vad_partition_sms);
  seg_ref_kernel<<<(unsigned)grid, kSegThreads, 0, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "seg_ref_kernel");
  return B2_OK;
}
