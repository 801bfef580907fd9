// K1s: serialized speech signals as references of the batched sync calls (b2_sync_tracks_sig, DESIGN.md section 4).
// sig_ref_kernel turns each signal video's stored float64 values into its reference frames (sig_ref.cuh) in the
// reference-signal buffer - floats, or the run path's packed bits - and flags a video with out-of-domain values;
// sentinel_kernel then overwrites every output of a flagged video's tracks with the B2_BEST_K_BAD_SIGNAL sentinel
// (and of a segment video without speech with B2_BEST_K_NO_SPEECH: seg_ref.cu sets those flags).
#include <algorithm>

#include "common.cuh"
#include "sig_ref.cuh"

namespace {

struct SigRefParams {
  const double* x;                  // stored values, absolute indices
  float* out;                       // the reference-signal buffer (uint32 words when packed)
  unsigned long long* first_bad;    // [call's V]: first out-of-domain frame (atomicMin), kSigNoBadFrame: none
  const long long* x_off;           // [n]: video i's values start at x + x_off[i]
  const long long* out_off;         // [n]: its frames (or words) start at out + out_off[i]
  const long long* len;             // [n]: its frame count R
  const long long* chunk_off;       // [n+1]: its chunks of kSigChunkFrames frames
  const int* vid;                   // [n]: its index in the call (first_bad)
  int n;
  float label;
  int packed;
};

// One CTA per chunk of 16384 frames of one video (grid-stride over the chunks of every listed video); warp w of the
// CTA owns 16 units of 32 frames.  Each lane issues its 16 loads before it stores anything, so a CTA keeps 128 KB of
// reads in flight and one CTA per SM streams on its own: the grid can be capped at the SM partition of the pipeline
// like the VAD's.  The values are read once (streaming loads).
__global__ void __launch_bounds__(kSigThreads, 1) sig_ref_kernel(SigRefParams p) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long total = p.chunk_off[p.n];
  for (long long c = blockIdx.x; c < total; c += gridDim.x) {
    int lo = 0, hi = p.n - 1;   // the video of chunk c: the last i with chunk_off[i] <= c
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(p.chunk_off + mid) <= c) lo = mid;
      else hi = mid - 1;
    }
    const long long R = __ldg(p.len + lo);
    const long long f0 = (c - __ldg(p.chunk_off + lo)) * kSigChunkFrames + (long long)warp * (kSigUnits * 32);
    if (f0 >= R) continue;
    const double* xv = p.x + __ldg(p.x_off + lo);
    double v[kSigUnits];
#pragma unroll
    for (int u = 0; u < kSigUnits; ++u) {
      const long long f = f0 + u * 32 + lane;
      v[u] = f < R ? __ldcs(xv + f) : 0.0;
    }
    long long bad_at = -1;
#pragma unroll
    for (int u = 0; u < kSigUnits; ++u) {
      const long long f = f0 + u * 32 + lane;
      const bool in = f < R;
      const float r = b2_sig_frame(v[u], p.label);
      const unsigned bad = __ballot_sync(0xffffffffu, in && b2_sig_out_of_domain(v[u]));
      if (bad && bad_at < 0) bad_at = f0 + u * 32 + (__ffs(bad) - 1);
      if (p.packed) {
        const unsigned word = __ballot_sync(0xffffffffu, in && r == 1.0f);
        if (lane == 0 && f0 + u * 32 < R)
          reinterpret_cast<uint32_t*>(p.out)[__ldg(p.out_off + lo) + ((f0 >> 5) + u)] = word;
      } else if (in) {
        p.out[__ldg(p.out_off + lo) + f] = r;
      }
    }
    if (bad_at >= 0 && lane == 0) atomicMin(p.first_bad + __ldg(p.vid + lo), (unsigned long long)bad_at);
  }
}

struct SentinelParams {
  const unsigned long long* flag;        // [call's V]: kSigNoBadFrame = unset
  const int* vid;                        // [n]: the flagged kind's videos
  const int* trk;                        // [2n]: their tracks trk[2i] .. trk[2i+1]-1
  double* bs;
  int32_t* bo;
  int32_t* bk;
  double* a_score;                       // may be null: [T * cols]
  int32_t* a_offset;                     // may be null
  int cols;
  double* ratio;                         // may be null: [T]
  double* evals;                         // may be null: [T * kGssEvals]
  int n_evals;
  int sentinel;
  int bad_if_set;                        // 1: a set flag marks the video, 0: an unset one
};

// One CTA per listed video; a video that is not marked leaves everything as it is.
__global__ void __launch_bounds__(128) sentinel_kernel(SentinelParams p) {
  const int i = blockIdx.x;
  if ((p.flag[p.vid[i]] != kSigNoBadFrame) != (p.bad_if_set != 0)) return;
  const long long t0 = p.trk[2 * i], t1 = p.trk[2 * i + 1];
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  for (long long t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
    p.bs[t] = nan;
    p.bo[t] = 0;
    p.bk[t] = p.sentinel;
    if (p.ratio) p.ratio[t] = nan;
  }
  for (long long j = t0 * p.cols + threadIdx.x; j < t1 * p.cols; j += blockDim.x) {
    if (p.a_score) p.a_score[j] = nan;
    if (p.a_offset) p.a_offset[j] = 0;
  }
  if (p.evals)
    for (long long j = t0 * p.n_evals + threadIdx.x; j < t1 * p.n_evals; j += blockDim.x) p.evals[j] = nan;
}

}  // namespace

int b2i_sig_ref_launch(b2_ctx* h, const double* d_x, const int64_t* x_off, const int64_t* out_off, int n_videos,
                       const int* videos, int n_sig, float label, bool packed, float* d_out,
                       unsigned long long* d_first_bad) {
  if (n_sig <= 0) return B2_OK;
  B2Range range("b2:sig_ref");
  std::vector<long long> xo(n_sig), oo(n_sig), len(n_sig), chunk_off(n_sig + 1, 0);
  std::vector<int> vid(n_sig);
  for (int i = 0; i < n_sig; ++i) {
    const int v = videos[i];
    xo[i] = x_off[v];
    oo[i] = out_off[v];
    len[i] = out_off[v + 1] - out_off[v];
    vid[i] = v;
    chunk_off[i + 1] = chunk_off[i] + (len[i] + kSigChunkFrames - 1) / kSigChunkFrames;
  }
  // the flags of the listed videos (and of the videos between them, which nothing reads)
  B2_CUDA(h, cudaMemsetAsync(d_first_bad + videos[0], 0xff, (size_t)(videos[n_sig - 1] - videos[0] + 1) * 8,
                             h->stream));
  const long long total = chunk_off[n_sig];
  if (total == 0) return B2_OK;
  MetaArena a;
  const size_t tbl = (size_t)n_sig * 8;
  B2_TRY(b2i_meta_begin(h, &a, 4 * tbl + 8 + (size_t)n_sig * 4 + 512));
  SigRefParams p;
  p.x_off = (const long long*)b2i_meta_put(&a, xo.data(), tbl);
  p.out_off = (const long long*)b2i_meta_put(&a, oo.data(), tbl);
  p.len = (const long long*)b2i_meta_put(&a, len.data(), tbl);
  p.chunk_off = (const long long*)b2i_meta_put(&a, chunk_off.data(), tbl + 8);
  p.vid = (const int*)b2i_meta_put(&a, vid.data(), (size_t)n_sig * 4);
  B2_TRY(b2i_meta_commit(&a));
  p.x = d_x;
  p.out = d_out;
  p.first_bad = d_first_bad;
  p.n = n_sig;
  p.label = label;
  p.packed = packed ? 1 : 0;
  long long grid = std::min<long long>(total, (long long)h->sm_count);
  // b2_sync_batch's pipeline: a later sub-batch's detector step keeps to the SM partition
  if (h->vad_partition_sms > 0) grid = std::min<long long>(grid, h->vad_partition_sms);
  sig_ref_kernel<<<(unsigned)grid, kSigThreads, 0, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "sig_ref_kernel");
  return B2_OK;
}

int b2i_sentinel_launch(b2_ctx* h, const unsigned long long* d_flag, const int* videos, int n_sig, const int* trk_off,
                        const B2SigBadOut& out, int sentinel, bool bad_if_set) {
  if (n_sig <= 0) return B2_OK;
  B2Range range("b2:sentinel");
  std::vector<int> trk(2 * (size_t)n_sig);
  for (int i = 0; i < n_sig; ++i) {
    trk[2 * i] = trk_off[videos[i]];
    trk[2 * i + 1] = trk_off[videos[i] + 1];
  }
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, (size_t)n_sig * 12 + 512));
  SentinelParams p;
  p.vid = (const int*)b2i_meta_put(&a, videos, (size_t)n_sig * 4);
  p.trk = (const int*)b2i_meta_put(&a, trk.data(), (size_t)n_sig * 8);
  B2_TRY(b2i_meta_commit(&a));
  p.flag = d_flag;
  p.bs = out.bs;
  p.bo = out.bo;
  p.bk = out.bk;
  p.a_score = out.a_score;
  p.a_offset = out.a_offset;
  p.cols = out.cols;
  p.ratio = out.ratio;
  p.evals = out.evals;
  p.n_evals = out.n_evals;
  p.sentinel = sentinel;
  p.bad_if_set = bad_if_set ? 1 : 0;
  sentinel_kernel<<<(unsigned)n_sig, 128, 0, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "sentinel_kernel");
  return B2_OK;
}
