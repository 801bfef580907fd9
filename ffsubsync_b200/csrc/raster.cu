// K2: subtitle cue list -> 100 Hz speech signal for K framerate ratios, K7: first/last speech
// frame, K6: max-score reduction over the ratio candidates of each pair.
//
// K2 replaces SubtitleScaler.fit (ffsubsync/subtitle_transformers.py:35-47) followed by
// SubtitleSpeechTransformer.fit (ffsubsync/speech_transformers.py:957-980).  The reference does
// this arithmetic in float64 through datetime.timedelta; it is reproduced bit for bit with
// explicitly rounded double operations (no FMA contraction):
//   scaled  = timedelta(seconds=t*ratio).total_seconds()
//           = (trunc(x)*1e6 + rint(frac(x)*1e6)) / 1e6,  x = t*ratio      (microsecond rounding)
//   first   = rint((scaled_start - start_seconds) * sample_rate)          (Python round: half-even)
//   last    = first + rint((scaled_end - scaled_start) * sample_rate)
//   samples[first:last] = min(1/ratio, 1)   with Python slice semantics (negative index wraps once)
// Every cue writes the same level, so the order of overlapping cues does not matter.
#include <algorithm>

#include "common.cuh"
#include "raster_math.cuh"

namespace {

struct RasterParams {
  const double* start_s;
  const double* end_s;
  const uint8_t* keep;        // may be null (= keep all)
  const long long* cue_off;   // [B+1]
  const double* ratios;       // [K] or [B*K]
  const double* levels;       // same shape as ratios, or null (= min(1/ratio, 1))
  const long long* out_off;   // [B*K+1]
  float* out;
  int B, K, per_pair, sample_rate, sig_base;
  double start_seconds;
};

// one warp per cue, grid.y = signal (b*K + k)
__global__ void __launch_bounds__(256) raster_cues_kernel(RasterParams p) {
  const int sig = blockIdx.y + p.sig_base;
  const int b = sig / p.K;
  const double ratio = p.per_pair ? p.ratios[sig] : p.ratios[sig - b * p.K];
  const long long c0 = p.cue_off[b], c1 = p.cue_off[b + 1];
  const long long n = p.out_off[sig + 1] - p.out_off[sig];
  float* out = p.out + p.out_off[sig];
  const float level = p.levels ? (float)(p.per_pair ? p.levels[sig] : p.levels[sig - b * p.K])
                               : (float)fmin(__ddiv_rn(1.0, ratio), 1.0);
  const int lane = threadIdx.x & 31;
  const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const long long nwarps = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long c = c0 + warp; c < c1; c += nwarps) {
    if (p.keep && !p.keep[c]) continue;
    long long first, last;
    b2_cue_bounds(p.start_s[c], p.end_s[c], ratio, p.start_seconds, p.sample_rate, n, first, last);
    for (long long i = first + lane; i < last; i += 32) out[i] = level;
  }
}

// K2b: the same cue arithmetic, output as a bit mask (bit i of word i/32 = frame i is inside a kept
// cue).  b2_sync_batch never materialises the float signals: the correlation kernel and the exact
// re-score read these masks (1/32 of the bytes).  One thread per (cue, ratio); a cue spans ~10
// words, cues of one signal rarely share a word, so the atomics are uncontended.
struct RasterBitsParams {
  const double* start_s;
  const double* end_s;
  const uint8_t* keep;         // may be null
  const long long* cue_off;    // [B+1]
  const double* ratios;        // [K]
  const long long* sig_off;    // [B*K+1]: only the differences (signal lengths) are used
  const long long* bits_off;   // [B*K+1] words
  uint32_t* bits;              // zeroed by the caller
  int K, sample_rate, sig_base;  // blockIdx.y + sig_base = signal (grid.y is limited to 65535)
  double start_seconds;
  // device-driven ratios (the GSS rounds, K = 1): when set, signal b has ratio sig_ratio[b], length
  // sig_len[b] and its mask at bits + b * sig_words; ratios / sig_off / bits_off are not read
  const double* sig_ratio;
  const long long* sig_len;
  long long sig_words;
};

__global__ void __launch_bounds__(256) raster_bits_kernel(RasterBitsParams p) {
  const int sig = blockIdx.y + p.sig_base;
  const int b = sig / p.K;
  const bool dev = p.sig_ratio != nullptr;
  const double ratio = dev ? p.sig_ratio[sig] : p.ratios[sig - b * p.K];
  const long long c0 = p.cue_off[b], c1 = p.cue_off[b + 1];
  const long long n = dev ? p.sig_len[sig] : p.sig_off[sig + 1] - p.sig_off[sig];
  uint32_t* out = p.bits + (dev ? sig * p.sig_words : p.bits_off[sig]);
  for (long long c = c0 + (long long)blockIdx.x * blockDim.x + threadIdx.x; c < c1;
       c += (long long)gridDim.x * blockDim.x) {
    if (p.keep && !p.keep[c]) continue;
    long long first, last;
    b2_cue_bounds(p.start_s[c], p.end_s[c], ratio, p.start_seconds, p.sample_rate, n, first, last);
    if (last <= first) continue;
    const long long w0 = first >> 5, w1 = (last - 1) >> 5;
    const uint32_t m0 = 0xffffffffu << (first & 31);
    const uint32_t m1 = 0xffffffffu >> (31 - ((last - 1) & 31));
    if (w0 == w1) {
      atomicOr(out + w0, m0 & m1);
    } else {
      atomicOr(out + w0, m0);
      for (long long w = w0 + 1; w < w1; ++w) atomicOr(out + w, 0xffffffffu);
      atomicOr(out + w1, m1);
    }
  }
}

// K2r: embedded-subtitle references (b2_sync_tracks_subs): the reference signal of a video with a subtitle
// stream is its cue list rasterised at ratio 1.0 and level 1.0 (SubtitleScaler(1.0) +
// SubtitleSpeechTransformer, speech_transformers.py:479-523), written into the reference-signal buffer at
// the video's own base between the detector's outputs.  One CTA per such video: zero the signal, then one
// warp per cue with the same cue arithmetic as raster_cues_kernel.
// K2p: PGS references (b2_sync_tracks_pgs, b2_rasterize_pgs) have the same structure with PGSSpeechTransformer's
// interval arithmetic (b2_pgs_bounds: every write lies in [0, n) of the video's own range) and no keep flags.
enum RefRule { kRefCues = 0, kRefPgs = 1 };

struct RasterRefParams {
  const double* start_s;
  const double* end_s;
  const uint8_t* keep;        // may be null (kRefPgs: not read)
  const long long* cue_off;   // [n_videos+1] absolute
  const long long* out_off;   // [n_videos+1] the reference-signal buffer's offsets
  const int* video;           // [grid.x] the videos (indices into cue_off / out_off) with a subtitle reference
  float* out;
  int sample_rate;
  double start_seconds;
};

template <int kRule>
__global__ void __launch_bounds__(256) raster_ref_kernel(RasterRefParams p) {
  const int v = p.video[blockIdx.x];
  const long long c0 = p.cue_off[v], c1 = p.cue_off[v + 1];
  const long long n = p.out_off[v + 1] - p.out_off[v];
  float* out = p.out + p.out_off[v];
  for (long long i = threadIdx.x; i < n; i += blockDim.x) out[i] = 0.0f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  for (long long c = c0 + (threadIdx.x >> 5); c < c1; c += blockDim.x >> 5) {
    long long first, last;
    if (kRule == kRefPgs) {
      b2_pgs_bounds(p.start_s[c], p.end_s[c], p.start_seconds, p.sample_rate, n, first, last);
    } else {
      if (p.keep && !p.keep[c]) continue;
      b2_cue_bounds(p.start_s[c], p.end_s[c], 1.0, p.start_seconds, p.sample_rate, n, first, last);
    }
    for (long long i = first + lane; i < last; i += 32) out[i] = 1.0f;
  }
}

// ---- K7 -------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bounds_kernel(const float* __restrict__ sig,
                                                      const long long* __restrict__ off, int n_sig,
                                                      long long* __restrict__ first,
                                                      long long* __restrict__ last) {
  const int s = blockIdx.x;
  const float* x = sig + off[s];
  const long long n = off[s + 1] - off[s];
  long long lo = n, hi = -1;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    if (x[i] > 0.5f) {  // speech_transformers.py:313
      if (i < lo) lo = i;
      if (i > hi) hi = i;
    }
  }
  __shared__ long long slo[256], shi[256];
  slo[threadIdx.x] = lo;
  shi[threadIdx.x] = hi;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      slo[threadIdx.x] = min(slo[threadIdx.x], slo[threadIdx.x + w]);
      shi[threadIdx.x] = max(shi[threadIdx.x], shi[threadIdx.x + w]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    first[s] = shi[0] < 0 ? -1 : slo[0];
    last[s] = shi[0];
  }
}

// ---- K6 -------------------------------------------------------------------------------------
// MaxScoreAligner.transform (ffsubsync/aligners.py:154-167): keep |offset| <= max_offset_samples,
// highest score wins, first in list order wins ties.
__global__ void __launch_bounds__(128) reduce_ratios_kernel(const double* __restrict__ score,
                                                             const int32_t* __restrict__ offset,
                                                             const int32_t* __restrict__ status,
                                                             int B, int K, long long max_off,
                                                             double* __restrict__ best_score,
                                                             int32_t* __restrict__ best_offset,
                                                             int32_t* __restrict__ best_k) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int bk = -1;
  double bs = 0.0;
  int bo = 0;
  for (int k = 0; k < K; ++k) {
    const size_t j = (size_t)b * K + k;
    if (status && (status[j] & B2_ALIGN_EMPTY)) continue;  // FFTAligner.fit raised for this one
    const int o = offset[j];
    if (max_off != B2_MAX_OFFSET_NONE && llabs((long long)o) > max_off) continue;
    const double s = score[j];
    if (bk < 0 || s > bs) {
      bk = k;
      bs = s;
      bo = o;
    }
  }
  best_k[b] = bk;
  best_score[b] = bs;
  best_offset[b] = bo;
}

// ---- fused-VAD blend (speech_transformers.py:281-294) ----------------------------------------
__global__ void __launch_bounds__(256) blend_kernel(const float* __restrict__ a,
                                                     const float* __restrict__ b, long long n,
                                                     int mode, double wa, double wb,
                                                     float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const float x = a[i], y = b[i];
    float r;
    if (mode == 0) r = fminf(x, y);
    else if (mode == 1) r = fmaxf(x, y);
    else r = (float)__dadd_rn(__dmul_rn(wa, (double)x), __dmul_rn(wb, (double)y));
    out[i] = r;
  }
}

}  // namespace

int b2i_blend_launch(b2_ctx* h, const float* d_a, const float* d_b, int64_t n, int mode, double wa,
                     double wb, float* d_out) {
  int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)h->sm_count * 8);
  blend_kernel<<<blocks, 256, 0, h->stream>>>(d_a, d_b, n, mode, wa, wb, d_out);
  B2_CHECK_LAUNCH(h, "blend_kernel");
  return B2_OK;
}

int b2i_raster_launch(b2_ctx* h, const double* cue_start, const double* cue_end,
                      const uint8_t* cue_keep, const int64_t* cue_off, int B, const double* ratios,
                      int K, int per_pair_ratios, const double* levels, int sample_rate,
                      double start_seconds, float* d_out, const int64_t* out_off) {
  B2Range range("b2:rasterize");
  // cue_off / out_off may be slices of larger tables (sub-batches): entries are absolute indices
  // into cue_start/... and d_out, only [cue_off[0], cue_off[B]) is uploaded (pointers rebased)
  const size_t J = (size_t)B * K;
  const size_t c0 = (size_t)cue_off[0];
  const size_t ncue = (size_t)cue_off[B] - c0;
  const size_t nr = per_pair_ratios ? J : (size_t)K;
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, ncue * 17 + (B + 1) * 8 + (J + 1) * 8 + nr * 16 + 1024));
  RasterParams p;
  p.start_s = (const double*)b2i_meta_put(&a, cue_start + c0, ncue * 8) - c0;
  p.end_s = (const double*)b2i_meta_put(&a, cue_end + c0, ncue * 8) - c0;
  p.keep = cue_keep ? (const uint8_t*)b2i_meta_put(&a, cue_keep + c0, ncue) - c0 : nullptr;
  p.cue_off = (const long long*)b2i_meta_put(&a, cue_off, (size_t)(B + 1) * 8);
  p.ratios = (const double*)b2i_meta_put(&a, ratios, nr * 8);
  p.levels = levels ? (const double*)b2i_meta_put(&a, levels, nr * 8) : nullptr;
  p.out_off = (const long long*)b2i_meta_put(&a, out_off, (J + 1) * 8);
  B2_TRY(b2i_meta_commit(&a));
  p.out = d_out;
  p.B = B;
  p.K = K;
  p.per_pair = per_pair_ratios;
  p.sample_rate = sample_rate;
  p.start_seconds = start_seconds;
  const size_t total = (size_t)(out_off[J] - out_off[0]);
  if (total) B2_CUDA(h, cudaMemsetAsync(d_out + out_off[0], 0, total * 4, h->stream));
  int64_t max_cues = 0;
  for (int b = 0; b < B; ++b) max_cues = std::max<int64_t>(max_cues, cue_off[b + 1] - cue_off[b]);
  if (max_cues == 0 || J == 0) return B2_OK;
  for (size_t j0 = 0; j0 < J; j0 += 65535) {
    p.sig_base = (int)j0;
    dim3 grid((unsigned)std::min<int64_t>((max_cues + 7) / 8, 64), (unsigned)std::min<size_t>(J - j0, 65535));
    raster_cues_kernel<<<grid, 256, 0, h->stream>>>(p);
    B2_CHECK_LAUNCH(h, "raster_cues_kernel");
  }
  return B2_OK;
}

int b2i_raster_ref_launch(b2_ctx* h, const double* cue_start, const double* cue_end, const uint8_t* cue_keep,
                          const int64_t* cue_off, const int64_t* out_off, int n_videos, const int* videos, int n_subs,
                          int sample_rate, double start_seconds, float* d_out, bool pgs) {
  if (n_subs <= 0) return B2_OK;
  B2Range range(pgs ? "b2:raster_pgs" : "b2:raster_ref");
  // cue_off / out_off are slices of the call's tables (a sub-batch): entries are absolute, only
  // [cue_off[0], cue_off[n_videos]) is uploaded (pointers rebased)
  const size_t c0 = (size_t)cue_off[0], nc = (size_t)cue_off[n_videos] - c0;
  const size_t tbl = (size_t)(n_videos + 1) * 8;
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, nc * 17 + 2 * tbl + (size_t)n_subs * 4 + 1024));
  RasterRefParams p;
  p.start_s = (const double*)b2i_meta_put(&a, cue_start + c0, nc * 8) - c0;
  p.end_s = (const double*)b2i_meta_put(&a, cue_end + c0, nc * 8) - c0;
  p.keep = cue_keep ? (const uint8_t*)b2i_meta_put(&a, cue_keep + c0, nc) - c0 : nullptr;
  p.cue_off = (const long long*)b2i_meta_put(&a, cue_off, tbl);
  p.out_off = (const long long*)b2i_meta_put(&a, out_off, tbl);
  p.video = (const int*)b2i_meta_put(&a, videos, (size_t)n_subs * 4);
  B2_TRY(b2i_meta_commit(&a));
  p.out = d_out;
  p.sample_rate = sample_rate;
  p.start_seconds = start_seconds;
  if (pgs) {
    raster_ref_kernel<kRefPgs><<<n_subs, 256, 0, h->stream>>>(p);
    B2_CHECK_LAUNCH(h, "raster_ref_kernel<pgs>");
  } else {
    raster_ref_kernel<kRefCues><<<n_subs, 256, 0, h->stream>>>(p);
    B2_CHECK_LAUNCH(h, "raster_ref_kernel");
  }
  return B2_OK;
}

int b2i_raster_bits_launch(b2_ctx* h, const B2CueSource* src, int B, int K, const int64_t* sig_off,
                           const long long* bits_off, uint32_t* d_bits) {
  B2Range range("b2:raster_bits");
  // cue_off / sig_off may be slices of larger tables (sub-batches), see b2i_raster_launch
  const size_t J = (size_t)B * K;
  const size_t c0 = (size_t)src->cue_off[0], nc = (size_t)src->cue_off[B] - c0;
  if (bits_off[J]) B2_CUDA(h, cudaMemsetAsync(d_bits, 0, (size_t)bits_off[J] * 4, h->stream));
  int64_t max_cues = 0;
  for (int b = 0; b < B; ++b) max_cues = std::max<int64_t>(max_cues, src->cue_off[b + 1] - src->cue_off[b]);
  if (max_cues == 0 || J == 0) return B2_OK;
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, nc * 17 + (B + 1) * 8 + (J + 1) * 16 + (size_t)K * 8 + 1024));
  RasterBitsParams p;
  p.start_s = (const double*)b2i_meta_put(&a, src->cue_start + c0, nc * 8) - c0;
  p.end_s = (const double*)b2i_meta_put(&a, src->cue_end + c0, nc * 8) - c0;
  p.keep = src->cue_keep ? (const uint8_t*)b2i_meta_put(&a, src->cue_keep + c0, nc) - c0 : nullptr;
  p.cue_off = (const long long*)b2i_meta_put(&a, src->cue_off, (size_t)(B + 1) * 8);
  p.ratios = (const double*)b2i_meta_put(&a, src->ratios, (size_t)K * 8);
  p.sig_off = (const long long*)b2i_meta_put(&a, sig_off, (J + 1) * 8);
  p.bits_off = (const long long*)b2i_meta_put(&a, bits_off, (J + 1) * 8);
  B2_TRY(b2i_meta_commit(&a));
  p.bits = d_bits;
  p.K = K;
  p.sample_rate = src->sample_rate;
  p.start_seconds = src->start_seconds;
  p.sig_ratio = nullptr;
  p.sig_len = nullptr;
  p.sig_words = 0;
  for (size_t j0 = 0; j0 < J; j0 += 65535) {
    p.sig_base = (int)j0;
    dim3 grid((unsigned)std::min<int64_t>((max_cues + 255) / 256, 64), (unsigned)std::min<size_t>(J - j0, 65535));
    raster_bits_kernel<<<grid, 256, 0, h->stream>>>(p);
    B2_CHECK_LAUNCH(h, "raster_bits_kernel");
  }
  return B2_OK;
}

int b2i_raster_bits_dev_launch(b2_ctx* h, const B2CueDev& cues, int n_sig, int64_t max_cues, const double* d_ratio,
                               const long long* d_len, long long sig_words, uint32_t* d_bits) {
  if (n_sig <= 0) return B2_OK;
  B2_CUDA(h, cudaMemsetAsync(d_bits, 0, (size_t)n_sig * sig_words * 4, h->stream));
  if (max_cues == 0) return B2_OK;
  RasterBitsParams p{};
  p.start_s = cues.start;
  p.end_s = cues.end;
  p.keep = cues.keep;
  p.cue_off = cues.cue_off;
  p.bits = d_bits;
  p.K = 1;
  p.sample_rate = cues.sample_rate;
  p.start_seconds = cues.start_seconds;
  p.sig_ratio = d_ratio;
  p.sig_len = d_len;
  p.sig_words = sig_words;
  for (int j0 = 0; j0 < n_sig; j0 += 65535) {
    p.sig_base = j0;
    dim3 grid((unsigned)std::min<int64_t>((max_cues + 255) / 256, 64), (unsigned)std::min(n_sig - j0, 65535));
    raster_bits_kernel<<<grid, 256, 0, h->stream>>>(p);
    B2_CHECK_LAUNCH(h, "raster_bits_kernel");
  }
  return B2_OK;
}

int b2i_bounds_launch(b2_ctx* h, const float* d_sig, const int64_t* off_host, int n,
                      int64_t* d_first, int64_t* d_last) {
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, (size_t)(n + 1) * 8 + 256));
  const long long* d_off = (const long long*)b2i_meta_put(&a, off_host, (size_t)(n + 1) * 8);
  B2_TRY(b2i_meta_commit(&a));
  bounds_kernel<<<n, 256, 0, h->stream>>>(d_sig, d_off, n, (long long*)d_first, (long long*)d_last);
  B2_CHECK_LAUNCH(h, "bounds_kernel");
  return B2_OK;
}

int b2i_reduce_launch(b2_ctx* h, const double* d_score, const int32_t* d_offset,
                      const int32_t* d_status, int B, int K, int64_t max_offset_samples,
                      double* d_best_score, int32_t* d_best_offset, int32_t* d_best_k) {
  B2Range range("b2:reduce_ratios");
  reduce_ratios_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(
      d_score, d_offset, d_status, B, K, (long long)max_offset_samples, d_best_score, d_best_offset, d_best_k);
  B2_CHECK_LAUNCH(h, "reduce_ratios_kernel");
  return B2_OK;
}
