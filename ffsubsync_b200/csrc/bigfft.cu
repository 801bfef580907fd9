// Large-window correlation: FFTAligner.fit with max_offset_samples=None (the reference's default,
// ffsubsync/aligners.py:25,67-80) or a mask wider than a few overlap-save tiles.
//
// Instead of tiling the N candidate offsets in 16 385-wide windows (corr.cu; every tile re-transforms
// every block) each signal gets ONE real FFT of the padded length N = 2^k >= R + S, computed as a
// four-step complex FFT of M = N/2 = M1 x 1024 points (bigfft.cuh): columns (F1), rows + untangle
// [+ product + inverse rows] (F2), inverse columns (F3).  The reference spectrum of a video is computed
// once (per slice of its tracks, when they exceed the workspace budget) and reused by the K ratio
// candidates of each of its tracks.  The N fp32 scores only nominate candidates (same
// worst-case round-off bound tau, same selection, exact float64 re-score and argmax as the windowed
// path); the maximum over the N-sized score arrays comes from per-tile maxima of F3, and the selection
// (corr.cu) counts hits per 4 096-offset chunk and compacts only the chunks that hold candidates.
//
// HBM traffic per (pair, ratio) at N = 2^21: F1 3 + 8 MB, F2 16 + 8 MB, F3 8 + 8 MB, selection 8 MB
// (+ 27 MB / K for the reference) against ~105 MFLOP per transform: memory and FP32 work are balanced,
// groups of pairs are sized so that a group's work arrays stay L2-resident between the steps.
#include <math.h>

#include <algorithm>
#include <map>

#include "common.cuh"
#include "bigfft.cuh"
#include "corr_jobs.cuh"

static_assert(kBigMinLog2n == bigfft::kMinQ1 + 11 && kBigMaxLog2n == bigfft::kMaxQ1 + 11,
              "padded lengths of the large-window path");

namespace {

using namespace bigfft;

struct BigXform {        // one transform = one real signal padded to N = 2 M
  long long src_off;     // element offset of the float signal, or word offset of the bit mask
  long long g_off;       // float2 offset of its M-point work array
  long long spec_off;    // reference: where its spectrum is stored (in place: == g_off);
                         // subtitles: the spectrum to multiply with
  long long score_off;   // subtitles: float offset of the N scores
  int len, S, m_lo, m_hi;
  int is_bits;
  float hi;
};

struct BigJob {          // one (pair, ratio) of the group
  int j;                 // global job index b * K + k
  int x_sub, x_ref;      // transform indices inside the group
};

constexpr int kFineCap = (1 << kMaxQ1) + (1 << (kMaxQ1 - 4)) + (1 << (kMaxQ1 - 8)) + 4;   // skewed size
constexpr size_t kBigSmemBytes = kSmemBytes + 1024 * 8 + (size_t)kSkew1024 * 8 + (size_t)kFineCap * 8 + 16 * 8 + 64;

struct Smem {
  float2 *buf, *tw1024, *fine32, *half_pos, *coarse, *fine, *row_tw;
};
__device__ __forceinline__ Smem carve(unsigned char* raw) {
  Smem s;
  s.buf = reinterpret_cast<float2*>(raw);
  s.tw1024 = s.buf + kM;
  s.fine32 = s.tw1024 + 1024;
  s.half_pos = s.fine32 + 32;
  s.coarse = s.half_pos + 1024;
  s.fine = s.coarse + kSkew1024;
  s.row_tw = s.fine + kFineCap;
  return s;
}

// L2 prefetch of what the NEXT tile of this CTA will load (one 512-thread CTA per SM cannot hide HBM
// latency with occupancy; the tile's own loads then hit L2).
__device__ __forceinline__ void l2_prefetch_bulk(const void* p, uint32_t bytes) {   // 16-byte aligned, multiple of 16
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void l2_prefetch_line(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}
// rows of an F2 tile (16 x 8 KB)
__device__ __forceinline__ void prefetch_f2_rows(const float2* base, int q1, int g, int tid) {
  if (tid < 16) l2_prefetch_bulk(base + ((size_t)f2_row_of_slot(q1, g, tid) << 10), kRow * 8);
}
// column group cg of a k1-major [M1][1024] array: M1 segments of cols * 8 bytes
__device__ __forceinline__ void prefetch_cols(const float2* base, int q1, int cg, int tid) {
  const int cl = 14 - q1, c0 = cg << cl, seg = 8 << cl;   // bytes per row segment
  for (int r = tid; r < (1 << q1); r += kThreads) {
    const char* p = reinterpret_cast<const char*>(base + ((size_t)r << 10) + c0);
    for (int b = 0; b < seg; b += 128) l2_prefetch_line(p + b);
  }
}

__device__ __forceinline__ float block_sum(float v, float* red) {   // all threads call; result on every thread
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int w = 0; w < kThreads / 32; ++w) r += red[w];   // fixed order: deterministic
  return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = -INFINITY;
  for (int w = 0; w < kThreads / 32; ++w) r = fmaxf(r, red[w]);
  return r;
}

// F1: forward column transforms + four-step twiddle.  Persistent over (transform, column group) tiles.
template <int Q1>
__global__ void __launch_bounds__(kThreads, 1)
    big_cols_forward_kernel(const float* __restrict__ sig, const uint32_t* __restrict__ bits,
                            const BigXform* __restrict__ xf, int n_tiles, float2* __restrict__ G,
                            float* __restrict__ tile_energy) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[kThreads / 32];
  const Smem sm = carve(smem_raw);
  const int tid = threadIdx.x;
  init_tables(sm.tw1024, sm.fine32, tid);
  init_big_tables(sm.half_pos, sm.coarse, sm.fine, Q1, tid);
  __syncthreads();
  const Tables t{sm.tw1024, sm.fine32};
  const BigTables bt{sm.tw1024, sm.fine32, sm.half_pos, sm.coarse, sm.fine};
  constexpr int tiles_per = (1 << Q1) / 16;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const BigXform X = xf[tile / tiles_per];
    const int cg = tile % tiles_per;
    const BigSource src{X.is_bits ? nullptr : sig + X.src_off, X.is_bits ? bits + X.src_off : nullptr, X.len, X.hi};
    const float ss = block_sum(f1_load(sm.buf, src, Q1, cg, tid), red);   // barriers inside
    if (tid == 0) tile_energy[tile] = ss;
    col_forward<Q1>(sm.buf, t, tid);
    __syncthreads();
    f1_store(sm.buf, bt, Q1, cg, tid, G + X.g_off);
    __syncthreads();
  }
}

// F2: row transforms.  MODE 0 (reference): untangle, store the packed real spectrum in place.
// MODE 1 (subtitles): untangle, conj(A) * B with the pair's stored spectrum, retangle, inverse row
// transforms, conjugate four-step twiddle, store in place.
template <int MODE>
__global__ void __launch_bounds__(kThreads, 1)
    big_rows_kernel(const BigXform* __restrict__ xf, int n_tiles, int q1, float2* __restrict__ G) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const Smem sm = carve(smem_raw);
  const int tid = threadIdx.x;
  init_tables(sm.tw1024, sm.fine32, tid);
  init_big_tables(sm.half_pos, sm.coarse, sm.fine, q1, tid);
  __syncthreads();
  const Tables t{sm.tw1024, sm.fine32};
  const BigTables bt{sm.tw1024, sm.fine32, sm.half_pos, sm.coarse, sm.fine};
  const int tiles_per = (1 << q1) / 16;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const BigXform X = xf[tile / tiles_per];
    const int g = tile % tiles_per;
    if (tile + (int)gridDim.x < n_tiles) {
      const int nt = tile + gridDim.x;
      const BigXform Xn = xf[nt / tiles_per];
      prefetch_f2_rows(G + Xn.g_off, q1, nt % tiles_per, tid);
      if (MODE == 1) prefetch_f2_rows(G + Xn.spec_off, q1, nt % tiles_per, tid);
    }
    f2_load(sm.buf, q1, g, tid, G + X.g_off);
    f2_row_twiddles(sm.row_tw, q1, g, tid);
    __syncthreads();
    rows_forward(sm.buf, t, tid);
    __syncthreads();
    if (MODE == 0) {
      f2_untangle_inplace(sm.buf, bt, q1, g, sm.row_tw, tid);
      __syncthreads();
      f2_store(sm.buf, q1, g, tid, G + X.spec_off);
    } else {
      f2_product_inplace(sm.buf, bt, q1, g, sm.row_tw, tid, G + X.spec_off);
      __syncthreads();
      rows_inverse(sm.buf, t, tid);
      __syncthreads();
      f2_store_twiddled(sm.buf, bt, q1, g, tid, G + X.g_off);
    }
    __syncthreads();
  }
}

// F3: inverse column transforms; scores, their maximum over the surviving window, sum of squares.
template <int Q1>
__global__ void __launch_bounds__(kThreads, 1)
    big_cols_inverse_kernel(const BigXform* __restrict__ xf, int n_tiles, const float2* __restrict__ G,
                            float* __restrict__ scores, float* __restrict__ tile_max,
                            float* __restrict__ tile_cn) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ float red[kThreads / 32];
  const Smem sm = carve(smem_raw);
  const int tid = threadIdx.x;
  init_tables(sm.tw1024, sm.fine32, tid);
  __syncthreads();
  const Tables t{sm.tw1024, sm.fine32};
  constexpr int tiles_per = (1 << Q1) / 16;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const BigXform X = xf[tile / tiles_per];
    const int cg = tile % tiles_per;
    if (tile + (int)gridDim.x < n_tiles) {
      const int nt = tile + gridDim.x;
      prefetch_cols(G + xf[nt / tiles_per].g_off, Q1, nt % tiles_per, tid);
    }
    f3_load(sm.buf, Q1, cg, tid, G + X.g_off);
    __syncthreads();
    col_inverse<Q1>(sm.buf, t, tid);
    __syncthreads();
    float mx = -INFINITY, cn = 0.f;
    f3_store(sm.buf, Q1, cg, tid, scores + X.score_off, X.S, X.m_lo, X.m_hi, mx, cn);
    mx = block_max(mx, red);
    cn = block_sum(cn, red);
    if (tid == 0) {
      tile_max[tile] = mx;
      tile_cn[tile] = cn;
    }
    __syncthreads();
  }
}

// ---- window maximum over N-sized score arrays ------------------------------------------------------
// per job: fp32 maximum over the surviving window and the round-off bound tau (corr_jobs.cuh)
__global__ void __launch_bounds__(256) big_stat_kernel(const BigJob* __restrict__ jobs, int tiles_per,
                                                        const float* __restrict__ ref_energy,
                                                        const float* __restrict__ sub_energy,
                                                        const float* __restrict__ tile_max,
                                                        const float* __restrict__ tile_cn,
                                                        float2* __restrict__ job_stat) {
  const BigJob jb = jobs[blockIdx.x];
  __shared__ float s_es[256], s_er[256], s_cn[256], s_mx[256];
  float es = 0.f, er = 0.f, cn = 0.f, mx = -INFINITY;
  for (int i = threadIdx.x; i < tiles_per; i += 256) {
    es += sub_energy[(size_t)jb.x_sub * tiles_per + i];
    er += ref_energy[(size_t)jb.x_ref * tiles_per + i];
    cn += tile_cn[(size_t)jb.x_sub * tiles_per + i];
    mx = fmaxf(mx, tile_max[(size_t)jb.x_sub * tiles_per + i]);
  }
  s_es[threadIdx.x] = es;
  s_er[threadIdx.x] = er;
  s_cn[threadIdx.x] = cn;
  s_mx[threadIdx.x] = mx;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      s_es[threadIdx.x] += s_es[threadIdx.x + w];
      s_er[threadIdx.x] += s_er[threadIdx.x + w];
      s_cn[threadIdx.x] += s_cn[threadIdx.x + w];
      s_mx[threadIdx.x] = fmaxf(s_mx[threadIdx.x], s_mx[threadIdx.x + w]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float tau = tau_bound(kTauFwd, sqrtf(s_es[0] * s_er[0]), kTauInv, sqrtf(s_cn[0]));
    job_stat[jb.j] = make_float2(s_mx[0], nomination_tau(tau));
  }
}

// jobs that never reach big_stat_kernel (empty input, everything masked) must not look like winners
// to their siblings' winner-only test
__global__ void big_init_stat_kernel(float2* __restrict__ job_stat, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) job_stat[j] = make_float2(-INFINITY, 0.f);
}

template <int Q1>
int launch_cols(b2_ctx* h, bool inverse, const float* d_sig, const uint32_t* d_bits, const BigXform* d_xf,
                int n_tiles, float2* G, float* scores, float* a0, float* a1) {
  const unsigned grid = (unsigned)std::min(n_tiles, h->sm_count);
  if (!inverse) {
    B2_CUDA(h, cudaFuncSetAttribute(big_cols_forward_kernel<Q1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)kBigSmemBytes));
    big_cols_forward_kernel<Q1><<<grid, kThreads, kBigSmemBytes, h->stream>>>(d_sig, d_bits, d_xf, n_tiles, G, a0);
    B2_CHECK_LAUNCH(h, "big_cols_forward_kernel");
  } else {
    B2_CUDA(h, cudaFuncSetAttribute(big_cols_inverse_kernel<Q1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)kBigSmemBytes));
    big_cols_inverse_kernel<Q1><<<grid, kThreads, kBigSmemBytes, h->stream>>>(d_xf, n_tiles, G, scores, a0, a1);
    B2_CHECK_LAUNCH(h, "big_cols_inverse_kernel");
  }
  return B2_OK;
}

int launch_cols_q(b2_ctx* h, int q1, bool inverse, const float* d_sig, const uint32_t* d_bits,
                  const BigXform* d_xf, int n_tiles, float2* G, float* scores, float* a0, float* a1) {
  switch (q1) {
    case 6: return launch_cols<6>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    case 7: return launch_cols<7>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    case 8: return launch_cols<8>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    case 9: return launch_cols<9>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    case 10: return launch_cols<10>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    case 11: return launch_cols<11>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    case 12: return launch_cols<12>(h, inverse, d_sig, d_bits, d_xf, n_tiles, G, scores, a0, a1);
    default: B2_FAIL(h, B2_ERR_UNSUPPORTED, "big align: unsupported transform size 2^%d", q1 + 11);
  }
}

}  // namespace

int b2i_align_big(b2_ctx* h, const float* d_ref, const float* d_sub, const uint32_t* d_bits, int V,
                  const int* trk_off, int K, std::vector<SelJob>& sel, const std::vector<long long>& idx_lo,
                  const std::vector<long long>& idx_hi, const std::vector<long long>& n_pad, int winner_only,
                  const B2CandBuffers& cb, const SelJob** d_sel_out, long long capture_j0) {
  B2Range range("b2:align_big (four-step FFT per signal)");
  const size_t J = (size_t)trk_off[V] * K;
  // transform size of a video = the largest padded length among the live jobs of its tracks (more zero
  // padding changes nothing: each job's offsets and surviving window come from ITS OWN padded length)
  std::map<int, std::vector<int>> videos_by_q1;
  for (int v = 0; v < V; ++v) {
    long long n_max = 0;
    for (size_t j = (size_t)trk_off[v] * K; j < (size_t)trk_off[v + 1] * K; ++j) {
      SelJob& s = sel[j];
      if (s.kind != 0) continue;
      n_max = std::max(n_max, n_pad[j]);
      s.o_first = -s.S;
      s.m_lo = (int)(n_pad[j] - idx_hi[j]);       // m = offset + S = N - 1 - idx
      s.m_hi = (int)(n_pad[j] - 1 - idx_lo[j]);
      s.n_tiles = 1;
      s.n_split = 1;
    }
    if (n_max == 0) continue;
    int lg = 0;
    while ((1LL << lg) < n_max) ++lg;
    videos_by_q1[lg - 11].push_back(v);
  }
  // A group is as many slices as keep the work arrays within the workspace budget.  A slice is a range of
  // tracks of one video with its own reference transform: a whole video when its K ratio jobs per track fit,
  // else as many tracks as fit (one track at least - a track's K jobs stay together, the winner-only test of
  // the selection compares them).
  size_t budget = (size_t)4 << 30;
  if (const char* e = getenv("B2_BIG_WS_MB")) budget = (size_t)std::max(64, atoi(e)) << 20;
  struct Slice { int t0, t1; };
  struct Group { int q1; std::vector<Slice> slices; };
  std::vector<Group> groups;
  for (auto& kv : videos_by_q1) {
    const size_t m = (size_t)1 << (kv.first + 10);
    const size_t per_ref = m * 8, per_track = (size_t)K * (m * 8 + m * 2 * 4);
    const size_t max_tracks = std::max<size_t>(1, budget > per_ref ? (budget - per_ref) / per_track : 0);
    size_t used = 0;
    for (int v : kv.second) {
      for (int t0 = trk_off[v]; t0 < trk_off[v + 1]; t0 += (int)max_tracks) {
        const int t1 = (int)std::min<size_t>(trk_off[v + 1], t0 + max_tracks);
        const size_t cost = per_ref + (size_t)(t1 - t0) * per_track;
        if (groups.empty() || groups.back().q1 != kv.first || (used + cost > budget && used > 0)) {
          groups.push_back({kv.first, {}});
          used = 0;
        }
        groups.back().slices.push_back({t0, t1});
        used += cost;
      }
    }
  }
  // score_off is group-local (the score workspace is reused by the next group)
  size_t max_g = 0, max_scores = 0, max_tiles = 0, max_cnt = 0;
  for (auto& g : groups) {
    const size_t m = (size_t)1 << (g.q1 + 10), n = 2 * m;
    size_t n_sub = 0;
    for (const Slice& sl : g.slices)
      for (size_t j = (size_t)sl.t0 * K; j < (size_t)sl.t1 * K; ++j) {
        SelJob& s = sel[j];
        if (s.kind != 0) continue;
        s.score_off = (long long)(n_sub * n);
        ++n_sub;
      }
    const size_t tiles_per = ((size_t)1 << g.q1) / 16;
    max_g = std::max(max_g, (g.slices.size() + n_sub) * m);
    max_scores = std::max(max_scores, n_sub * n);
    max_tiles = std::max(max_tiles, (g.slices.size() + 3 * n_sub) * tiles_per);
    max_cnt = std::max(max_cnt, n_sub * ((n + kChunk - 1) / kChunk));
  }
  // The job table is read by kernels of EVERY group and by the common tail, i.e. long after later
  // metadata arenas have been committed - outside the reuse contract of the arena ring (a slot may be
  // recycled 8 arenas later).  It lives in its own workspace.
  void *d_selv, *h_selv;
  B2_TRY(b2i_ws(h, b2_ctx::WS_META, J * sizeof(SelJob) + 256, &d_selv));
  // staged through a pinned buffer of the handle (a copy from pageable memory would first wait for
  // the stream to drain); the event guards the buffer against the next call
  if (!h->pinned_ev[0]) B2_CUDA(h, cudaEventCreateWithFlags(&h->pinned_ev[0], cudaEventDisableTiming));
  B2_CUDA(h, cudaEventSynchronize(h->pinned_ev[0]));
  B2_TRY(b2i_pinned(h, 0, J * sizeof(SelJob) + 256, &h_selv));
  memcpy(h_selv, sel.data(), J * sizeof(SelJob));
  B2_CUDA(h, cudaMemcpyAsync(d_selv, h_selv, J * sizeof(SelJob), cudaMemcpyHostToDevice, h->stream));
  B2_CUDA(h, cudaEventRecord(h->pinned_ev[0], h->stream));
  const SelJob* d_sel = (const SelJob*)d_selv;
  *d_sel_out = d_sel;
  B2_CUDA(h, cudaMemsetAsync(cb.work_count, 0, sizeof(int), h->stream));
  B2_CUDA(h, cudaMemsetAsync(cb.cand_cnt, 0, J * sizeof(int), h->stream));   // jobs that are not live: no candidates
  big_init_stat_kernel<<<(unsigned)((J + 255) / 256), 256, 0, h->stream>>>(cb.job_stat, (int)J);
  B2_CHECK_LAUNCH(h, "big_init_stat_kernel");
  // capture: the jobs that join no group (empty input, all masked) now, the others after their group
  const bool capture = h->capture.scores != nullptr;
  if (capture) B2_TRY(b2i_capture_launch(h, d_sel, nullptr, (int)J, nullptr, cb, capture_j0));
  if (groups.empty()) return B2_OK;

  void *d_g, *d_s;
  B2_TRY(b2i_ws(h, b2_ctx::WS_SPEC, max_g * 8 + 256, &d_g));
  B2_TRY(b2i_ws(h, b2_ctx::WS_SCORES, max_scores * 4 + max_tiles * 4 + max_cnt * 4 + 1024, &d_s));
  float2* G = (float2*)d_g;
  float* scores = (float*)d_s;
  float* tile_arr = scores + max_scores;                 // ref_energy | sub_energy | tile_max | tile_cn
  int* chunk_cnt = (int*)(tile_arr + max_tiles);
  B2_CUDA(h, cudaFuncSetAttribute(big_rows_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)kBigSmemBytes));
  B2_CUDA(h, cudaFuncSetAttribute(big_rows_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)kBigSmemBytes));

  for (auto& g : groups) {
    const int q1 = g.q1;
    const size_t m = (size_t)1 << (q1 + 10), n = 2 * m;
    const int tiles_per = (1 << q1) / 16;
    std::vector<BigXform> xr, xs;
    std::vector<BigJob> jobs;
    for (size_t pi = 0; pi < g.slices.size(); ++pi) {
      const Slice& sl = g.slices[pi];
      BigXform r;
      memset(&r, 0, sizeof(r));
      bool have_ref = false;
      for (size_t j = (size_t)sl.t0 * K; j < (size_t)sl.t1 * K; ++j) {
        const SelJob& s = sel[j];
        if (s.kind != 0) continue;
        if (!have_ref) {
          r.src_off = s.ref_off;
          r.len = s.R;
          r.g_off = (long long)(pi * m);
          r.spec_off = r.g_off;
          have_ref = true;
        }
        BigXform x;
        memset(&x, 0, sizeof(x));
        x.is_bits = s.bits_off >= 0 ? 1 : 0;
        x.src_off = x.is_bits ? s.bits_off : s.sub_off;
        x.hi = 2.f * s.sub_level - 1.f;
        x.len = s.S;
        x.S = s.S;
        x.m_lo = s.m_lo;
        x.m_hi = s.m_hi;
        x.g_off = (long long)((g.slices.size() + xs.size()) * m);
        x.spec_off = r.g_off;
        x.score_off = s.score_off;
        jobs.push_back({(int)j, (int)xs.size(), (int)pi});
        xs.push_back(x);
      }
      xr.push_back(r);   // a slice without live jobs keeps a zero-length dummy (never referenced)
    }
    const int n_ref = (int)xr.size(), n_sub = (int)xs.size();
    if (n_sub == 0) continue;
    std::vector<int> jlist;   // the group's global job indices (selection, capture)
    for (const BigJob& jb : jobs) jlist.push_back(jb.j);
    MetaArena ga;
    B2_TRY(b2i_meta_begin(h, &ga, (xr.size() + xs.size()) * sizeof(BigXform) + jobs.size() * sizeof(BigJob) +
                                      jlist.size() * sizeof(int) + 256));
    const BigXform* d_xr = (const BigXform*)b2i_meta_put(&ga, xr.data(), xr.size() * sizeof(BigXform));
    const BigXform* d_xs = (const BigXform*)b2i_meta_put(&ga, xs.data(), xs.size() * sizeof(BigXform));
    const BigJob* d_jobs = (const BigJob*)b2i_meta_put(&ga, jobs.data(), jobs.size() * sizeof(BigJob));
    const int* d_jlist = (const int*)b2i_meta_put(&ga, jlist.data(), jlist.size() * sizeof(int));
    B2_TRY(b2i_meta_commit(&ga));
    float* ref_energy = tile_arr;
    float* sub_energy = ref_energy + (size_t)n_ref * tiles_per;
    float* tile_max = sub_energy + (size_t)n_sub * tiles_per;
    float* tile_cn = tile_max + (size_t)n_sub * tiles_per;
    const int n_chunks = (int)((n + kChunk - 1) / kChunk);
    const unsigned rows_grid_r = (unsigned)std::min(n_ref * tiles_per, h->sm_count);
    const unsigned rows_grid_s = (unsigned)std::min(n_sub * tiles_per, h->sm_count);

    B2_TRY(launch_cols_q(h, q1, false, d_ref, nullptr, d_xr, n_ref * tiles_per, G, nullptr, ref_energy, nullptr));
    big_rows_kernel<0><<<rows_grid_r, kThreads, kBigSmemBytes, h->stream>>>(d_xr, n_ref * tiles_per, q1, G);
    B2_CHECK_LAUNCH(h, "big_rows_kernel<ref>");
    B2_TRY(launch_cols_q(h, q1, false, d_sub, d_bits, d_xs, n_sub * tiles_per, G, nullptr, sub_energy, nullptr));
    big_rows_kernel<1><<<rows_grid_s, kThreads, kBigSmemBytes, h->stream>>>(d_xs, n_sub * tiles_per, q1, G);
    B2_CHECK_LAUNCH(h, "big_rows_kernel<sub>");
    B2_TRY(launch_cols_q(h, q1, true, nullptr, nullptr, d_xs, n_sub * tiles_per, G, scores, tile_max, tile_cn));
    big_stat_kernel<<<n_sub, 256, 0, h->stream>>>(d_jobs, tiles_per, ref_energy, sub_energy, tile_max, tile_cn,
                                                  cb.job_stat);
    B2_CHECK_LAUNCH(h, "big_stat_kernel");
    // before the next group overwrites the score workspace
    B2_TRY(b2i_select_launch(h, d_sel, d_jlist, n_sub, scores, n_chunks, K, winner_only, chunk_cnt, cb));
    if (capture) B2_TRY(b2i_capture_launch(h, d_sel, d_jlist, n_sub, scores, cb, capture_j0));
  }
  return B2_OK;
}
