// K3r-K4r: run-length correlation of the subtitle bit masks against a two-level reference (the cue-mode
// path of b2_sync_batch / b2_sync_tracks; arithmetic and error bound in runcorr.cuh, DESIGN.md section 4
// "K4r").  Every score of the window is computed in float64 from exact integer counts; the offsets within
// epsilon of the window maximum go to the same exact re-score and pick as the FFT paths' nominations.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "corr_jobs.cuh"
#include "job_plan.cuh"
#include "runcorr.cuh"

namespace {

using namespace runcorr;
static_assert(kMaxWindow == kRunMaxWindow, "run path window bound");

struct RunRef {        // one video's reference
  long long ref_off;   // element offset of its float signal (packed: word offset of its bits)
  long long q_off;     // entry offset of its packed bits (rc_ref_entries(R) entries)
  int R;
};

struct RunStat {       // one (track, ratio) job of run_corr_kernel
  double mx;           // largest score of the window
  double eps;          // rc_eps of the job
  int total;           // offsets with score >= mx - eps
  int arg;             // largest offset attaining mx
};

// Exclusive prefix sum over the CTA (blockDim.x a multiple of 32); *total = the sum.  sh: 33 ints.
__device__ __forceinline__ int block_excl_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = lane < nw ? sh[lane] : 0;
    const int own = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    sh[lane] = s - own;
    if (lane == 31) sh[32] = s;
  }
  __syncthreads();
  const int r = sh[warp] + x - v;
  *total = sh[32];
  __syncthreads();  // sh is reused by the next call
  return r;
}

// Reference bits of one video per CTA: m = (r == 1.0f), packed 32 to a word with the count of the bits
// below each word (rc_ref_entries layout: a zero guard word before, zero words up to index (R >> 5) + 1).
// A warp turns 32 x 32 consecutive floats into 32 words with ballots (coalesced loads).
__global__ void __launch_bounds__(1024) ref_bits_kernel(const float* __restrict__ ref, const RunRef* __restrict__ vids,
                                                        uint2* __restrict__ q_all) {
  __shared__ int sh[33];
  const RunRef v = vids[blockIdx.x];
  const float* r = ref + v.ref_off;
  uint2* q = q_all + v.q_off;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_words = (v.R >> 5) + 2;  // words 0 .. (R >> 5) + 1
  if (threadIdx.x == 0) q[0] = make_uint2(0u, 0u);
  int carry = 0;
  for (int w0 = 0; w0 < n_words; w0 += blockDim.x) {
    const int wb = w0 + 32 * warp;  // this warp's 32 words
    float x[32];
#pragma unroll
    for (int u = 0; u < 32; ++u) {
      const long long i = 32LL * (wb + u) + lane;
      x[u] = i < v.R ? __ldg(r + i) : 0.f;
    }
    uint32_t mine = 0;
#pragma unroll
    for (int u = 0; u < 32; ++u) {
      const long long i = 32LL * (wb + u) + lane;
      const uint32_t bal = __ballot_sync(0xffffffffu, i < v.R && x[u] == 1.0f);
      if (lane == u) mine = bal;
    }
    const int w = wb + lane;
    int tot;
    const int ex = block_excl_scan(__popc(mine), sh, &tot);
    if (w < n_words) q[w + 1] = make_uint2(mine, (uint32_t)(carry + ex));
    carry += tot;
  }
}

// The same table from a reference the detector wrote as packed bits (words 0 .. (R + 31) / 32 - 1 from
// v.ref_off on, zero past frame R - 1): one coalesced word per thread and a scan of their counts.
__global__ void __launch_bounds__(1024) ref_words_scan_kernel(const uint32_t* __restrict__ ref_words,
                                                              const RunRef* __restrict__ vids,
                                                              uint2* __restrict__ q_all) {
  __shared__ int sh[33];
  const RunRef v = vids[blockIdx.x];
  const uint32_t* r = ref_words + v.ref_off;
  uint2* q = q_all + v.q_off;
  const int n_in = (v.R + 31) >> 5;    // words the detector wrote
  const int n_words = (v.R >> 5) + 2;  // words 0 .. (R >> 5) + 1
  if (threadIdx.x == 0) q[0] = make_uint2(0u, 0u);
  int carry = 0;
  for (int w0 = 0; w0 < n_words; w0 += blockDim.x) {
    const int w = w0 + threadIdx.x;
    const uint32_t mine = w < n_in ? __ldg(r + w) : 0u;
    int tot;
    const int ex = block_excl_scan(__popc(mine), sh, &tot);
    if (w < n_words) q[w + 1] = make_uint2(mine, (uint32_t)(carry + ex));
    carry += tot;
  }
}

// The run path's reference table of every video in vids: from the float reference, or the packed bits
int launch_ref_table(b2_ctx* h, const float* d_ref, bool ref_packed, const RunRef* d_vids, size_t n_vids, uint2* q) {
  if (n_vids == 0) return B2_OK;
  if (ref_packed) {
    ref_words_scan_kernel<<<(unsigned)n_vids, 1024, 0, h->stream>>>(reinterpret_cast<const uint32_t*>(d_ref), d_vids,
                                                                    q);
    B2_CHECK_LAUNCH(h, "ref_words_scan_kernel");
  } else {
    ref_bits_kernel<<<(unsigned)n_vids, 1024, 0, h->stream>>>(d_ref, d_vids, q);
    B2_CHECK_LAUNCH(h, "ref_bits_kernel");
  }
  return B2_OK;
}

// One CTA per (track, ratio) job: blockDim.x / 32 >= ceil(window / 32) threads, thread t owning the offsets
// o_lo + 32 t .. + 31.  Dynamic shared memory: 3 x max_runs ints (run starts, ends, lengths before).
// CAPTURE (b2_capture_nominations): every score also goes, rounded to float32, to the capture row of the job
// (cap.scores[(cap_j0 + j) * cap.stride + offset - o_lo]) from the loop that takes the maximum.
template <bool CAPTURE>
__global__ void __launch_bounds__(kMaxThreads) run_corr_kernel(const SelJob* __restrict__ sel,
                                                                const long long* __restrict__ job_q,
                                                                const uint2* __restrict__ q_all,
                                                                const uint32_t* __restrict__ sub_bits,
                                                                float ref_label, int max_runs,
                                                                RunStat* __restrict__ stat,
                                                                int* __restrict__ cand_off,
                                                                B2Capture cap, long long cap_j0) {
  extern __shared__ int rsm[];
  int* ra = rsm;
  int* rb = ra + max_runs;
  int* rl = rb + max_runs;
  __shared__ int sh[33];
  __shared__ double smx[32];
  __shared__ int sarg[32];
  const int j = blockIdx.x, tid = threadIdx.x, nthr = blockDim.x;
  const SelJob job = sel[j];
  if (job.kind != 0 || job.m_lo > job.m_hi) {
    if (tid == 0) stat[j] = RunStat{-INFINITY, 0.0, 0, 0};
    return;
  }
  const int R = job.R, S = job.S;
  const uint32_t* bits = sub_bits + job.bits_off;
  // 1. runs of the mask: transitions at e in [0, S] (frames < 0 and >= S count as 0), in order
  const int nws = S >> 5;
  int n_end = 0;
  for (int w0 = 0; w0 <= nws; w0 += nthr) {
    const int w = w0 + tid;
    uint32_t t = 0;
    if (w <= nws) {
      const int nb = S - 32 * w;  // valid bits of word w (> 0 except for w = S/32 when S % 32 == 0)
      const uint32_t x = nb >= 32 ? __ldg(bits + w) : (nb > 0 ? __ldg(bits + w) & ((1u << nb) - 1u) : 0u);
      const uint32_t prev = w > 0 ? __ldg(bits + w - 1) : 0u;  // word w-1 lies wholly below S
      t = x ^ ((x << 1) | (prev >> 31));
    }
    int tot;
    int idx = n_end + block_excl_scan(__popc(t), sh, &tot);
    while (t) {
      const int e = 32 * w + __ffs(t) - 1;
      t &= t - 1;
      if (idx < 2 * max_runs) (idx & 1 ? rb : ra)[idx >> 1] = e;
      ++idx;
    }
    n_end += tot;
  }
  const int nr = min(n_end >> 1, max_runs);  // a run holds at least one cue: never cut here
  __syncthreads();
  for (int r0 = 0, carry = 0; r0 < nr; r0 += nthr) {
    const int r = r0 + tid;
    const int len = r < nr ? rb[r] - ra[r] : 0;
    int tot;
    const int ex = block_excl_scan(len, sh, &tot);
    if (r < nr) rl[r] = carry + ex;
    carry += tot;
  }
  __syncthreads();
  // 2. UM over this thread's 32 offsets, then every score
  const uint2* q = q_all + job_q[j];
  const int o_lo = job.o_first + job.m_lo, o_hi = job.o_first + job.m_hi;
  const int o0 = o_lo + kOffsetsPerThread * tid;
  const int n_mine = o0 <= o_hi ? min(kOffsetsPerThread, o_hi - o0 + 1) : 0;
  const RcLevels lv = rc_levels(job.sub_level, ref_label);
  int cnt[32], base = 0;
  if (n_mine > 0) {
    rc_thread_counts(q, R, ra, rb, nr, o0, cnt, base);
  } else {
#pragma unroll
    for (int t = 0; t < 32; ++t) cnt[t] = 0;
  }
  double best = -INFINITY;
  int barg = INT_MIN;
  {
    int um = base;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i < n_mine) {
        const double g = rc_score(q, R, S, ra, rb, rl, nr, o0 + i, um, lv);
        if (CAPTURE) cap.scores[(cap_j0 + j) * cap.stride + kOffsetsPerThread * tid + i] = (float)g;
        if (g >= best) {  // increasing offsets: ties go to the largest
          best = g;
          barg = o0 + i;
        }
      }
      um += cnt[i] - nr;
    }
  }
  // 3. window maximum (ties: largest offset)
  for (int d = 16; d > 0; d >>= 1) {
    const double ob = __shfl_xor_sync(0xffffffffu, best, d);
    const int oa = __shfl_xor_sync(0xffffffffu, barg, d);
    if (ob > best || (ob == best && oa > barg)) {
      best = ob;
      barg = oa;
    }
  }
  if ((tid & 31) == 0) {
    smx[tid >> 5] = best;
    sarg[tid >> 5] = barg;
  }
  __syncthreads();
  double mx = smx[0];
  int arg = sarg[0];
  for (int w = 1; w < (nthr >> 5); ++w)
    if (smx[w] > mx || (smx[w] == mx && sarg[w] > arg)) {
      mx = smx[w];
      arg = sarg[w];
    }
  // 4. nominations: every offset within eps of the maximum, largest first, at most kCandMax
  const double eps = rc_eps((double)min(R, S), lv);
  const double cut = mx - eps;
  uint32_t hit = 0;
  {
    int um = base;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i < n_mine && rc_score(q, R, S, ra, rb, rl, nr, o0 + i, um, lv) >= cut) hit |= 1u << i;
      um += cnt[i] - nr;
    }
  }
  int total;
  const int h = __popc(hit);
  int rank = block_excl_scan(h, sh, &total);
  rank = total - rank - h;  // hits at larger offsets (higher threads)
  while (hit && rank < kCandMax) {
    const int i = 31 - __clz(hit);
    hit &= ~(1u << i);
    cand_off[(size_t)j * kCandMax + rank] = o0 + i;
    ++rank;
  }
  if (tid == 0) stat[j] = RunStat{mx, eps, total, arg};
}

// Per job, once the K jobs of its track are done: winner-only pruning with eps in place of tau, the
// candidate count and the job's slots in the re-score work list (what nominate_select_kernel does on the
// FFT paths).  job_stat = (float) (maximum, eps): what pick_kernel reports for a pruned ratio.
__global__ void __launch_bounds__(128) run_finalize_kernel(const SelJob* __restrict__ sel, int n_jobs, int K,
                                                            int winner_only, const RunStat* __restrict__ stat,
                                                            B2CandBuffers cb) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_jobs) return;
  const SelJob job = sel[j];
  if (job.kind != 0 || job.m_lo > job.m_hi) {
    cb.cand_cnt[j] = 0;
    cb.job_stat[j] = make_float2(-INFINITY, 0.f);
    return;
  }
  const RunStat st = stat[j];
  cb.job_stat[j] = make_float2((float)st.mx, (float)st.eps);
  if (winner_only && !job.no_prune) {
    const int b0 = (j / K) * K;
    double best_floor = -INFINITY;
    for (int k = 0; k < K; ++k) {
      const RunStat s = stat[b0 + k];
      best_floor = fmax(best_floor, s.mx - s.eps);
    }
    // the reported score of a pruned ratio is its maximum rounded to float32: that must stay below
    // the winner's exact score too, or reduce_ratios_kernel could prefer it
    if (fmax(st.mx, (double)(float)st.mx) + st.eps < best_floor) {
      cb.cand_off[(size_t)j * kCandMax] = st.arg;
      cb.cand_cnt[j] = -1;
      return;
    }
  }
  cb.cand_cnt[j] = st.total;
  const int n = min(st.total, kCandMax);
  const int slot = atomicAdd(cb.work_count, n);
  for (int i = 0; i < n; ++i) cb.work_list[slot + i] = (j << 5) | i;
}

}  // namespace

int b2i_align_runs(b2_ctx* h, const float* d_ref, const int64_t* ref_off, int V, const int* trk_off, int K,
                   std::vector<SelJob>& sel, const uint32_t* d_bits, int max_runs, float ref_label, int winner_only,
                   bool ref_packed, const B2CandBuffers& cb, const SelJob** d_sel_out, long long capture_j0) {
  B2Range range("b2:align runs (ref_bits or ref_words_scan, run_corr, finalize)");
  const size_t J = sel.size();
  std::vector<RunRef> vids;
  std::vector<long long> job_q(J, 0);
  long long q_total = 0;
  int max_thr = 32;
  for (int v = 0; v < V; ++v) {
    const int R = (int)(ref_off[v + 1] - ref_off[v]);
    bool any = false;
    for (size_t j = (size_t)trk_off[v] * K; j < (size_t)trk_off[v + 1] * K; ++j) {
      SelJob& s = sel[j];
      if (s.kind != 0) continue;
      // the job's own window: offsets o_first + m_lo .. o_first + m_hi with o_first = its first offset
      const long long w = (long long)s.m_hi - s.m_lo + 1;
      s.o_first = s.m_lo;
      s.m_lo = 0;
      s.m_hi = (int)(w - 1);
      max_thr = std::max<int>(max_thr, (int)(32 * ceil_div64(ceil_div64(w, kOffsetsPerThread), 32)));
      job_q[j] = q_total;
      any = true;
    }
    if (!any) continue;
    vids.push_back(RunRef{(long long)ref_off[v], q_total, R});
    q_total += rc_ref_entries(R);
  }
  if (max_thr > kMaxThreads) B2_FAIL(h, B2_ERR_UNSUPPORTED, "align runs: window wider than %d offsets", kMaxWindow);
  void* d_ws;
  const size_t q_bytes = ((size_t)q_total * 8 + 15) & ~size_t(15);
  B2_TRY(b2i_ws(h, b2_ctx::WS_RUNS, q_bytes + J * sizeof(RunStat) + 64, &d_ws));
  uint2* q = (uint2*)d_ws;
  RunStat* stat = (RunStat*)((char*)d_ws + q_bytes);
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, J * sizeof(SelJob) + J * 8 + vids.size() * sizeof(RunRef) + 256));
  const SelJob* d_sel = (const SelJob*)b2i_meta_put(&a, sel.data(), J * sizeof(SelJob));
  const long long* d_job_q = (const long long*)b2i_meta_put(&a, job_q.data(), J * 8);
  const RunRef* d_vids = vids.empty() ? nullptr : (const RunRef*)b2i_meta_put(&a, vids.data(), vids.size() * sizeof(RunRef));
  B2_TRY(b2i_meta_commit(&a));
  *d_sel_out = d_sel;
  B2_TRY(launch_ref_table(h, d_ref, ref_packed, d_vids, vids.size(), q));
  max_runs = std::max(1, max_runs);
  const size_t smem = (size_t)3 * max_runs * sizeof(int);
  const bool capture = h->capture.scores != nullptr;
  auto kernel = capture ? run_corr_kernel<true> : run_corr_kernel<false>;
  B2_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)J, (unsigned)max_thr, smem, h->stream>>>(d_sel, d_job_q, q, d_bits, ref_label, max_runs, stat,
                                                             cb.cand_off, h->capture, capture_j0);
  B2_CHECK_LAUNCH(h, "run_corr_kernel");
  B2_CUDA(h, cudaMemsetAsync(cb.work_count, 0, sizeof(int), h->stream));
  run_finalize_kernel<<<(unsigned)((J + 127) / 128), 128, 0, h->stream>>>(d_sel, (int)J, K, winner_only, stat, cb);
  B2_CHECK_LAUNCH(h, "run_finalize_kernel");
  // the window scores are in the capture already: win / stat / cand as the finalize left them
  if (capture) B2_TRY(b2i_capture_launch(h, d_sel, nullptr, (int)J, nullptr, cb, capture_j0, /*scores_written=*/true));
  return B2_OK;
}

// ---- GSS rounds (b2_sync_tracks_gss) ----------------------------------------------------------------
// One chain's golden-section search, queued on h->stream with no synchronisation: the packed reference once,
// then per round gss_step_kernel (the round's ratio, length and run-path job per track, from the previous
// round's exact score) -> zero + rasterise the masks at those ratios -> run_corr_kernel -> run_finalize_kernel
// (K = 1) -> rescore_kernel -> pick_kernel, and finally the combine.  Every host-side input of a round is
// uploaded once per chain, in one metadata arena that no later arena of the chain can recycle (the rounds
// begin none).
int b2i_gss_launch(b2_ctx* h, const float* d_ref, const int64_t* ref_off, int V, const int* trk_off, int K,
                   const B2CueSource& src, const double* max_end, int64_t max_offset_samples, const B2GssOut& out) {
  B2Range range("b2:gss rounds (step, raster_bits, run_corr, finalize, rescore, pick) x 17");
  const int T = trk_off[V] - trk_off[0];
  if (T <= 0) return B2_OK;
  // the mask's window holds at most 2 max_offset_samples offsets whatever the length (DESIGN.md "K8g");
  // the caller has checked that this fits one CTA and that every track has at most kRunMaxCues cues
  if (max_offset_samples < 0 || max_offset_samples > kMaxWindow / 2)
    B2_FAIL(h, B2_ERR_UNSUPPORTED, "gss: max_offset_samples %lld is outside [0, %d]", (long long)max_offset_samples,
            kMaxWindow / 2);
  const long long w_bound = std::max<long long>(1, 2 * (long long)max_offset_samples);
  const int max_thr = (int)(32 * ceil_div64(ceil_div64(w_bound, kOffsetsPerThread), 32));
  std::vector<GssTrack> trk(T);
  std::vector<RunRef> vids;
  std::vector<long long> job_q(T, 0);
  long long q_total = 0, sig_words = 1;
  int max_runs = 1;
  const long long c0 = src.cue_off[0], nc = src.cue_off[T] - c0;
  for (int v = 0; v < V; ++v) {
    const long long R = ref_off[v + 1] - ref_off[v];
    if (R < 0 || R > 0x3fffffff) B2_FAIL(h, B2_ERR_BAD_ARG, "gss: bad reference length at %d", v);
    if (trk_off[v + 1] == trk_off[v]) continue;
    vids.push_back(RunRef{(long long)ref_off[v], q_total, (int)R});
    for (int t = trk_off[v]; t < trk_off[v + 1]; ++t) {
      // the mask capacity at the interval's upper end: the length is monotone in the ratio
      const long long s_max = b2_signal_length(max_end[t], B2_GSS_HI, src.sample_rate);
      if (s_max > 0x3fffffff) B2_FAIL(h, B2_ERR_BAD_ARG, "gss: subtitle signal of track %d too long", t);
      sig_words = std::max(sig_words, (s_max >> 5) + 2);
      trk[t] = GssTrack{(long long)ref_off[v], 0, max_end[t], (int)R};
      job_q[t] = q_total;
      max_runs = std::max<int>(max_runs, (int)std::min<long long>(src.cue_off[t + 1] - src.cue_off[t], kRunMaxCues));
    }
    q_total += rc_ref_entries((int)R);
  }
  long long max_cues = 0;
  for (int t = 0; t < T; ++t) {
    trk[t].bits_off = (long long)t * sig_words;
    max_cues = std::max<long long>(max_cues, src.cue_off[t + 1] - src.cue_off[t]);
  }
  std::vector<long long> cue_rel(T + 1);
  for (int t = 0; t <= T; ++t) cue_rel[t] = src.cue_off[t] - c0;

  // device workspace of the chain
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at = (at + bytes + 255) & ~size_t(255); return o; };
  const size_t o_q = take((size_t)q_total * 8), o_stat = take((size_t)T * sizeof(RunStat)),
               o_lane = take((size_t)T * sizeof(B2GssLane)), o_sel = take((size_t)T * sizeof(SelJob)),
               o_x = take((size_t)T * 8), o_len = take((size_t)T * 8), o_rs = take((size_t)T * 8),
               o_ro = take((size_t)T * 4), o_rst = take((size_t)T * 4), o_bits = take((size_t)T * sig_words * 4),
               o_cp = take((size_t)T * kCandMax * kRescoreSeg * 8), o_js = take((size_t)T * 8),
               o_co = take((size_t)T * kCandMax * 4), o_cc = take((size_t)T * 4),
               o_wl = take((size_t)T * kCandMax * 4), o_wc = take(16);
  void* d_ws;
  B2_TRY(b2i_ws(h, b2_ctx::WS_GSS, at + 256, &d_ws));
  char* base = (char*)d_ws;
  uint2* q = (uint2*)(base + o_q);
  RunStat* stat = (RunStat*)(base + o_stat);
  B2GssLane* lane = (B2GssLane*)(base + o_lane);
  SelJob* d_sel = (SelJob*)(base + o_sel);
  double* d_x = (double*)(base + o_x);
  long long* d_len = (long long*)(base + o_len);
  double* r_score = (double*)(base + o_rs);
  int32_t* r_offset = (int32_t*)(base + o_ro);
  int32_t* r_status = (int32_t*)(base + o_rst);
  uint32_t* d_bits = (uint32_t*)(base + o_bits);
  B2CandBuffers cb;
  cb.cand_partial = (double*)(base + o_cp);
  cb.job_stat = (float2*)(base + o_js);
  cb.cand_off = (int*)(base + o_co);
  cb.cand_cnt = (int*)(base + o_cc);
  cb.work_list = (int*)(base + o_wl);
  cb.work_count = (int*)(base + o_wc);

  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, (size_t)nc * 17 + (size_t)(T + 1) * 8 + (size_t)T * (sizeof(GssTrack) + 8) +
                                   vids.size() * sizeof(RunRef) + 1024));
  B2CueDev cues;
  cues.start = (const double*)b2i_meta_put(&a, src.cue_start + c0, (size_t)nc * 8);
  cues.end = (const double*)b2i_meta_put(&a, src.cue_end + c0, (size_t)nc * 8);
  cues.keep = src.cue_keep ? (const uint8_t*)b2i_meta_put(&a, src.cue_keep + c0, (size_t)nc) : nullptr;
  cues.cue_off = (const long long*)b2i_meta_put(&a, cue_rel.data(), (size_t)(T + 1) * 8);
  cues.sample_rate = src.sample_rate;
  cues.start_seconds = src.start_seconds;
  const GssTrack* d_trk = (const GssTrack*)b2i_meta_put(&a, trk.data(), (size_t)T * sizeof(GssTrack));
  const long long* d_job_q = (const long long*)b2i_meta_put(&a, job_q.data(), (size_t)T * 8);
  const RunRef* d_vids = (const RunRef*)b2i_meta_put(&a, vids.data(), vids.size() * sizeof(RunRef));
  B2_TRY(b2i_meta_commit(&a));

  B2_TRY(launch_ref_table(h, d_ref, src.ref_packed, d_vids, vids.size(), q));
  const size_t smem = (size_t)3 * max_runs * sizeof(int);
  B2_CUDA(h, cudaFuncSetAttribute(run_corr_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  for (int r = 0; r < kGssEvals; ++r) {
    B2_TRY(b2i_gss_step_launch(h, r, T, d_trk, lane, r_score, d_sel, d_x, d_len,
                               out.evals, max_offset_samples, src.sample_rate));
    B2_TRY(b2i_raster_bits_dev_launch(h, cues, T, max_cues, d_x, d_len, sig_words, d_bits));
    run_corr_kernel<false><<<(unsigned)T, (unsigned)max_thr, smem, h->stream>>>(
        d_sel, d_job_q, q, d_bits, src.ref_label, max_runs, stat, cb.cand_off, B2Capture{}, 0);
    B2_CHECK_LAUNCH(h, "run_corr_kernel");
    B2_CUDA(h, cudaMemsetAsync(cb.work_count, 0, sizeof(int), h->stream));
    run_finalize_kernel<<<(unsigned)((T + 127) / 128), 128, 0, h->stream>>>(d_sel, T, 1, /*winner_only=*/0, stat, cb);
    B2_CHECK_LAUNCH(h, "run_finalize_kernel");
    B2_TRY(b2i_rescore_pick(h, d_sel, (size_t)T, d_ref, nullptr, d_bits, cb, r_score, r_offset, r_status,
                            src.ref_packed, src.ref_label));
  }
  return b2i_gss_combine_launch(h, T, K, d_trk, d_x, r_score, r_offset, max_offset_samples, out);
}
