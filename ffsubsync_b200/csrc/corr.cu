// K3-K5: batched cross-correlation of reference / subtitle speech signals over a window of
// candidate offsets, + exact re-scoring and argmax.  Replaces FFTAligner.fit
// (ffsubsync/aligners.py:50-80, mask :31-43, argmax :45-48).
//
// What the reference computes (SURVEY.md section 8a, rows A1-A4), in closed form:
//     score(o) = sum_j s'[j] * r'[j + o],   x' = 2x - 1,  terms outside either signal = 0
// for the offsets o = N-1-idx-S that survive the max_offset mask, and returns the maximum
// (first index = largest offset among equals).
//
// How it is computed here.  Only a window [o_lo, o_hi] of offsets is wanted (12 000 of them for
// the default --max-offset-seconds 60), so the subtitle signal is cut into blocks of
// L = P - W + 1 samples; each block and the P reference samples it can meet are transformed with
// a P = 2^15 point real FFT that lives entirely in shared memory, conj(A)*B is accumulated over
// the blocks in registers, and ONE inverse transform yields the W scores (overlap-save
// correlation).  The reference-side spectra are computed once per video and reused by all K
// ratio candidates of each of its subtitle tracks (b2_sync_batch: one track per video).  The fp32 scores only nominate candidates: every offset within a first-order
// worst-case round-off bound (tau, below) of the maximum is re-scored exactly (float64 direct sum), so the returned
// offset and score do not depend on FFT round-off.  Offset ranges wider than P/2 are tiled.
#include <math.h>

#include <algorithm>
#include <cmath>

#include "align_path.h"
#include "common.cuh"
#include "corr.cuh"
#include "corr_jobs.cuh"
#include "job_plan.cuh"

namespace {

using namespace corr;
static_assert(kP == kAlignBlock, "overlap-save block of the host planner");

struct SpecItem {      // one reference block to transform
  long long ref_off;   // element offset of the pair's reference signal
  int R;
  int i0;              // reference index of sample 0 of the block (may be negative)
};

struct SubJob {        // one (pair, ratio, offset tile)
  long long sub_off;
  long long score_off; // where the tile's Wt scores go
  long long spec_base; // index of the spectrum of block blk_lo
  int S, blk_lo, blk_hi, n_out, energy_slot;
  // bit-mask mode (b2_sync_batch): the subtitle signal is one bit per frame (raster_bits_kernel)
  long long bits_off;  // word offset of this (pair, ratio)'s speech bit mask
  float hi;            // 2*min(1/ratio, 1) - 1: value of a frame inside a cue after x -> 2x-1
};

// bit-mask mode: the speech bits of the current and the next block (kP/32 words each) sit behind
// the twiddle tables in shared memory
constexpr size_t kSmemBytesBits = kSmemBytes + 2 * (size_t)(kP / 32) * 4;

// Bulk L2 prefetch (16-byte aligned address, size a multiple of 16).
__device__ __forceinline__ void l2_prefetch(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}

// ------------------------------------------------------------------------------------------
// Bulk L2 prefetch of [p, p + n floats), trimmed to 16-byte granules inside the range.
__device__ __forceinline__ void l2_prefetch_floats(const float* p, int n) {
  if (n <= 0) return;
  const uintptr_t a0 = (reinterpret_cast<uintptr_t>(p) + 15) & ~uintptr_t(15);
  const uintptr_t a1 = reinterpret_cast<uintptr_t>(p + n) & ~uintptr_t(15);
  if (a1 > a0) l2_prefetch(reinterpret_cast<const void*>(a0), (uint32_t)(a1 - a0));
}

// Persistent over the reference blocks (one CTA per SM): twiddle tables are built once per CTA
// and the next item's samples are pulled into L2 while the current one is transformed.
__global__ void __maxnreg__(96)  // leaves registers for a co-resident VAD CTA of b2_sync_batch's pipeline
    ref_spectra_kernel(const float* __restrict__ ref, const SpecItem* __restrict__ items, int n_items,
                       float4* __restrict__ spec, float* __restrict__ spec_energy) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* buf = reinterpret_cast<float2*>(smem_raw);
  float2* tw1024 = buf + kM;
  float2* fine32 = tw1024 + 1024;
  __shared__ float red[kThreads / 32];
  const int tid = threadIdx.x;
  init_tables(tw1024, fine32, tid);
  __syncthreads();
  const Tables t{tw1024, fine32};
  const PairCtx pc = pair_ctx(t, tid);
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const SpecItem it = items[item];
    if (tid == 0 && item + (int)gridDim.x < n_items) {
      const SpecItem nx = items[item + gridDim.x];
      const int lo = nx.i0 < 0 ? -nx.i0 : 0, hi = min(nx.R - nx.i0, kP);
      l2_prefetch_floats(ref + nx.ref_off + nx.i0 + lo, hi - lo);
    }
    float ss = float_pass1(buf, t, tid, ref + it.ref_off + it.i0, it.i0 < 0 ? -it.i0 : 0,
                           min(it.R - it.i0, kP));
    forward_rest(buf, t, tid);
    spec_store(buf, t, pc, tid, spec + (size_t)item * kPairs);
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    if ((tid & 31) == 0) red[tid >> 5] = ss;
    __syncthreads();  // also: every thread is done reading buf before the next item overwrites it
    if (tid == 0) {
      float e = 0.f;
      for (int w = 0; w < kThreads / 32; ++w) e += red[w];
      spec_energy[item] = e;
    }
  }
}

// BITS = false: the subtitle signal is a float array in global memory (b2_align_batch).
// BITS = true : it is a bit mask, one bit per frame (b2_sync_batch: raster_bits_kernel writes the
//   K masks of a pair straight from the cue list, 1/32 of the bytes of the float signals, and the
//   exact re-score reads the same masks).  The words of block blk+1 are fetched while block blk is
//   transformed (registers -> shared memory, double buffered).
// The 64 accumulator floats of each thread (conj(A)*B summed over the blocks) live in registers:
// 128 registers x 512 threads is the whole register file of an SM, and shared memory is taken by
// the transform buffer (a further 128 KB of accumulators would exceed the 227 KB a block may use).
template <bool BITS>
__device__ __forceinline__ void sub_correlate_body(
    const float* __restrict__ sub, const SubJob* __restrict__ jobs, const float4* __restrict__ spec,
    const float* __restrict__ spec_energy, int L, float* __restrict__ scores,
    float4* __restrict__ job_energy, const uint32_t* __restrict__ sub_bits) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float2* buf = reinterpret_cast<float2*>(smem_raw);
  float2* tw1024 = buf + kM;
  float2* fine32 = tw1024 + 1024;
  uint32_t* bit_words = reinterpret_cast<uint32_t*>(smem_raw + kSmemBytes);  // [2][kP/32] (BITS only)
  __shared__ float red[kThreads / 32];
  const int tid = threadIdx.x;
  const SubJob job = jobs[blockIdx.x];
  float* out = scores + job.score_off;
  if (job.blk_lo >= job.blk_hi) {  // no subtitle block meets the reference at these offsets
    for (int m = tid; m < job.n_out; m += kThreads) out[m] = 0.f;
    if (tid == 0) job_energy[job.energy_slot] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  init_tables(tw1024, fine32, tid);
  const int wpb = L >> 5;  // mask words per block (L is a multiple of 32)
  const uint32_t* bits = BITS ? sub_bits + job.bits_off : nullptr;
  if (BITS) {
    const uint32_t* src = bits + (long long)job.blk_lo * wpb;
    uint32_t* dst = bit_words + (job.blk_lo & 1) * (kP / 32);
    for (int w = tid; w < wpb; w += kThreads) dst[w] = __ldg(src + w);
  }
  __syncthreads();
  const Tables t{tw1024, fine32};
  const PairCtx pc = pair_ctx(t, tid);
  SubState st;
  sub_state_clear(st);
  float er = 0.f;
  for (int blk = job.blk_lo; blk < job.blk_hi; ++blk) {
    const int j0 = blk * L;
    const bool more = blk + 1 < job.blk_hi;
    if (tid == 0 && more) {
      // pull the next block's samples and reference spectrum into L2 while this block computes
      const int jn = j0 + L;
      if (!BITS) l2_prefetch_floats(sub + job.sub_off + jn, min(job.S - jn, L));
      l2_prefetch(spec + (size_t)(job.spec_base + (blk + 1 - job.blk_lo)) * kPairs, kPairs * 16);
    }
    uint32_t nw0 = 0, nw1 = 0;  // next block's mask words: loaded now, parked in smem after the math
    if (BITS) {
      const uint32_t* src = bits + (long long)(blk + 1) * wpb;
      if (more && tid < wpb) nw0 = __ldg(src + tid);
      if (more && tid + kThreads < wpb) nw1 = __ldg(src + tid + kThreads);
      st.ss += bits_pass1(buf, t, tid, bit_words + (blk & 1) * (kP / 32), min(job.S - j0, L), L, job.hi);
      forward_rest(buf, t, tid);
    } else {
      BlockSource s;
      s.src = sub + job.sub_off + j0;
      s.t_lo = 0;
      s.t_hi = min(job.S - j0, L);
      st.ss += forward_block(buf, t, tid, s);
    }
    const size_t item = (size_t)(job.spec_base + (blk - job.blk_lo));
    sub_accumulate(st, buf, t, pc, tid, spec + item * kPairs);
    er += spec_energy[item];
    if (BITS) {  // the other buffer was last read in block blk-1's first pass
      uint32_t* dst = bit_words + ((blk + 1) & 1) * (kP / 32);
      dst[tid] = nw0;
      dst[tid + kThreads] = nw1;
    }
    __syncthreads();  // buf is rewritten by the next block's first pass
  }
  sub_retangle_store(st, buf, t, pc, tid);
  __syncthreads();
  inverse_passes_1(buf, tid);
  __syncthreads();
  inverse_passes_2(buf, t, tid);
  __syncthreads();
  inverse_passes_3(buf, t, tid);
  __syncthreads();
  inverse_passes_4(buf, t, tid);
  __syncthreads();
  for (int m = tid; m < job.n_out; m += kThreads) out[m] = window_value(buf, m);
  // ||c||_2^2 of the whole inverse-transform output (all kP real values, in score units): the
  // quantity the inverse transform's round-off is relative to (tau, window_max_kernel)
  float cn = 0.f;
  for (int i = tid; i < kM; i += kThreads) {
    const float2 z = buf[i];
    cn = fmaf(z.x, z.x, fmaf(z.y, z.y, cn));
  }
  cn *= kOutScale * kOutScale;
  float ss = st.ss;
  for (int o = 16; o > 0; o >>= 1) {
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    cn += __shfl_xor_sync(0xffffffffu, cn, o);
  }
  __shared__ float red2[kThreads / 32];
  if ((tid & 31) == 0) {
    red[tid >> 5] = ss;
    red2[tid >> 5] = cn;
  }
  __syncthreads();
  if (tid == 0) {
    float e = 0.f, c2 = 0.f;
    for (int w = 0; w < kThreads / 32; ++w) {
      e += red[w];
      c2 += red2[w];
    }
    job_energy[job.energy_slot] = make_float4(e, er, c2, (float)(job.blk_hi - job.blk_lo));
  }
}

// Product kernel, one CTA of 512 threads per SM (accumulators in registers, see above).
__global__ void __launch_bounds__(kThreads, 1)
    sub_correlate_kernel(const float* __restrict__ sub, const SubJob* __restrict__ jobs,
                         const float4* __restrict__ spec, const float* __restrict__ spec_energy,
                         int L, float* __restrict__ scores, float4* __restrict__ job_energy) {
  sub_correlate_body<false>(sub, jobs, spec, spec_energy, L, scores, job_energy, nullptr);
}

// b2_sync_batch: subtitle signals as bit masks (no float subtitle signal in HBM).
__global__ void __launch_bounds__(kThreads, 1)
    sub_correlate_bits_kernel(const SubJob* __restrict__ jobs, const float4* __restrict__ spec,
                              const float* __restrict__ spec_energy, int L,
                              float* __restrict__ scores, float4* __restrict__ job_energy,
                              const uint32_t* __restrict__ sub_bits) {
  sub_correlate_body<true>(nullptr, jobs, spec, spec_energy, L, scores, job_energy, sub_bits);
}

// ---- window maximum ----------------------------------------------------------------------------
// fp32 maximum of the surviving window and the round-off bound tau, per (pair, ratio).
__global__ void __launch_bounds__(256) window_max_kernel(const SelJob* __restrict__ jobs,
                                                          float* __restrict__ scores,
                                                          const float4* __restrict__ job_energy,
                                                          float2* __restrict__ job_stat, int wt) {
  const SelJob job = jobs[blockIdx.x];
  const int tid = threadIdx.x;
  __shared__ float smax[256];
  if (job.kind != 0 || job.m_lo > job.m_hi) {
    if (tid == 0) job_stat[blockIdx.x] = make_float2(-INFINITY, 0.f);
    return;
  }
  float* c = scores + job.score_off;
  if (job.n_split > 1) {  // add the partial score arrays (fixed order: deterministic) into the first
    const int n = job.n_tiles * wt;
    for (int m = tid; m < n; m += 256) {
      float v = c[m];
      for (int sp = 1; sp < job.n_split; ++sp) v += c[(size_t)sp * n + m];
      c[m] = v;
    }
    __syncthreads();
  }
  float mx = -INFINITY;
  for (int m = job.m_lo + tid; m <= job.m_hi; m += 256) mx = fmaxf(mx, c[m]);
  smax[tid] = mx;
  __syncthreads();
  for (int w = 128; w > 0; w >>= 1) {
    if (tid < w) smax[tid] = fmaxf(smax[tid], smax[tid + w]);
    __syncthreads();
  }
  if (tid == 0) {
    float tau = 0.f;
    for (int i = 0; i < job.n_tiles; ++i) {
      // energies add over the chunks of a tile (Cauchy-Schwarz); the norms of the partial inverse
      // transforms add (triangle inequality); blocks beyond kTauBlocks add u each to the
      // accumulation term
      float ex = 0.f, ey = 0.f, cn = 0.f, blocks = 0.f;
      for (int sp = 0; sp < job.n_split; ++sp) {
        const float4 e = job_energy[job.energy_slot + i * job.n_split + sp];
        ex += e.x;
        ey += e.y;
        cn += sqrtf(e.z);
        blocks = fmaxf(blocks, e.w);
      }
      const float fwd = kTauFwd + fmaxf(0.f, blocks - (float)kTauBlocks);
      tau = fmaxf(tau, tau_bound(fwd, sqrtf(ex * ey), kTauInv + (float)(job.n_split - 1), cn));
    }
    job_stat[blockIdx.x] = make_float2(smax[0], nomination_tau(tau));
  }
}

// ---- candidate selection (both paths) --------------------------------------------------------------
// Per (pair, ratio): every offset whose fp32 score is within tau of the fp32 maximum (job_stat), taken
// from the LARGEST offset down (np.argmax returns the lowest index = largest offset among equal values;
// offset o = o_first + m, so that is the largest m), at most kCandMax of them.  nominate_count_kernel
// counts the hits per kChunk-offset chunk of m, nominate_select_kernel walks only the chunks that hold
// hits.  Job i of a launch is jlist[i] (NULL: i).

// The cut of a job: fp32 maximum minus tau.  With winner_only (b2_sync_batch when only the best ratio
// is wanted) a (pair, ratio) whose fp32 maximum cannot reach the best ratio's even after round-off
// (mx + tau < max_k (mx_k - tau_k)) is not re-scored: it keeps only its fp32 argmax (cut = mx) and is
// flagged B2_ALIGN_APPROX.  Off for a pair with no_prune set.
__device__ __forceinline__ float nomination_cut(const SelJob& job, const float2* __restrict__ job_stat, int j,
                                                int K, int winner_only, bool& approx_only) {
  const float2 stat = job_stat[j];
  approx_only = false;
  if (winner_only && !job.no_prune) {
    const int b0 = (j / K) * K;
    float best_floor = -INFINITY;
    for (int k = 0; k < K; ++k) {
      const float2 s = job_stat[b0 + k];
      best_floor = fmaxf(best_floor, s.x - s.y);
    }
    if (stat.x + stat.y < best_floor) {
      approx_only = true;
      return stat.x;
    }
  }
  return stat.x - stat.y;
}

// Grid: jobs on x, chunks on y (a grid-stride loop: a window may have more than 65 535 chunks).
__global__ void __launch_bounds__(256) nominate_count_kernel(const SelJob* __restrict__ sel,
                                                              const int* __restrict__ jlist,
                                                              const float* __restrict__ scores,
                                                              const float2* __restrict__ job_stat, int K,
                                                              int winner_only, int n_chunks,
                                                              int* __restrict__ chunk_cnt) {
  const int j = jlist ? jlist[blockIdx.x] : (int)blockIdx.x;
  const SelJob job = sel[j];
  if (job.kind != 0 || job.m_lo > job.m_hi) return;  // nominate_select_kernel reads no count
  __shared__ int s_cnt[8];
  bool approx;
  const float cut = nomination_cut(job, job_stat, j, K, winner_only, approx);
  const float* c = scores + job.score_off;
  for (int ch = blockIdx.y; ch < n_chunks; ch += gridDim.y) {
    const int lo = max(job.m_lo, ch * kChunk), hi = min(job.m_hi, ch * kChunk + (kChunk - 1));
    int cnt = 0;
    for (int m = lo + threadIdx.x; m <= hi; m += 256) cnt += c[m] >= cut;
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) tot += s_cnt[w];
      chunk_cnt[(size_t)blockIdx.x * n_chunks + ch] = tot;
    }
    __syncthreads();  // s_cnt is rewritten by the next chunk
  }
}

// Ordered compaction, one CTA per job; publishes the job's candidates to the re-score work list.
__global__ void __launch_bounds__(256) nominate_select_kernel(const SelJob* __restrict__ sel,
                                                               const int* __restrict__ jlist,
                                                               const float* __restrict__ scores,
                                                               const float2* __restrict__ job_stat, int K,
                                                               int winner_only, int n_chunks,
                                                               const int* __restrict__ chunk_cnt,
                                                               int* __restrict__ cand_off,
                                                               int* __restrict__ cand_cnt,
                                                               int* __restrict__ work_list,
                                                               int* __restrict__ work_count) {
  const int j = jlist ? jlist[blockIdx.x] : (int)blockIdx.x;
  const SelJob job = sel[j];
  const int tid = threadIdx.x;
  __shared__ int scount;
  __shared__ int swarp[8];
  if (job.kind != 0 || job.m_lo > job.m_hi) {
    if (tid == 0) cand_cnt[j] = 0;
    return;
  }
  bool approx_only;
  const float cut = nomination_cut(job, job_stat, j, K, winner_only, approx_only);
  const float* c = scores + job.score_off;
  // 1. the (at most kCandMax) highest chunks that hold candidates, in descending order, and the total
  __shared__ int hit_chunk[kCandMax];
  __shared__ int n_hit, s_total;
  if (tid == 0) {
    scount = 0;
    n_hit = 0;
    s_total = 0;
  }
  __syncthreads();
  const int* cnt = chunk_cnt + (size_t)blockIdx.x * n_chunks;
  for (int top = n_chunks - 1; top >= 0; top -= 256) {
    const int ch = top - tid;
    const int here = ch >= 0 ? cnt[ch] : 0;
    const unsigned ball = __ballot_sync(0xffffffffu, here > 0);
    int wsum = here;
    for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
    if ((tid & 31) == 0) {
      swarp[tid >> 5] = __popc(ball);
      atomicAdd(&s_total, wsum);
    }
    __syncthreads();
    int before = n_hit;
    for (int w = 0; w < (tid >> 5); ++w) before += swarp[w];
    before += __popc(ball & ((1u << (tid & 31)) - 1u));
    if (here > 0 && before < kCandMax) hit_chunk[before] = ch;
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < 8; ++w) tot += swarp[w];
      n_hit += tot;
    }
    __syncthreads();
  }
  const int total = s_total;
  const int n_walk = min(n_hit, kCandMax);
  // 2. ordered compaction inside those chunks
  for (int h = 0; h < n_walk; ++h) {
    if (scount >= kCandMax) break;  // uniform: scount is read after a barrier
    const int ch = hit_chunk[h];
    const int lo = max(job.m_lo, ch * kChunk), hi = min(job.m_hi, ch * kChunk + (kChunk - 1));
    for (int top = hi; top >= lo; top -= 256) {
      const int m = top - tid;
      const bool hit = (m >= lo) && (c[m] >= cut);
      const unsigned ball = __ballot_sync(0xffffffffu, hit);
      if ((tid & 31) == 0) swarp[tid >> 5] = __popc(ball);
      __syncthreads();
      int before = scount;
      for (int w = 0; w < (tid >> 5); ++w) before += swarp[w];
      before += __popc(ball & ((1u << (tid & 31)) - 1u));
      if (hit && before < kCandMax) cand_off[(size_t)j * kCandMax + before] = job.o_first + m;
      __syncthreads();
      if (tid == 0) {
        int tot = 0;
        for (int w = 0; w < 8; ++w) tot += swarp[w];
        scount += tot;
      }
      __syncthreads();
    }
  }
  if (approx_only) {  // slot 0 holds the largest offset attaining the fp32 maximum
    if (tid == 0) cand_cnt[j] = -1;
    return;
  }
  if (tid == 0) {
    cand_cnt[j] = total;
    scount = min(total, kCandMax);
    swarp[0] = atomicAdd(work_count, scount);  // slots in the global re-score work list
  }
  __syncthreads();
  if (tid < scount) work_list[swarp[0] + tid] = (j << 5) | tid;
}

// ---- exact re-score ----------------------------------------------------------------------------
// score(o) = sum over the overlap of (2 s[j] - 1)(2 r[j+o] - 1) in float64.  Each candidate's
// overlap is cut into kRescoreSeg segments handled by different CTAs (persistent grid over the
// work list); every partial sum has a fixed summation order and pick_kernel adds the partials in
// segment order, so the result is deterministic.
// PACKED_REF (run-path chains whose detector wrote packed bits): `ref` holds, from job.ref_off on, the words of
// the reference's bits m = (r == 1.0f); frame value r = m ? 1.0f : ref_label is rebuilt as a float, so every
// product and the summation order are those of the float reference, and the sums are bit-identical.  The float
// variant (every other chain) reads the float signal and never its last argument.
template <bool PACKED_REF>
__global__ void __launch_bounds__(256) rescore_kernel(const SelJob* __restrict__ jobs,
                                                       const float* __restrict__ ref,
                                                       const float* __restrict__ sub,
                                                       const int* __restrict__ cand_off,
                                                       const int* __restrict__ work_list,
                                                       const int* __restrict__ work_count,
                                                       const uint32_t* __restrict__ sub_bits,
                                                       double* __restrict__ cand_partial, float ref_label) {
  __shared__ double sh[256];
  const int total = *work_count * kRescoreSeg;
  for (int w = blockIdx.x; w < total; w += gridDim.x) {
    const int item = work_list[w / kRescoreSeg], seg = w % kRescoreSeg;
    const int j = item >> 5, ci = item & 31;
    const SelJob job = jobs[j];
    const int o = cand_off[(size_t)j * kCandMax + ci];
    const float* r = ref + job.ref_off;
    const float* s = sub + job.sub_off;
    const int j_lo = max(0, -o), j_hi = min(job.S, job.R - o);
    const int len = max(0, j_hi - j_lo);
    const int per = (len + kRescoreSeg - 1) / kRescoreSeg;
    const int a0 = j_lo + seg * per, a1 = min(j_hi, a0 + per);
    double acc = 0.0;
    int i = a0 + threadIdx.x;
    if (PACKED_REF) {
      // both signals as bits (cue mode): reference frame i + o >= 0 is bit (i + o) & 31 of its word, the same
      // bit position for all u as for the mask
      const uint32_t* bits = sub_bits + job.bits_off;
      const uint32_t* rbits = reinterpret_cast<const uint32_t*>(ref) + job.ref_off;
      const double hi = 2.0 * (double)job.sub_level - 1.0;
      const int rsh = (i + o) & 31;
      for (; i + 7 * 256 < a1; i += 8 * 256) {  // 16 independent loads in flight per thread
        uint32_t bw[8];
        float rv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          bw[u] = __ldg(bits + ((i + u * 256) >> 5));
          rv[u] = ((__ldg(rbits + ((i + u * 256 + o) >> 5)) >> rsh) & 1u) ? 1.0f : ref_label;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u)
          acc = fma(((bw[u] >> (i & 31)) & 1u) ? hi : -1.0, 2.0 * (double)rv[u] - 1.0, acc);
      }
      for (; i < a1; i += 256) {
        const double a = ((__ldg(bits + (i >> 5)) >> (i & 31)) & 1u) ? hi : -1.0;
        const float rv = ((__ldg(rbits + ((i + o) >> 5)) >> rsh) & 1u) ? 1.0f : ref_label;
        acc = fma(a, 2.0 * (double)rv - 1.0, acc);
      }
    } else if (job.bits_off >= 0) {
      // bit-mask mode: subtitle frame i is bit i of the mask written by raster_bits_kernel;
      // its value after x -> 2x-1 is (2*level - 1) inside a cue and -1 outside
      const uint32_t* bits = sub_bits + job.bits_off;
      const double hi = 2.0 * (double)job.sub_level - 1.0;
      for (; i + 7 * 256 < a1; i += 8 * 256) {  // 16 independent loads in flight per thread
        uint32_t bw[8];
        float rv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          bw[u] = __ldg(bits + ((i + u * 256) >> 5));
          rv[u] = __ldg(r + i + u * 256 + o);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u)  // 256 = 0 (mod 32): the bit position is the same for all u
          acc = fma(((bw[u] >> (i & 31)) & 1u) ? hi : -1.0, 2.0 * (double)rv[u] - 1.0, acc);
      }
      for (; i < a1; i += 256) {
        const double a = ((__ldg(bits + (i >> 5)) >> (i & 31)) & 1u) ? hi : -1.0;
        const double b = 2.0 * (double)__ldg(r + i + o) - 1.0;
        acc = fma(a, b, acc);
      }
    }
    for (; i + 3 * 256 < a1; i += 4 * 256) {  // 8 independent loads in flight per thread
      float sv[4], rv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        sv[u] = __ldg(s + i + u * 256);
        rv[u] = __ldg(r + i + u * 256 + o);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        acc = fma(2.0 * (double)sv[u] - 1.0, 2.0 * (double)rv[u] - 1.0, acc);
    }
    for (; i < a1; i += 256) {
      const double a = 2.0 * (double)__ldg(s + i) - 1.0;
      const double b = 2.0 * (double)__ldg(r + i + o) - 1.0;
      acc = fma(a, b, acc);
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int h = 128; h > 0; h >>= 1) {
      if (threadIdx.x < h) sh[threadIdx.x] += sh[threadIdx.x + h];
      __syncthreads();
    }
    if (threadIdx.x == 0) cand_partial[((size_t)j * kCandMax + ci) * kRescoreSeg + seg] = sh[0];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(128) pick_kernel(const SelJob* __restrict__ jobs, int n_jobs,
                                                    const int* __restrict__ cand_off,
                                                    const int* __restrict__ cand_cnt,
                                                    const double* __restrict__ cand_partial,
                                                    const float2* __restrict__ job_stat,
                                                    double* __restrict__ score,
                                                    int32_t* __restrict__ offset,
                                                    int32_t* __restrict__ status) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_jobs) return;
  const SelJob job = jobs[j];
  if (job.kind == 1) {
    score[job.out_index] = 0.0;
    offset[job.out_index] = 0;
    status[job.out_index] = B2_ALIGN_EMPTY;
    return;
  }
  if (job.kind == 2 || job.m_lo > job.m_hi) {
    score[job.out_index] = -INFINITY;  // np.argmax of an all -inf array: index 0
    offset[job.out_index] = job.masked_offset;
    status[job.out_index] = B2_ALIGN_ALL_MASKED;
    return;
  }
  const int cnt = cand_cnt[j];
  if (cnt < 0) {  // winner_only: this ratio cannot win, fp32 result reported
    score[job.out_index] = (double)job_stat[j].x;
    offset[job.out_index] = cand_off[(size_t)j * kCandMax];
    status[job.out_index] = B2_ALIGN_APPROX;
    return;
  }
  const int n = min(cnt, kCandMax);
  double bs = -INFINITY;
  int bo = 0;
  for (int c = 0; c < n; ++c) {
    double s = 0.0;
    for (int g = 0; g < kRescoreSeg; ++g) s += cand_partial[((size_t)j * kCandMax + c) * kRescoreSeg + g];
    const int o = cand_off[(size_t)j * kCandMax + c];
    if (c == 0 || s > bs || (s == bs && o > bo)) {
      bs = s;
      bo = o;
    }
  }
  score[job.out_index] = bs;
  offset[job.out_index] = bo;
  status[job.out_index] = cnt > kCandMax ? B2_ALIGN_CAND_OVERFLOW : B2_ALIGN_OK;
}

// ---- diagnostics: b2_capture_nominations ----------------------------------------------------------
// One CTA per job: the fp32 scores of its surviving window (m_lo..m_hi, offset o_first + m), its
// (maximum, tau) and its candidate count, as the selection kernels left them.  scores_written: the run
// path's kernel has written the window scores; only (maximum, epsilon) and the count are left.
__global__ void __launch_bounds__(256) capture_nominations_kernel(const SelJob* __restrict__ jobs,
                                                                   const int* __restrict__ jlist,
                                                                   const float* __restrict__ scores,
                                                                   const float2* __restrict__ job_stat,
                                                                   const int* __restrict__ cand_cnt,
                                                                   B2Capture cap, long long j0, int scores_written) {
  const int j = jlist ? jlist[blockIdx.x] : (int)blockIdx.x;
  const SelJob job = jobs[j];
  const bool live = job.kind == 0 && job.m_lo <= job.m_hi;
  if (live && !scores && !scores_written) return;  // written by the launch that has its scores
  const long long g = j0 + j;
  const int n = live ? job.m_hi - job.m_lo + 1 : 0;
  if (threadIdx.x == 0) {
    const float2 s = job_stat[j];
    cap.win[2 * g] = live ? (long long)job.o_first + job.m_lo : 0;
    cap.win[2 * g + 1] = n;
    cap.stat[2 * g] = s.x;
    cap.stat[2 * g + 1] = s.y;
    cap.cand[g] = cand_cnt[j];
  }
  if (n == 0 || scores_written) return;
  const float* c = scores + job.score_off + job.m_lo;
  float* out = cap.scores + g * cap.stride;
  for (int i = threadIdx.x; i < n; i += 256) out[i] = c[i];
}

// ---- host planning ----------------------------------------------------------------------------
long long floor_div(long long a, long long b) {
  long long q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) --q;
  return q;
}

}  // namespace

int b2i_select_launch(b2_ctx* h, const SelJob* d_sel, const int* d_jlist, int n, const float* scores,
                      int n_chunks, int K, int winner_only, int* chunk_cnt, const B2CandBuffers& cb) {
  if (n <= 0) return B2_OK;
  const dim3 grid((unsigned)n, (unsigned)std::min(n_chunks, 65535));
  nominate_count_kernel<<<grid, 256, 0, h->stream>>>(d_sel, d_jlist, scores, cb.job_stat, K, winner_only,
                                                     n_chunks, chunk_cnt);
  B2_CHECK_LAUNCH(h, "nominate_count_kernel");
  nominate_select_kernel<<<(unsigned)n, 256, 0, h->stream>>>(d_sel, d_jlist, scores, cb.job_stat, K, winner_only,
                                                             n_chunks, chunk_cnt, cb.cand_off, cb.cand_cnt,
                                                             cb.work_list, cb.work_count);
  B2_CHECK_LAUNCH(h, "nominate_select_kernel");
  return B2_OK;
}

int b2i_capture_launch(b2_ctx* h, const SelJob* d_sel, const int* d_jlist, int n, const float* scores,
                       const B2CandBuffers& cb, long long j0, bool scores_written) {
  if (n <= 0) return B2_OK;
  capture_nominations_kernel<<<(unsigned)n, 256, 0, h->stream>>>(d_sel, d_jlist, scores, cb.job_stat, cb.cand_cnt,
                                                                  h->capture, j0, scores_written ? 1 : 0);
  B2_CHECK_LAUNCH(h, "capture_nominations_kernel");
  return B2_OK;
}

int b2i_align_launch(b2_ctx* h, const float* d_ref, const int64_t* ref_off, int V, const int* trk_off,
                     const float* d_sub, const int64_t* sub_off, int B, int K, int64_t max_offset_samples,
                     double* d_score, int32_t* d_offset, int32_t* d_status, int winner_only,
                     const B2CueSource* cue_src, long long capture_j0) {
  B2Range range("b2:align (ref_spectra, sub_correlate, select, rescore, pick)");
  const size_t J = (size_t)B * K;
  std::vector<int> ident;   // no track table: reference b is read by pair b alone
  if (!trk_off) {
    ident.resize(B + 1);
    for (int b = 0; b <= B; ++b) ident[b] = b;
    trk_off = ident.data();
    V = B;
  }
  // cue mode (b2_sync_batch): the subtitle signals exist only as bit masks, rasterised from the cue
  // list by raster_bits_kernel below (sub_off then only carries the signal lengths)
  const bool cue_mode = cue_src != nullptr;
  // the jobs, windows and tiling (align_path.h: the sync calls' planner runs the same code)
  B2AlignJobs aj;
  if (const int st = b2_plan_align_jobs(ref_off, V, trk_off, sub_off, B, K, max_offset_samples, h->log2_quirk_mask,
                                        cue_mode ? cue_src->ratios : nullptr, &aj)) {
    h->err = aj.err;
    return st;
  }
  std::vector<SelJob>& sel = aj.sel;
  const std::vector<long long>& bits_off = aj.bits_off;
  std::vector<B2AlignPairPlan>& pp = aj.pp;
  const long long max_w = aj.max_w;
  const bool capture = h->capture.scores != nullptr;
  if (capture)
    for (size_t j = 0; j < J; ++j)
      if (sel[j].kind == 0 && (long long)sel[j].m_hi - sel[j].m_lo + 1 > h->capture.stride)
        B2_FAIL(h, B2_ERR_BAD_ARG, "capture: job %lld has %lld surviving offsets, stride %lld",
                capture_j0 + (long long)j, (long long)sel[j].m_hi - sel[j].m_lo + 1, h->capture.stride);
  const int Wt = aj.Wt, L = aj.L;
  uint32_t* d_bits = nullptr;
  if (cue_mode) {
    void* db;
    B2_TRY(b2i_ws(h, b2_ctx::WS_SIG_SUB, (size_t)bits_off[J] * 4 + 64, &db));
    d_bits = (uint32_t*)db;
    B2_TRY(b2i_raster_bits_launch(h, cue_src, B, K, sub_off, bits_off.data(), d_bits));
    B2_CUDA(h, cudaFuncSetAttribute(sub_correlate_bits_kernel,
                                    cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytesBits));
  }
  void* d_cand;
  B2_TRY(b2i_ws(h, b2_ctx::WS_CAND, J * kCandMax * (8 * kRescoreSeg + 8) + J * 12 + 64, &d_cand));
  B2CandBuffers cb;
  cb.cand_partial = (double*)d_cand;
  cb.job_stat = (float2*)(cb.cand_partial + J * kCandMax * kRescoreSeg);
  cb.cand_off = (int*)(cb.job_stat + J);
  cb.cand_cnt = cb.cand_off + J * kCandMax;
  cb.work_list = cb.cand_cnt + J;
  cb.work_count = cb.work_list + J * kCandMax;
  if (J >= (1u << 26)) B2_FAIL(h, B2_ERR_UNSUPPORTED, "align: B*K too large for one call");

  // the path (align_path.h); B2_ALIGN_PATH=tiled|big|runs: test / A-B knob
  const B2AlignPathChoice path =
      b2_align_path(aj, trk_off, V, K, cue_mode ? cue_src->cue_off : nullptr, cue_mode && cue_src->ref_two_level,
                    cue_mode ? cue_src->ref_label : 0.0f, getenv("B2_ALIGN_PATH"), capture);
  // a packed reference (the detector wrote bits, no floats) is planned for run-path chains only
  const bool ref_packed = cue_mode && cue_src->ref_packed;
  if (ref_packed && path.path != B2_PATH_RUNS)
    B2_FAIL(h, B2_ERR_UNSUPPORTED, "align: internal error: packed reference on a chain that takes the %s path",
            path.path == B2_PATH_BIG ? "large-window" : "tiled");
  if (path.path == B2_PATH_RUNS) {
    const SelJob* d_sel_runs = nullptr;
    B2_TRY(b2i_align_runs(h, d_ref, ref_off, V, trk_off, K, sel, d_bits, path.max_runs, cue_src->ref_label,
                          winner_only, ref_packed, cb, &d_sel_runs, capture_j0));
    return b2i_rescore_pick(h, d_sel_runs, J, d_ref, d_sub, d_bits, cb, d_score, d_offset, d_status, ref_packed,
                            cue_src->ref_label);
  }
  if (path.path == B2_PATH_BIG) {
    const SelJob* d_sel_big = nullptr;
    B2_TRY(b2i_align_big(h, d_ref, d_sub, d_bits, V, trk_off, K, sel, aj.idx_lo, aj.idx_hi, aj.n_pad, winner_only,
                         cb, &d_sel_big, capture_j0));
    return b2i_rescore_pick(h, d_sel_big, J, d_ref, d_sub, d_bits, cb, d_score, d_offset, d_status);
  }

  // score buffers + per-(pair,ratio) bookkeeping
  // Small batches: with fewer (pair, ratio, tile) jobs than SMs the block loop of a job (35 blocks
  // for a 2 h signal) would run on a handful of SMs.  The block range of every job is then cut into
  // n_split chunks, each CTA inverse-transforms its own partial accumulator (the inverse FFT is
  // linear) into its own partial score array, and window_max_kernel adds the partial arrays in a
  // fixed order.  Costs one extra inverse transform per chunk, so chunks keep >= 4 blocks.
  long long n_jobs_total = 0, max_blocks = 1;
  for (int v = 0; v < V; ++v) {
    B2AlignPairPlan& p = pp[v];
    p.n_tiles = p.any ? (int)ceil_div64(p.o_max - p.o_min + 1, Wt) : 0;
    for (size_t j = (size_t)trk_off[v] * K; j < (size_t)trk_off[v + 1] * K; ++j) {
      const SelJob& s = sel[j];
      if (s.kind != 0) continue;
      n_jobs_total += p.n_tiles;
      max_blocks = std::max<long long>(max_blocks, ceil_div64(s.S, L));
    }
  }
  int n_split = 1;
  if (n_jobs_total > 0 && n_jobs_total < 2LL * h->sm_count)
    n_split = (int)std::max<long long>(1, std::min<long long>(ceil_div64(2LL * h->sm_count, n_jobs_total),
                                                               max_blocks / 4));
  if (const char* e = getenv("B2_ALIGN_SPLIT")) n_split = std::max(1, atoi(e));  // test / tuning knob
  long long score_total = 0, energy_total = 0, max_score_len = 0;
  for (int v = 0; v < V; ++v) {
    B2AlignPairPlan& p = pp[v];
    for (size_t j = (size_t)trk_off[v] * K; j < (size_t)trk_off[v + 1] * K; ++j) {
      SelJob& s = sel[j];
      if (s.kind != 0) continue;
      max_score_len = std::max(max_score_len, (long long)p.n_tiles * Wt);
      s.o_first = (int)p.o_min;
      s.m_lo -= (int)p.o_min;
      s.m_hi -= (int)p.o_min;
      s.score_off = score_total;
      s.energy_slot = (int)energy_total;
      s.n_tiles = p.n_tiles;
      s.n_split = n_split;
      score_total += (long long)p.n_tiles * Wt * n_split;
      energy_total += (long long)p.n_tiles * n_split;
    }
  }

  const int n_chunks = (int)std::max<long long>(1, ceil_div64(max_score_len, kChunk));
  void* d_scores;
  B2_TRY(b2i_ws(h, b2_ctx::WS_SCORES,
                (size_t)(score_total + 16) * 4 + (size_t)(energy_total + 2) * 16 + J * n_chunks * 4, &d_scores));
  float* scores = (float*)d_scores;
  float4* job_energy = (float4*)((char*)d_scores + (((size_t)(score_total + 16) * 4 + 15) & ~size_t(15)));
  int* chunk_cnt = (int*)(job_energy + energy_total);

  B2_CUDA(h, cudaFuncSetAttribute(ref_spectra_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)kSmemBytes));
  B2_CUDA(h, cudaFuncSetAttribute(sub_correlate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)kSmemBytes));

  // Work is issued in groups so that the reference spectra of a group fit the workspace cap.
  const size_t kSpecBytes = (size_t)kPairs * 16;
  const size_t cap_items = std::max<size_t>(64, ((size_t)6 << 30) / kSpecBytes);
  std::vector<SpecItem> items;
  std::vector<SubJob> jobs;
  auto flush = [&]() -> int {
    if (jobs.empty()) {
      items.clear();
      return B2_OK;
    }
    void* d_spec;
    B2_TRY(b2i_ws(h, b2_ctx::WS_SPEC, items.size() * kSpecBytes + items.size() * 4 + 256, &d_spec));
    float4* spec = (float4*)d_spec;
    float* spec_energy = (float*)((char*)d_spec + items.size() * kSpecBytes);
    MetaArena a;
    B2_TRY(b2i_meta_begin(h, &a, items.size() * sizeof(SpecItem) + jobs.size() * sizeof(SubJob) + 256));
    const SpecItem* d_items = (const SpecItem*)b2i_meta_put(&a, items.data(), items.size() * sizeof(SpecItem));
    const SubJob* d_jobs = (const SubJob*)b2i_meta_put(&a, jobs.data(), jobs.size() * sizeof(SubJob));
    B2_TRY(b2i_meta_commit(&a));
    if (!items.empty()) {
      // persistent: one CTA per SM
      const unsigned grid = (unsigned)std::min<size_t>(items.size(), (size_t)h->sm_count);
      ref_spectra_kernel<<<grid, kThreads, kSmemBytes, h->stream>>>(d_ref, d_items, (int)items.size(),
                                                                    spec, spec_energy);
      B2_CHECK_LAUNCH(h, "ref_spectra_kernel");
    }
    if (cue_mode)
      sub_correlate_bits_kernel<<<(unsigned)jobs.size(), kThreads, kSmemBytesBits, h->stream>>>(
          d_jobs, spec, spec_energy, L, scores, job_energy, d_bits);
    else
      sub_correlate_kernel<<<(unsigned)jobs.size(), kThreads, kSmemBytes, h->stream>>>(
          d_sub, d_jobs, spec, spec_energy, L, scores, job_energy);
    B2_CHECK_LAUNCH(h, "sub_correlate_kernel");
    items.clear();
    jobs.clear();
    return B2_OK;
  };

  // the reference blocks of a (video, tile) are transformed once and read by every track and ratio of the video
  for (int v = 0; v < V; ++v) {
    const B2AlignPairPlan& p = pp[v];
    if (!p.any) continue;
    const long long R = ref_off[v + 1] - ref_off[v];
    const size_t j_lo = (size_t)trk_off[v] * K, j_hi = (size_t)trk_off[v + 1] * K;
    long long nblk_max = 0;
    for (size_t j = j_lo; j < j_hi; ++j) {
      const SelJob& s = sel[j];
      if (s.kind == 0) nblk_max = std::max<long long>(nblk_max, ceil_div64(s.S, L));
    }
    for (int tile = 0; tile < p.n_tiles; ++tile) {
      const long long o_t = p.o_min + (long long)tile * Wt;
      const long long blk_lo = std::max(0LL, floor_div(-o_t - kP, L) + 1);
      const long long blk_hi = std::min<long long>(nblk_max, R - o_t > 0 ? ceil_div64(R - o_t, L) : 0LL);
      const long long n_items = std::max(0LL, blk_hi - blk_lo);
      if (items.size() + (size_t)n_items > cap_items) B2_TRY(flush());
      const long long spec_base = (long long)items.size();
      for (long long blk = blk_lo; blk < blk_hi; ++blk) {
        SpecItem it;
        it.ref_off = ref_off[v];
        it.R = (int)R;
        it.i0 = (int)(blk * L + o_t);
        items.push_back(it);
      }
      for (size_t j = j_lo; j < j_hi; ++j) {
        const SelJob& s = sel[j];
        if (s.kind != 0) continue;
        const long long job_hi = std::min<long long>(blk_hi, ceil_div64(s.S, L));
        const long long n_blk = std::max(0LL, job_hi - blk_lo);
        for (int sp = 0; sp < n_split; ++sp) {
          const long long c_lo = blk_lo + n_blk * sp / n_split, c_hi = blk_lo + n_blk * (sp + 1) / n_split;
          SubJob jb;
          jb.sub_off = s.sub_off;
          jb.S = s.S;
          jb.score_off = s.score_off + ((long long)sp * p.n_tiles + tile) * Wt;
          jb.spec_base = spec_base + (c_lo - blk_lo);
          jb.blk_lo = (int)c_lo;
          jb.blk_hi = (int)c_hi;
          jb.n_out = Wt;
          jb.energy_slot = s.energy_slot + tile * n_split + sp;
          jb.bits_off = 0;
          jb.hi = 0.f;
          if (cue_mode) {
            jb.bits_off = s.bits_off;
            jb.hi = 2.f * s.sub_level - 1.f;  // the value load_block16 gives the float signal
          }
          jobs.push_back(jb);
        }
      }
    }
  }
  B2_TRY(flush());

  B2Range range_sel("b2:select+rescore+pick");

  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, J * sizeof(SelJob) + 256));
  const SelJob* d_sel = (const SelJob*)b2i_meta_put(&a, sel.data(), J * sizeof(SelJob));
  B2_TRY(b2i_meta_commit(&a));
  B2_CUDA(h, cudaMemsetAsync(cb.work_count, 0, sizeof(int), h->stream));
  window_max_kernel<<<(unsigned)J, 256, 0, h->stream>>>(d_sel, scores, job_energy, cb.job_stat, Wt);
  B2_CHECK_LAUNCH(h, "window_max_kernel");
  B2_TRY(b2i_select_launch(h, d_sel, nullptr, (int)J, scores, n_chunks, K, winner_only, chunk_cnt, cb));
  if (capture) B2_TRY(b2i_capture_launch(h, d_sel, nullptr, (int)J, scores, cb, capture_j0));
  return b2i_rescore_pick(h, d_sel, J, d_ref, d_sub, d_bits, cb, d_score, d_offset, d_status);
}

int b2i_rescore_pick(b2_ctx* h, const SelJob* d_sel, size_t J, const float* d_ref, const float* d_sub,
                     const uint32_t* d_bits, const B2CandBuffers& cb, double* d_score, int32_t* d_offset,
                     int32_t* d_status, bool ref_packed, float ref_label) {
  auto rescore = ref_packed ? rescore_kernel<true> : rescore_kernel<false>;
  rescore<<<(unsigned)(h->sm_count * 8), 256, 0, h->stream>>>(
      d_sel, d_ref, d_sub, cb.cand_off, cb.work_list, cb.work_count, d_bits, cb.cand_partial, ref_label);
  B2_CHECK_LAUNCH(h, "rescore_kernel");
  pick_kernel<<<(unsigned)((J + 127) / 128), 128, 0, h->stream>>>(d_sel, (int)J, cb.cand_off, cb.cand_cnt,
                                                                   cb.cand_partial, cb.job_stat, d_score,
                                                                   d_offset, d_status);
  B2_CHECK_LAUNCH(h, "pick_kernel");
  return B2_OK;
}
