// K9s: per-segment offsets with a split penalty over the reference signals of a finished batched sync call
// (b2_split_tracks; objective and arithmetic in split.cuh, DESIGN.md section 4 "K9s").  The chain, all on the
// handle's stream: split_ref_kernel (each video's two levels and its packed bits) -> raster_bits_kernel (the
// tracks' masks at their own ratios) -> per track group split_dp_kernel (the programme, one CTA per track, a
// switch word per unit and thread to the workspace) -> split_backtrack_kernel (the path, its score and the
// per-cue offsets).  b2_split_tracks_capped (at most N segments) runs split_capped_dp_kernel (N layers of the
// programme on one cluster per track) and split_capped_backtrack_kernel in the last two places;
// b2_split_tracks_directed (offsets monotone in one direction) split_directed_dp_kernel and
// split_directed_backtrack_kernel.
#include <limits.h>
#include <math.h>

#include <algorithm>
#include <type_traits>

#include <cooperative_groups.h>

#include "common.cuh"
#include "job_plan.cuh"
#include "split.cuh"

using namespace split;
namespace cg = cooperative_groups;

namespace {

struct SplitVideo {
  long long ref_off;   // element offset of its frames
  long long q_off;     // entry offset of its packed bits (rc_ref_entries(R) entries)
  int R;
};

struct SplitLevel {
  double beta;         // the level other than 1.0 (0.0 when every frame is 1.0)
  long long bad;       // first frame with a third level (or a non-finite beta), -1 if none
};

struct SplitTrack {
  long long q_off, bits_off, unit_base, dec_base;
  long long c0, c1;    // cue range, relative to the uploaded cue arrays
  double ratio;
  float level;
  int vid;             // index into the prepared videos
  int R, S, o_lo, W, nthr, live;
};

// One CTA per video: beta = the first frame != 1.0, the first frame that is neither 1.0 nor beta, and the
// run path's packed table (rc_ref_entries layout) of m = (r == 1.0), 32 x 32 frames per warp with ballots.
template <typename T>
__global__ void __launch_bounds__(1024) split_ref_kernel(const T* __restrict__ ref, const SplitVideo* __restrict__ vids,
                                                         uint2* __restrict__ q_all, SplitLevel* __restrict__ lvl) {
  __shared__ int sh[33];
  __shared__ int s_first, s_bad;
  const SplitVideo v = vids[blockIdx.x];
  const T* r = ref + v.ref_off;
  uint2* q = q_all + v.q_off;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    s_first = INT_MAX;
    s_bad = INT_MAX;
    q[0] = make_uint2(0u, 0u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < v.R; i += blockDim.x)
    if ((double)r[i] != 1.0) {  // a thread's first hit is its smallest
      atomicMin(&s_first, i);
      break;
    }
  __syncthreads();
  const double beta = s_first < v.R ? (double)r[s_first] : 0.0;
  if (threadIdx.x == 0 && s_first < v.R && !isfinite(beta)) atomicMin(&s_bad, s_first);
  const int n_words = (v.R >> 5) + 2;  // words 0 .. (R >> 5) + 1
  int carry = 0;
  for (int w0 = 0; w0 < n_words; w0 += blockDim.x) {
    const int wb = w0 + 32 * warp;  // this warp's 32 words
    uint32_t mine = 0;
#pragma unroll 4
    for (int u = 0; u < 32; ++u) {
      const long long i = 32LL * (wb + u) + lane;
      const double x = i < v.R ? (double)__ldg(r + i) : 0.0;
      if (i < v.R && x != 1.0 && x != beta) atomicMin(&s_bad, (int)i);
      const uint32_t bal = __ballot_sync(0xffffffffu, i < v.R && x == 1.0);
      if (lane == u) mine = bal;
    }
    const int w = wb + lane;
    int tot;
    const int ex = runcorr::rc_block_excl_scan(__popc(mine), sh, &tot);
    if (w < n_words) q[w + 1] = make_uint2(mine, (uint32_t)(carry + ex));
    carry += tot;
  }
  __syncthreads();
  if (threadIdx.x == 0) lvl[blockIdx.x] = SplitLevel{beta, s_bad < v.R ? (long long)s_bad : -1LL};
}

// One track per cluster of C CTAs (kCluster false: a plain launch, C = 1), the tracks order[g0 + cluster]: cluster
// thread g = rank * blockDim.x + tid owns the offsets o_lo + 32 g .. + 31.  Every CTA decodes the runs into its own
// dynamic shared memory (2 x max_runs ints: run starts, ends).  Per unit j >= 1 each thread writes its switch word to
// dec[dec_base + j * nthr + g] (nthr: the track's threads over the whole cluster), rank 0's thread 0 the unit's
// argmax to arg[unit_base + j]; rank 0 writes the runs to runs[unit_base + r].
//
// Barriers: the early exit depends on the track alone, so a cluster takes it as a whole, before any barrier or
// shared-memory traffic.  Otherwise every CTA runs the same nu units (all decode the same runs), each with one
// __syncthreads and one cluster barrier whether or not it owns offsets, then one final cluster barrier, so no CTA
// exits while another may still read its slots.  CTA and cluster slots alternate between units: a slot written
// at unit j + 2 was last read at unit j, before the barriers of unit j + 1.
template <bool kCluster>
__global__ void __launch_bounds__(kCtaThreads) split_dp_kernel(const SplitTrack* __restrict__ trk,
                                                               const int* __restrict__ order, int g0,
                                                               const uint2* __restrict__ q_all,
                                                               const SplitLevel* __restrict__ lvl,
                                                               const uint32_t* __restrict__ sub_bits, int max_runs,
                                                               double penalty, uint32_t* __restrict__ dec,
                                                               int* __restrict__ arg, int2* __restrict__ runs,
                                                               int* __restrict__ n_units) {
  extern __shared__ int rsm[];
  int* ra = rsm;
  int* rb = ra + max_runs;
  __shared__ int sh[33];
  __shared__ double smx[2][kCtaThreads / 32];
  __shared__ int sarg[2][kCtaThreads / 32];
  __shared__ double cmx[2];
  __shared__ int carg[2];
  int C = 1, rank = 0;
  if constexpr (kCluster) {
    C = (int)cg::this_cluster().num_blocks();
    rank = (int)cg::this_cluster().block_rank();
  }
  const int t = order[g0 + (int)blockIdx.x / C], tid = threadIdx.x, nw = blockDim.x >> 5;
  const SplitTrack k = trk[t];
  if (!k.live || lvl[k.vid].bad >= 0) {
    if (rank == 0 && tid == 0) n_units[t] = k.live ? -1 : 0;
    return;
  }
  const int n_end = runcorr::rc_decode_runs(sub_bits + k.bits_off, k.S, max_runs, ra, rb, sh);
  const int nr = min(n_end >> 1, max_runs);
  __syncthreads();
  if (rank == 0) {
    for (int r = tid; r < nr; r += blockDim.x) runs[k.unit_base + r] = make_int2(ra[r], rb[r]);
    if (nr == 0 && tid == 0) runs[k.unit_base] = make_int2(0, 0);  // no run: the one unit [0, S)
  }
  const int nu = nr > 0 ? nr : 1;
  const uint2* q = q_all + k.q_off;
  const SpLevels l = sp_levels(k.level, lvl[k.vid].beta);
  const int g = rank * (int)blockDim.x + tid;
  const int o0 = k.o_lo + kOffsetsPerThread * g;
  const int n_mine = max(0, min(kOffsetsPerThread, k.W - kOffsetsPerThread * g));
  double v[32];
  double c = 0.0;
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra, rb, nr, k.S, j);
    double best = -INFINITY;
    int barg = INT_MIN;
    uint32_t d = 0;
    if (n_mine > 0) d = sp_thread_step(q, k.R, u, o0, n_mine, j == 0, c, l, v, best, barg);
    if (j > 0 && g < k.nthr) dec[k.dec_base + (long long)j * k.nthr + g] = d;
    // unit maximum (ties: largest offset): the warp, the CTA's warps, then the cluster's CTAs
    for (int s = 16; s > 0; s >>= 1)
      sp_merge(best, barg, __shfl_xor_sync(0xffffffffu, best, s), __shfl_xor_sync(0xffffffffu, barg, s));
    if ((tid & 31) == 0) {
      smx[j & 1][tid >> 5] = best;
      sarg[j & 1][tid >> 5] = barg;
    }
    __syncthreads();
    double mx = smx[j & 1][0];
    int am = sarg[j & 1][0];
    for (int w = 1; w < nw; ++w) sp_merge(mx, am, smx[j & 1][w], sarg[j & 1][w]);
    if constexpr (kCluster) {
      cg::cluster_group cl = cg::this_cluster();
      if (tid == 0) {
        cmx[j & 1] = mx;
        carg[j & 1] = am;
      }
      cl.sync();  // barrier.cluster arrive (release) / wait (acquire): the C slots are visible
      mx = *cl.map_shared_rank(&cmx[j & 1], 0);
      am = *cl.map_shared_rank(&carg[j & 1], 0);
      for (int r = 1; r < C; ++r)
        sp_merge(mx, am, *cl.map_shared_rank(&cmx[j & 1], r), *cl.map_shared_rank(&carg[j & 1], r));
    }
    if (rank == 0 && tid == 0) arg[k.unit_base + j] = am;
    c = sp_sub(mx, penalty);
  }
  if constexpr (kCluster) cg::this_cluster().sync();
  if (rank == 0 && tid == 0) n_units[t] = nu;
}

// One CTA per track of the group: thread 0 walks the units back from the last unit's argmax (a set switch bit
// sends unit j - 1 to its own argmax), then sums u_j(o_j) forwards; every thread then gives its cues the offset
// of the unit holding their rasterised start frame, clamped into [0, S).
struct SplitCues {
  const double* start;
  const double* end;
  int sample_rate;
  double start_seconds;
};

// split_capped_backtrack_kernel's epilogue, the lines split_backtrack_kernel below runs inline (kept there as they
// were, so that kernel's code does not change).  The path uo[0 .. nu - 1] of a track: its segment count and the sum
// of u_j(uo[j]) (one thread)
__device__ __forceinline__ void split_path_score(const SplitTrack& k, int t, int nu, const int* uo, const uint2* q_all,
                                                 const SplitLevel* lvl, const int2* runs, int* n_segments,
                                                 double* split_score) {
  const int nr = runs[k.unit_base].y == 0 ? 0 : nu;  // a run is never empty: (0, 0) marks none
  const SpLevels l = sp_levels(k.level, lvl[k.vid].beta);
  const uint2* q = q_all + k.q_off;
  double score = 0.0;
  int seg = 1;
  for (int j = 0; j < nu; ++j) {
    SpUnit u;
    if (nr == 0) {
      u = SpUnit{0, 0, 0, k.S};
    } else {
      u.start = j == 0 ? 0 : runs[k.unit_base + j - 1].y;
      u.a = runs[k.unit_base + j].x;
      u.b = runs[k.unit_base + j].y;
      u.end = j == nu - 1 ? k.S : u.b;
    }
    if (j > 0 && uo[j] != uo[j - 1]) ++seg;
    score = sp_add(score, sp_unit_score(q, k.R, u, uo[j], l));
  }
  n_segments[t] = seg;
  split_score[t] = score;
}

// Every cue of the track (all threads of the CTA): the offset of the unit holding its rasterised start frame
__device__ __forceinline__ void split_cue_offsets(const SplitTrack& k, int nu, const int2* runs, const int* unit_off,
                                                  const SplitCues& cues, int* cue_offset) {
  for (long long i = k.c0 + threadIdx.x; i < k.c1; i += blockDim.x) {
    int off = 0;
    if (nu > 0) {
      long long first, last;
      b2_cue_bounds(cues.start[i], cues.end[i], k.ratio, cues.start_seconds, cues.sample_rate, k.S, first, last);
      const int f = (int)(first < 0 ? 0 : (first > k.S - 1 ? k.S - 1 : first));
      int lo = 0, hi = nu - 1;  // first unit whose run ends after f; the last unit when none does
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (runs[k.unit_base + mid].y > f) hi = mid;
        else lo = mid + 1;
      }
      off = unit_off[k.unit_base + lo];
    }
    cue_offset[i] = off;
  }
}

__global__ void __launch_bounds__(256) split_backtrack_kernel(const SplitTrack* __restrict__ trk, int t0,
                                                              const uint2* __restrict__ q_all,
                                                              const SplitLevel* __restrict__ lvl,
                                                              const uint32_t* __restrict__ dec,
                                                              const int* __restrict__ arg,
                                                              const int2* __restrict__ runs,
                                                              const int* __restrict__ n_units, int* unit_off,
                                                              SplitCues cues, int* __restrict__ cue_offset,
                                                              int* __restrict__ n_segments,
                                                              double* __restrict__ split_score) {
  __shared__ int s_nu;
  const int t = t0 + blockIdx.x;
  const SplitTrack k = trk[t];
  if (threadIdx.x == 0) {
    const int nu = n_units[t];
    s_nu = nu;
    if (nu <= 0) {
      n_segments[t] = nu;
      split_score[t] = NAN;
    } else {
      int* uo = unit_off + k.unit_base;
      int o = arg[k.unit_base + nu - 1];
      for (int j = nu - 1; j >= 0; --j) {
        uo[j] = o;
        if (j > 0) {
          const int m = o - k.o_lo;
          if ((dec[k.dec_base + (long long)j * k.nthr + (m >> 5)] >> (m & 31)) & 1u) o = arg[k.unit_base + j - 1];
        }
      }
      const int nr = runs[k.unit_base].y == 0 ? 0 : nu;  // a run is never empty: (0, 0) marks none
      const SpLevels l = sp_levels(k.level, lvl[k.vid].beta);
      const uint2* q = q_all + k.q_off;
      double score = 0.0;
      int seg = 1;
      for (int j = 0; j < nu; ++j) {
        SpUnit u;
        if (nr == 0) {
          u = SpUnit{0, 0, 0, k.S};
        } else {
          u.start = j == 0 ? 0 : runs[k.unit_base + j - 1].y;
          u.a = runs[k.unit_base + j].x;
          u.b = runs[k.unit_base + j].y;
          u.end = j == nu - 1 ? k.S : u.b;
        }
        if (j > 0 && uo[j] != uo[j - 1]) ++seg;
        score = sp_add(score, sp_unit_score(q, k.R, u, uo[j], l));
      }
      n_segments[t] = seg;
      split_score[t] = score;
    }
  }
  __syncthreads();
  const int nu = s_nu;
  for (long long i = k.c0 + threadIdx.x; i < k.c1; i += blockDim.x) {
    int off = 0;
    if (nu > 0) {
      long long first, last;
      b2_cue_bounds(cues.start[i], cues.end[i], k.ratio, cues.start_seconds, cues.sample_rate, k.S, first, last);
      const int f = (int)(first < 0 ? 0 : (first > k.S - 1 ? k.S - 1 : first));
      int lo = 0, hi = nu - 1;  // first unit whose run ends after f; the last unit when none does
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (runs[k.unit_base + mid].y > f) hi = mid;
        else lo = mid + 1;
      }
      off = unit_off[k.unit_base + lo];
    }
    cue_offset[i] = off;
  }
}

// b2_split_tracks_capped (at most N segments): one track per cluster of N x C CTAs, C = ceil(W / kCtaWindow) as for
// split_dp_kernel<true> (C = 1: CTAs of the bucket's widest track's threads).  CTA rank r runs layer kl = r / C (kl:
// the switches allowed so far) over window part p = r % C, part thread g = p * blockDim.x + tid owning the offsets
// o_lo + 32 g .. + 31 with the unchanged sp_thread_step.  Layer 0 never switches (c = -inf); layer kl >= 1 switches to
// c = M_{j-1,kl-1} - penalty.  Per unit j each CTA publishes its maximum in an alternating slot; after the cluster
// barrier it merges its own layer's C slots (the unit's argmax, which part 0 writes to arg[(unit_base + j) * N + kl])
// and layer kl - 1's C slots (its next c), each in rank order.  Switch words go to
// dec[dec_base + (j * N + kl) * nthr + g]; part 0 of layer kl writes the last unit's maximum to profile[t * N + kl].
//
// Barriers as split_dp_kernel<true>: the early exit depends on the track alone and comes before any barrier; then every
// CTA (past the window or in a layer the track cannot reach alike) runs the decode's barriers and, per unit, one
// __syncthreads and one cluster barrier, and one final cluster barrier.  A slot written at unit j + 2 was last read
// (by its own layer and the layer above) at unit j, before the barriers of unit j + 1.
__global__ void __launch_bounds__(kCtaThreads) split_capped_dp_kernel(const SplitTrack* __restrict__ trk,
                                                                      const int* __restrict__ order, int g0, int N,
                                                                      const uint2* __restrict__ q_all,
                                                                      const SplitLevel* __restrict__ lvl,
                                                                      const uint32_t* __restrict__ sub_bits,
                                                                      int max_runs, double penalty,
                                                                      uint32_t* __restrict__ dec,
                                                                      int* __restrict__ arg, int2* __restrict__ runs,
                                                                      int* __restrict__ n_units,
                                                                      double* __restrict__ profile) {
  extern __shared__ int rsm[];
  int* ra = rsm;
  int* rb = ra + max_runs;
  __shared__ int sh[33];
  __shared__ double smx[2][kCtaThreads / 32];
  __shared__ int sarg[2][kCtaThreads / 32];
  __shared__ double cmx[2];
  __shared__ int carg[2];
  cg::cluster_group cl = cg::this_cluster();
  const int NC = (int)cl.num_blocks(), rank = (int)cl.block_rank(), C = NC / N;
  const int layer = rank / C, part = rank - layer * C;
  const int t = order[g0 + (int)blockIdx.x / NC], tid = threadIdx.x, nw = blockDim.x >> 5;
  const SplitTrack k = trk[t];
  if (!k.live || lvl[k.vid].bad >= 0) {
    if (rank == 0 && tid < N) profile[(long long)t * N + tid] = NAN;  // N <= kMaxSegments <= 32 <= blockDim.x
    if (rank == 0 && tid == 0) n_units[t] = k.live ? -1 : 0;
    return;
  }
  const int n_end = runcorr::rc_decode_runs(sub_bits + k.bits_off, k.S, max_runs, ra, rb, sh);
  const int nr = min(n_end >> 1, max_runs);
  __syncthreads();
  if (rank == 0) {
    for (int r = tid; r < nr; r += blockDim.x) runs[k.unit_base + r] = make_int2(ra[r], rb[r]);
    if (nr == 0 && tid == 0) runs[k.unit_base] = make_int2(0, 0);  // no run: the one unit [0, S)
  }
  const int nu = nr > 0 ? nr : 1;
  const uint2* q = q_all + k.q_off;
  const SpLevels l = sp_levels(k.level, lvl[k.vid].beta);
  const int g = part * (int)blockDim.x + tid;
  const int o0 = k.o_lo + kOffsetsPerThread * g;
  const int n_mine = max(0, min(kOffsetsPerThread, k.W - kOffsetsPerThread * g));
  const int own = layer * C;  // the first rank of this layer (the layer below: own - C)
  double v[32];
  double c = -INFINITY;
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra, rb, nr, k.S, j);
    double best = -INFINITY;
    int barg = INT_MIN;
    uint32_t d = 0;
    if (n_mine > 0) d = sp_thread_step(q, k.R, u, o0, n_mine, j == 0, c, l, v, best, barg);
    if (j > 0 && g < k.nthr) dec[k.dec_base + ((long long)j * N + layer) * k.nthr + g] = d;
    for (int s = 16; s > 0; s >>= 1)
      sp_merge(best, barg, __shfl_xor_sync(0xffffffffu, best, s), __shfl_xor_sync(0xffffffffu, barg, s));
    if ((tid & 31) == 0) {
      smx[j & 1][tid >> 5] = best;
      sarg[j & 1][tid >> 5] = barg;
    }
    __syncthreads();
    double mx = smx[j & 1][0];
    int am = sarg[j & 1][0];
    for (int w = 1; w < nw; ++w) sp_merge(mx, am, smx[j & 1][w], sarg[j & 1][w]);
    if (tid == 0) {
      cmx[j & 1] = mx;
      carg[j & 1] = am;
    }
    cl.sync();  // barrier.cluster arrive (release) / wait (acquire): the N x C slots are visible
    if (part == 0 && tid == 0) {
      mx = *cl.map_shared_rank(&cmx[j & 1], own);
      am = *cl.map_shared_rank(&carg[j & 1], own);
      for (int r = 1; r < C; ++r)
        sp_merge(mx, am, *cl.map_shared_rank(&cmx[j & 1], own + r), *cl.map_shared_rank(&carg[j & 1], own + r));
      arg[(k.unit_base + j) * N + layer] = am;
      if (j == nu - 1) profile[(long long)t * N + layer] = mx;
    }
    if (layer > 0) {
      mx = *cl.map_shared_rank(&cmx[j & 1], own - C);
      am = *cl.map_shared_rank(&carg[j & 1], own - C);
      for (int r = 1; r < C; ++r)
        sp_merge(mx, am, *cl.map_shared_rank(&cmx[j & 1], own - C + r), *cl.map_shared_rank(&carg[j & 1], own - C + r));
      c = sp_sub(mx, penalty);
    }
  }
  cl.sync();
  if (rank == 0 && tid == 0) n_units[t] = nu;
}

// The capped path: thread 0 walks back from the top layer's last argmax, a set switch bit at (layer kl, unit j) sending
// unit j - 1 to layer kl - 1's argmax; the score and the cue offsets as split_backtrack_kernel.
__global__ void __launch_bounds__(256) split_capped_backtrack_kernel(const SplitTrack* __restrict__ trk, int t0, int N,
                                                                     const uint2* __restrict__ q_all,
                                                                     const SplitLevel* __restrict__ lvl,
                                                                     const uint32_t* __restrict__ dec,
                                                                     const int* __restrict__ arg,
                                                                     const int2* __restrict__ runs,
                                                                     const int* __restrict__ n_units, int* unit_off,
                                                                     SplitCues cues, int* __restrict__ cue_offset,
                                                                     int* __restrict__ n_segments,
                                                                     double* __restrict__ split_score) {
  __shared__ int s_nu;
  const int t = t0 + blockIdx.x;
  const SplitTrack k = trk[t];
  if (threadIdx.x == 0) {
    const int nu = n_units[t];
    s_nu = nu;
    if (nu <= 0) {
      n_segments[t] = nu;
      split_score[t] = NAN;
    } else {
      int* uo = unit_off + k.unit_base;
      int kl = N - 1;
      int o = arg[(k.unit_base + nu - 1) * N + kl];
      for (int j = nu - 1; j >= 0; --j) {
        uo[j] = o;
        if (j > 0 && kl > 0) {
          const int m = o - k.o_lo;
          if ((dec[k.dec_base + ((long long)j * N + kl) * k.nthr + (m >> 5)] >> (m & 31)) & 1u) {
            --kl;
            o = arg[(k.unit_base + j - 1) * N + kl];
          }
        }
      }
      split_path_score(k, t, nu, uo, q_all, lvl, runs, n_segments, split_score);
    }
  }
  __syncthreads();
  split_cue_offsets(k, s_nu, runs, unit_off, cues, cue_offset);
}

// b2_split_tracks_directed (offsets only grow, kDir = +1, or only shrink, kDir = -1, along the track): split_dp_kernel's
// layout, launch and barriers with sp_thread_step_dir.  The step of unit j needs, per thread, the maximum of V_{j-1}
// over the offsets before its own (kDir = -1: after them), so each unit ends with a cluster-wide exclusive scan of the
// thread maxima in offset order: a warp scan with shuffles, the warps' totals through alternating shared slots after
// the unit's __syncthreads (every thread takes the warps before its own), the CTAs' totals through alternating
// distributed-shared-memory slots after the unit's cluster barrier (rank r takes the ranks before it, kDir = -1 after
// it).  Per unit j >= 1 each thread writes its switch word to dec[dec_base + 2 j nthr + g] and its record word (the
// records of V_{j-1}) to dec[dec_base + (2 j + 1) nthr + g]; rank 0's thread 0 writes the last unit's argmax (the
// warps' and CTAs' maxima merged with sp_merge at that unit only) to arg[unit_base + nu - 1].  Barriers as
// split_dp_kernel: the early exit is the track's, then per unit one __syncthreads and one cluster barrier in every
// CTA, owning offsets or not, and one final cluster barrier.
template <int kDir, bool kCluster>
__global__ void __launch_bounds__(kCtaThreads) split_directed_dp_kernel(const SplitTrack* __restrict__ trk,
                                                                        const int* __restrict__ order, int g0,
                                                                        const uint2* __restrict__ q_all,
                                                                        const SplitLevel* __restrict__ lvl,
                                                                        const uint32_t* __restrict__ sub_bits,
                                                                        int max_runs, double penalty,
                                                                        uint32_t* __restrict__ dec,
                                                                        int* __restrict__ arg, int2* __restrict__ runs,
                                                                        int* __restrict__ n_units) {
  extern __shared__ int rsm[];
  int* ra = rsm;
  int* rb = ra + max_runs;
  __shared__ int sh[33];
  __shared__ double smx[2][kCtaThreads / 32];
  __shared__ int sarg[2][kCtaThreads / 32];
  __shared__ double cmx[2];
  __shared__ int carg[2];
  int C = 1, rank = 0;
  if constexpr (kCluster) {
    C = (int)cg::this_cluster().num_blocks();
    rank = (int)cg::this_cluster().block_rank();
  }
  const int t = order[g0 + (int)blockIdx.x / C], tid = threadIdx.x, nw = blockDim.x >> 5;
  const int lane = tid & 31, warp = tid >> 5;
  const SplitTrack k = trk[t];
  if (!k.live || lvl[k.vid].bad >= 0) {
    if (rank == 0 && tid == 0) n_units[t] = k.live ? -1 : 0;
    return;
  }
  const int n_end = runcorr::rc_decode_runs(sub_bits + k.bits_off, k.S, max_runs, ra, rb, sh);
  const int nr = min(n_end >> 1, max_runs);
  __syncthreads();
  if (rank == 0) {
    for (int r = tid; r < nr; r += blockDim.x) runs[k.unit_base + r] = make_int2(ra[r], rb[r]);
    if (nr == 0 && tid == 0) runs[k.unit_base] = make_int2(0, 0);  // no run: the one unit [0, S)
  }
  const int nu = nr > 0 ? nr : 1;
  const uint2* q = q_all + k.q_off;
  const SpLevels l = sp_levels(k.level, lvl[k.vid].beta);
  const int g = rank * (int)blockDim.x + tid;
  const int o0 = k.o_lo + kOffsetsPerThread * g;
  const int n_mine = max(0, min(kOffsetsPerThread, k.W - kOffsetsPerThread * g));
  double v[32];
  double p = -INFINITY;  // the maximum of V_{j-1} over the offsets on the kDir side behind this thread's
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra, rb, nr, k.S, j);
    double best = -INFINITY;
    int barg = INT_MIN;
    uint32_t d = 0, rec = 0;
    if (n_mine > 0) d = sp_thread_step_dir<kDir>(q, k.R, u, o0, n_mine, j == 0, p, penalty, l, v, best, barg, rec);
    if (j > 0 && g < k.nthr) {
      uint32_t* w = dec + k.dec_base + 2LL * j * k.nthr + g;
      w[0] = d;
      w[k.nthr] = rec;
    }
    // exclusive scan of the thread maxima in the direction's order: lanes ...
    double incl = best;
    for (int s = 1; s < 32; s <<= 1) {
      const double y = kDir > 0 ? __shfl_up_sync(0xffffffffu, incl, s) : __shfl_down_sync(0xffffffffu, incl, s);
      if (kDir > 0 ? lane >= s : lane + s < 32) incl = y > incl ? y : incl;
    }
    double ex = kDir > 0 ? __shfl_up_sync(0xffffffffu, incl, 1) : __shfl_down_sync(0xffffffffu, incl, 1);
    if (lane == (kDir > 0 ? 0 : 31)) ex = -INFINITY;
    const bool last = j == nu - 1;  // the same in every thread of the cluster
    if (last)
      for (int s = 16; s > 0; s >>= 1)
        sp_merge(best, barg, __shfl_xor_sync(0xffffffffu, best, s), __shfl_xor_sync(0xffffffffu, barg, s));
    if (lane == (kDir > 0 ? 31 : 0)) {  // the lane holding the warp's total (and, at the last unit, its argmax)
      smx[j & 1][warp] = incl;
      sarg[j & 1][warp] = barg;
    }
    __syncthreads();
    // ... the warps ...
    for (int w = kDir > 0 ? 0 : warp + 1; w < (kDir > 0 ? warp : nw); ++w) {
      const double x = smx[j & 1][w];
      ex = x > ex ? x : ex;
    }
    double mx = -INFINITY;
    int am = INT_MIN;
    if (tid == 0)
      for (int w = 0; w < nw; ++w) sp_merge(mx, am, smx[j & 1][w], sarg[j & 1][w]);
    // ... and the CTAs
    if constexpr (kCluster) {
      cg::cluster_group cl = cg::this_cluster();
      if (tid == 0) {
        cmx[j & 1] = mx;
        carg[j & 1] = am;
      }
      cl.sync();  // barrier.cluster arrive (release) / wait (acquire): the C slots are visible
      for (int r = kDir > 0 ? 0 : rank + 1; r < (kDir > 0 ? rank : C); ++r) {
        const double x = *cl.map_shared_rank(&cmx[j & 1], r);
        ex = x > ex ? x : ex;
      }
      if (last && rank == 0 && tid == 0)
        for (int r = 1; r < C; ++r)
          sp_merge(mx, am, *cl.map_shared_rank(&cmx[j & 1], r), *cl.map_shared_rank(&carg[j & 1], r));
    }
    if (last && rank == 0 && tid == 0) arg[k.unit_base + j] = am;
    p = ex;
  }
  if constexpr (kCluster) cg::this_cluster().sync();
  if (rank == 0 && tid == 0) n_units[t] = nu;
}

// The directed path: thread 0 walks back from the last unit's argmax; a set switch bit at (j, o) sends unit j - 1 to
// the nearest record of V_{j-1} behind o (dir = +1: the largest record below o, -1: the smallest above), which is the
// argmax of V_{j-1} over that side with ties to the largest offset.  The score and the cue offsets as
// split_backtrack_kernel.
__global__ void __launch_bounds__(256) split_directed_backtrack_kernel(const SplitTrack* __restrict__ trk, int t0,
                                                                       int dir, const uint2* __restrict__ q_all,
                                                                       const SplitLevel* __restrict__ lvl,
                                                                       const uint32_t* __restrict__ dec,
                                                                       const int* __restrict__ arg,
                                                                       const int2* __restrict__ runs,
                                                                       const int* __restrict__ n_units, int* unit_off,
                                                                       SplitCues cues, int* __restrict__ cue_offset,
                                                                       int* __restrict__ n_segments,
                                                                       double* __restrict__ split_score) {
  __shared__ int s_nu;
  const int t = t0 + blockIdx.x;
  const SplitTrack k = trk[t];
  if (threadIdx.x == 0) {
    const int nu = n_units[t];
    s_nu = nu;
    if (nu <= 0) {
      n_segments[t] = nu;
      split_score[t] = NAN;
    } else {
      int* uo = unit_off + k.unit_base;
      int m = arg[k.unit_base + nu - 1] - k.o_lo;
      for (int j = nu - 1; j >= 0; --j) {
        uo[j] = k.o_lo + m;
        if (j > 0) {
          const uint32_t* w = dec + k.dec_base + 2LL * j * k.nthr;
          if ((w[m >> 5] >> (m & 31)) & 1u) {  // a switch has a record behind it: the scans stop inside the window
            const uint32_t* rw = w + k.nthr;
            if (dir > 0) {
              int i = (m - 1) >> 5;
              uint32_t b = rw[i] & ((2u << ((m - 1) & 31)) - 1u);  // bits <= m - 1
              while (b == 0) b = rw[--i];
              m = 32 * i + 31 - __clz(b);
            } else {
              int i = (m + 1) >> 5;
              uint32_t b = rw[i] & ~((1u << ((m + 1) & 31)) - 1u);  // bits >= m + 1
              while (b == 0) b = rw[++i];
              m = 32 * i + __ffs(b) - 1;
            }
          }
        }
      }
      split_path_score(k, t, nu, uo, q_all, lvl, runs, n_segments, split_score);
    }
  }
  __syncthreads();
  split_cue_offsets(k, s_nu, runs, unit_off, cues, cue_offset);
}

// b2_split_tracks_breaks (breaks d_1 .. d_nb, nb + 1 <= kL = 32 / kM layers): the layers live inside the thread and the
// offsets are spread over the cluster.  Cluster thread g = rank * blockDim.x + tid owns the kM offsets o_lo + kM g ..
// and all layers' V for them in registers (kL x kM <= 32 doubles), so C = ceil(W / (kM kCtaThreads)); every launch is a
// cluster launch (C = 1: one CTA of the bucket's widest track's threads).  Per unit each thread runs
// sp_thread_step_breaks, then each layer m >= 1 needs the maximum of V_{j,m-1} over the offsets on the d_m side of its
// own for the next unit: per layer, an exclusive scan of the thread maxima in d_m's order, lanes by shuffles, the
// warps' totals through alternating shared slots after the unit's __syncthreads, the CTAs' totals through alternating
// distributed-shared-memory slots after the unit's cluster barrier.  Per unit j >= 1 each thread writes its switch word
// to dec[dec_base + 2 j nthr + g] and its record word to dec[dec_base + (2 j + 1) nthr + g] (bit m kM + i: layer m,
// offset i).  At the last unit each layer's maximum and its largest argmax (sp_merge over lanes, warps and CTAs) go to
// profile[t (nb + 1) + m] and arg[(unit_base + nu - 1)(nb + 1) + m].
//
// Barriers as split_dp_kernel<true>: the early exit depends on the track alone and comes before any barrier; then every
// CTA, owning offsets or not, runs the decode's barriers, per unit one __syncthreads and one cluster barrier, and one
// final cluster barrier.  A slot written at unit j + 2 was last read at unit j, before the barriers of unit j + 1.
template <int kM>
__global__ void __launch_bounds__(kCtaThreads) split_breaks_dp_kernel(const SplitTrack* __restrict__ trk,
                                                                      const int* __restrict__ order, int g0,
                                                                      const uint2* __restrict__ q_all,
                                                                      const SplitLevel* __restrict__ lvl,
                                                                      const uint32_t* __restrict__ sub_bits,
                                                                      int max_runs, double penalty, int nb, uint32_t up,
                                                                      uint32_t* __restrict__ dec,
                                                                      int* __restrict__ arg, int2* __restrict__ runs,
                                                                      int* __restrict__ n_units,
                                                                      double* __restrict__ profile) {
  constexpr int kL = 32 / kM, kW = kCtaThreads / 32;
  extern __shared__ int rsm[];
  int* ra = rsm;
  int* rb = ra + max_runs;
  __shared__ int sh[33];
  __shared__ double smx[2][kL][kW];  // the warps' scan totals per layer
  __shared__ double cmx[2][kL];      // the CTA's
  __shared__ double lmx[kL][kW];     // the last unit's maxima and argmaxes: the warps' ...
  __shared__ int larg[kL][kW];
  __shared__ double lcmx[kL];        // ... and the CTA's
  __shared__ int lcarg[kL];
  cg::cluster_group cl = cg::this_cluster();
  const int C = (int)cl.num_blocks(), rank = (int)cl.block_rank();
  const int t = order[g0 + (int)blockIdx.x / C], tid = threadIdx.x, nw = blockDim.x >> 5;
  const int lane = tid & 31, warp = tid >> 5, L = nb + 1;
  const SplitTrack k = trk[t];
  if (!k.live || lvl[k.vid].bad >= 0) {
    if (rank == 0 && tid < L) profile[(long long)t * L + tid] = NAN;  // L <= 16 <= blockDim.x
    if (rank == 0 && tid == 0) n_units[t] = k.live ? -1 : 0;
    return;
  }
  const int n_end = runcorr::rc_decode_runs(sub_bits + k.bits_off, k.S, max_runs, ra, rb, sh);
  const int nr = min(n_end >> 1, max_runs);
  __syncthreads();
  if (rank == 0) {
    for (int r = tid; r < nr; r += blockDim.x) runs[k.unit_base + r] = make_int2(ra[r], rb[r]);
    if (nr == 0 && tid == 0) runs[k.unit_base] = make_int2(0, 0);  // no run: the one unit [0, S)
  }
  const int nu = nr > 0 ? nr : 1;
  const uint2* q = q_all + k.q_off;
  const SpLevels l = sp_levels(k.level, lvl[k.vid].beta);
  const int g = rank * (int)blockDim.x + tid;
  const int o0 = k.o_lo + kM * g;
  const int n_mine = max(0, min(kM, k.W - kM * g));
  double v[kL][kM];
  double p[kL];
#pragma unroll
  for (int m = 0; m < kL; ++m) {
    p[m] = -INFINITY;
#pragma unroll
    for (int i = 0; i < kM; ++i) v[m][i] = -INFINITY;
  }
  for (int j = 0; j < nu; ++j) {
    const SpUnit u = sp_unit(ra, rb, nr, k.S, j);
    uint32_t d = 0, rec = 0;
    if (n_mine > 0) sp_thread_step_breaks<kL, kM>(q, k.R, u, o0, n_mine, j == 0, nb, up, p, penalty, l, v, d, rec);
    if (j > 0 && g < k.nthr) {
      uint32_t* w = dec + k.dec_base + 2LL * j * k.nthr + g;
      w[0] = d;
      w[k.nthr] = rec;
    }
    // per layer m >= 1: the exclusive scan of the thread maxima of layer m - 1 in d_m's order, lanes ...
#pragma unroll
    for (int m = 1; m < kL; ++m) {
      if (m > nb) continue;
      const bool fwd = (up >> m) & 1u;
      double incl = v[m - 1][0];
#pragma unroll
      for (int i = 1; i < kM; ++i) incl = v[m - 1][i] > incl ? v[m - 1][i] : incl;
      for (int s = 1; s < 32; s <<= 1) {
        const double y = __shfl_sync(0xffffffffu, incl, fwd ? lane - s : lane + s);
        if (fwd ? lane >= s : lane + s < 32) incl = y > incl ? y : incl;
      }
      const double ex = __shfl_sync(0xffffffffu, incl, fwd ? lane - 1 : lane + 1);
      p[m] = lane == (fwd ? 0 : 31) ? -INFINITY : ex;
      if (lane == (fwd ? 31 : 0)) smx[j & 1][m][warp] = incl;  // the lane holding the warp's total
    }
    const bool last = j == nu - 1;  // the same in every thread of the cluster
    if (last) {
#pragma unroll
      for (int m = 0; m < kL; ++m) {
        if (m > nb) continue;
        double best = -INFINITY;
        int barg = INT_MIN;
#pragma unroll
        for (int i = 0; i < kM; ++i)
          if (i < n_mine && v[m][i] >= best) {  // increasing offsets: ties go to the largest
            best = v[m][i];
            barg = o0 + i;
          }
        for (int s = 16; s > 0; s >>= 1)
          sp_merge(best, barg, __shfl_xor_sync(0xffffffffu, best, s), __shfl_xor_sync(0xffffffffu, barg, s));
        if (lane == 0) {
          lmx[m][warp] = best;
          larg[m][warp] = barg;
        }
      }
    }
    __syncthreads();
    // ... the warps ...
#pragma unroll
    for (int m = 1; m < kL; ++m) {
      if (m > nb) continue;
      const bool fwd = (up >> m) & 1u;
      double ex = p[m];
      for (int w = fwd ? 0 : warp + 1; w < (fwd ? warp : nw); ++w) {
        const double x = smx[j & 1][m][w];
        ex = x > ex ? x : ex;
      }
      p[m] = ex;
    }
    if (tid < L) {  // thread m: layer m's CTA scan total (m >= 1; at the last unit also its maximum and argmax)
      if (tid > 0) {
        double mx = -INFINITY;
        for (int w = 0; w < nw; ++w) mx = smx[j & 1][tid][w] > mx ? smx[j & 1][tid][w] : mx;
        cmx[j & 1][tid] = mx;
      }
      if (last) {
        double lm = -INFINITY;
        int la = INT_MIN;
        for (int w = 0; w < nw; ++w) sp_merge(lm, la, lmx[tid][w], larg[tid][w]);
        lcmx[tid] = lm;
        lcarg[tid] = la;
      }
    }
    cl.sync();  // barrier.cluster arrive (release) / wait (acquire): the C slots are visible
    // ... and the CTAs
#pragma unroll
    for (int m = 1; m < kL; ++m) {
      if (m > nb) continue;
      const bool fwd = (up >> m) & 1u;
      double ex = p[m];
      for (int r = fwd ? 0 : rank + 1; r < (fwd ? rank : C); ++r) {
        const double x = *cl.map_shared_rank(&cmx[j & 1][m], r);
        ex = x > ex ? x : ex;
      }
      p[m] = ex;
    }
    if (last && rank == 0 && tid < L) {
      double lm = lcmx[tid];
      int la = lcarg[tid];
      for (int r = 1; r < C; ++r) sp_merge(lm, la, *cl.map_shared_rank(&lcmx[tid], r), *cl.map_shared_rank(&lcarg[tid], r));
      profile[(long long)t * L + tid] = lm;
      arg[(k.unit_base + j) * L + tid] = la;
    }
  }
  cl.sync();
  if (rank == 0 && tid == 0) n_units[t] = nu;
}

// The path along stated breaks: thread 0 starts at the overall maximum of the last unit over (layer, offset), ties to
// the largest offset and then the smallest layer; a set switch bit at (j, m, o) sends unit j - 1 to layer m - 1 at the
// nearest record of V_{j-1,m-1} on the d_m side of o (up: bit m set when d_m = +1), which is the argmax of V_{j-1,m-1}
// over that side with ties to the largest offset.  The score and the cue offsets as split_backtrack_kernel.
__global__ void __launch_bounds__(256) split_breaks_backtrack_kernel(const SplitTrack* __restrict__ trk, int t0, int nb,
                                                                     uint32_t up, int kM,
                                                                     const uint2* __restrict__ q_all,
                                                                     const SplitLevel* __restrict__ lvl,
                                                                     const uint32_t* __restrict__ dec,
                                                                     const int* __restrict__ arg,
                                                                     const double* __restrict__ profile,
                                                                     const int2* __restrict__ runs,
                                                                     const int* __restrict__ n_units, int* unit_off,
                                                                     SplitCues cues, int* __restrict__ cue_offset,
                                                                     int* __restrict__ n_segments,
                                                                     double* __restrict__ split_score) {
  __shared__ int s_nu;
  const int t = t0 + blockIdx.x;
  const SplitTrack k = trk[t];
  if (threadIdx.x == 0) {
    const int nu = n_units[t];
    s_nu = nu;
    if (nu <= 0) {
      n_segments[t] = nu;
      split_score[t] = NAN;
    } else {
      const int L = nb + 1;
      const int* a = arg + (k.unit_base + nu - 1) * L;
      const double* pr = profile + (long long)t * L;
      int ml = 0;  // the end: the largest maximum, then the largest offset, then the smallest layer
      for (int m = 1; m < L; ++m)
        if (pr[m] > pr[ml] || (pr[m] == pr[ml] && a[m] > a[ml])) ml = m;
      int* uo = unit_off + k.unit_base;
      int x = a[ml] - k.o_lo;  // window index of the offset
      const uint32_t mask = (1u << kM) - 1u;  // kM <= 16
      for (int j = nu - 1; j >= 0; --j) {
        uo[j] = k.o_lo + x;
        if (j > 0 && ml > 0) {
          const uint32_t* w = dec + k.dec_base + 2LL * j * k.nthr;
          const int sh = ml * kM;
          if ((w[x / kM] >> (sh + x % kM)) & 1u) {  // a switch has a record behind it: the scans stop in the window
            const uint32_t* rw = w + k.nthr;
            if ((up >> ml) & 1u) {
              int i = (x - 1) / kM;
              uint32_t b = (rw[i] >> sh) & mask & ((2u << ((x - 1) % kM)) - 1u);  // bits <= x - 1
              while (b == 0) b = (rw[--i] >> sh) & mask;
              x = kM * i + 31 - __clz(b);
            } else {
              int i = (x + 1) / kM;
              uint32_t b = (rw[i] >> sh) & mask & ~((1u << ((x + 1) % kM)) - 1u);  // bits >= x + 1
              while (b == 0) b = (rw[++i] >> sh) & mask;
              x = kM * i + __ffs(b) - 1;
            }
            --ml;
          }
        }
      }
      split_path_score(k, t, nu, uo, q_all, lvl, runs, n_segments, split_score);
    }
  }
  __syncthreads();
  split_cue_offsets(k, s_nu, runs, unit_off, cues, cue_offset);
}

// The widest cluster (CTAs, from kMaxCluster down) of kernel at kCtaThreads threads and the largest run table that
// the device co-schedules, into *out.
template <typename Kernel>
int split_query_cluster(b2_ctx* h, Kernel kernel, const char* name, int* out) {
  const size_t smem = (size_t)2 * kMaxRuns * sizeof(int);
  B2_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  for (int C = kMaxCluster; C >= 1; --C) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)C);
    cfg.blockDim = dim3((unsigned)kCtaThreads);
    cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = (unsigned)C;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    int n = 0;
    const cudaError_t e = cudaOccupancyMaxActiveClusters(&n, kernel, &cfg);
    if (e == cudaSuccess && n > 0) {
      *out = C;
      return B2_OK;
    }
    (void)cudaGetLastError();  // a size the device refuses is an answer, not an error
  }
  B2_FAIL(h, B2_ERR_CUDA, "split: the device co-schedules no cluster of %s", name);
}

}  // namespace

// The widest clusters of split_dp_kernel and of split_capped_dp_kernel (each queried for its own kernel) that the
// device co-schedules; once per handle.
int b2i_split_max_cluster(b2_ctx* h) {
  if (h->split_max_cluster > 0) return B2_OK;
  return split_query_cluster(h, split_dp_kernel<true>, "split_dp_kernel", &h->split_max_cluster);
}

int b2i_split_capped_max_cluster(b2_ctx* h) {
  if (h->split_capped_max_cluster > 0) return B2_OK;
  return split_query_cluster(h, split_capped_dp_kernel, "split_capped_dp_kernel", &h->split_capped_max_cluster);
}

// split_directed_dp_kernel's widest cluster: the narrower of its two directions' (the same code but for the order of
// the walk and the scan).
int b2i_split_directed_max_cluster(b2_ctx* h) {
  if (h->split_directed_max_cluster > 0) return B2_OK;
  int up = 0, down = 0;
  B2_TRY(split_query_cluster(h, split_directed_dp_kernel<1, true>, "split_directed_dp_kernel<1>", &up));
  B2_TRY(split_query_cluster(h, split_directed_dp_kernel<-1, true>, "split_directed_dp_kernel<-1>", &down));
  h->split_directed_max_cluster = std::min(up, down);
  return B2_OK;
}

// split_breaks_dp_kernel's offsets per thread for nb breaks: the most that leave room for nb + 1 layers of them in 32
// registers' worth of doubles (8 instantiations), and the index of that instantiation
static int split_breaks_offsets(int nb) { return 32 / (nb + 1); }
static int split_breaks_shape(int kM) {
  return kM >= 16 ? 0 : kM >= 10 ? 1 : kM >= 8 ? 2 : kM >= 6 ? 3 : kM >= 5 ? 4 : kM >= 4 ? 5 : kM >= 3 ? 6 : 7;
}

// The widest cluster of split_breaks_dp_kernel<kM> (each instantiation queried for itself); once per handle and kM.
int b2i_split_breaks_max_cluster(b2_ctx* h, int kM) {
  int* out = &h->split_breaks_max_cluster[split_breaks_shape(kM)];
  if (*out > 0) return B2_OK;
  switch (kM) {
    case 16: return split_query_cluster(h, split_breaks_dp_kernel<16>, "split_breaks_dp_kernel<16>", out);
    case 10: return split_query_cluster(h, split_breaks_dp_kernel<10>, "split_breaks_dp_kernel<10>", out);
    case 8: return split_query_cluster(h, split_breaks_dp_kernel<8>, "split_breaks_dp_kernel<8>", out);
    case 6: return split_query_cluster(h, split_breaks_dp_kernel<6>, "split_breaks_dp_kernel<6>", out);
    case 5: return split_query_cluster(h, split_breaks_dp_kernel<5>, "split_breaks_dp_kernel<5>", out);
    case 4: return split_query_cluster(h, split_breaks_dp_kernel<4>, "split_breaks_dp_kernel<4>", out);
    case 3: return split_query_cluster(h, split_breaks_dp_kernel<3>, "split_breaks_dp_kernel<3>", out);
    default: return split_query_cluster(h, split_breaks_dp_kernel<2>, "split_breaks_dp_kernel<2>", out);
  }
}

int b2i_split_launch(b2_ctx* h, const void* d_ref, bool ref_f64, const int64_t* ref_off, int V,
                     const int32_t* track_video, int T, const double* cue_start, const double* cue_end,
                     const uint8_t* cue_keep, const int64_t* cue_off, const double* ratio, const int64_t* len,
                     int sample_rate, double start_seconds, int64_t max_offset_samples, double penalty,
                     bool refuse_three_levels, const void* h_ref, bool h_ref_f64, bool wide, int* d_cue_offset,
                     int* d_n_segments, double* d_split_score, int max_segments, double* d_profile, int direction,
                     const int32_t* breaks, int n_breaks) {
  B2Range range("b2:split (split_ref, raster_bits, split_dp, split_backtrack)");
  if (T <= 0) return B2_OK;
  // the envelope: b2_split_tracks up to kMaxWindow offsets (clusters of 1 or 2 CTAs), b2_split_tracks_wide up to
  // the widest cluster of kCtaThreads-thread CTAs this device co-schedules, b2_split_tracks_capped up to N x C CTAs
  // of the widest cluster of split_capped_dp_kernel, b2_split_tracks_directed up to the widest cluster of
  // split_directed_dp_kernel, b2_split_tracks_breaks up to the widest cluster of split_breaks_dp_kernel<kM> of
  // kCtaThreads x kM offsets a CTA
  const bool capped = max_segments > 0, broken = n_breaks > 0;
  const int N = capped ? max_segments : broken ? n_breaks + 1 : 1;
  const int per_thread = broken ? split_breaks_offsets(n_breaks) : kOffsetsPerThread;  // offsets a thread owns
  const int cta_window = kCtaThreads * per_thread;
  uint32_t up = 0;  // bit m: d_m = +1
  for (int m = 1; m <= n_breaks; ++m) up |= (uint32_t)(breaks[m - 1] > 0) << m;
  long long max_window = kMaxWindow;
  if (broken) {
    if (n_breaks > kMaxBreaks)
      B2_FAIL(h, B2_ERR_UNSUPPORTED, "split: %d breaks is more than %d", n_breaks, kMaxBreaks);
    B2_TRY(b2i_split_breaks_max_cluster(h, per_thread));
    max_window = (long long)cta_window * h->split_breaks_max_cluster[split_breaks_shape(per_thread)];
  } else if (capped) {
    if (N > kMaxSegments) B2_FAIL(h, B2_ERR_UNSUPPORTED, "split: max_segments %d is more than %d", N, kMaxSegments);
    B2_TRY(b2i_split_capped_max_cluster(h));
    max_window = (long long)kCtaWindow * (h->split_capped_max_cluster / N);
  } else if (direction != 0) {
    B2_TRY(b2i_split_directed_max_cluster(h));
    max_window = (long long)kCtaWindow * h->split_directed_max_cluster;
  } else if (wide) {
    B2_TRY(b2i_split_max_cluster(h));
    max_window = (long long)kCtaWindow * h->split_max_cluster;
  }
  // ---- plan: videos, windows, workspace ----
  std::vector<int> vid_of(V, -1);
  std::vector<SplitVideo> vids;
  std::vector<SplitTrack> trk(T);
  std::vector<double> d_ratio_h(T, 1.0);
  std::vector<long long> len_h(T, 0), unit_bound(T, 0);
  long long q_total = 0, sig_words = 1, units = 0, max_cues = 0;
  int max_runs = 1;
  const long long c_base = cue_off[0];
  for (int t = 0; t < T; ++t) {
    SplitTrack& k = trk[t];
    memset(&k, 0, sizeof(k));
    k.c0 = cue_off[t] - c_base;
    k.c1 = cue_off[t + 1] - c_base;
    max_cues = std::max(max_cues, k.c1 - k.c0);
    const int v = track_video[t];
    const long long R = ref_off[v + 1] - ref_off[v];
    if (std::isnan(ratio[t]) || R == 0) continue;  // skipped; an empty reference has no alignment
    const B2JobPlan p = b2_plan_job(R, len[t], max_offset_samples, h->log2_quirk_mask);
    if (p.kind != 0) continue;  // no offset survives the mask
    const long long W = p.o_hi - p.o_lo + 1;
    if (W > max_window) {
      if (broken)
        B2_FAIL(h, B2_ERR_UNSUPPORTED,
                "split: track %d: a window of %lld offsets is wider than %lld, the widest at %d breaks (a cluster of %lld "
                "CTAs of %d offsets, %d offsets a thread; the widest cluster of this kernel the device "
                "co-schedules)", t, W, max_window, n_breaks, max_window / cta_window, cta_window, per_thread);
      if (capped)
        B2_FAIL(h, B2_ERR_UNSUPPORTED,
                "split: track %d: a window of %lld offsets is wider than %lld at %d segments (%d segments x %lld CTAs of "
                "%d offsets; %d CTAs make the widest cluster this device co-schedules)", t, W, max_window, N, N,
                (long long)ceil_div64(W, kCtaWindow), kCtaWindow, h->split_capped_max_cluster);
      if (direction != 0)
        B2_FAIL(h, B2_ERR_UNSUPPORTED,
                "split: track %d: a window of %lld offsets is wider than %lld (a cluster of %d CTAs of %d offsets, "
                "the widest of the directed split this device co-schedules)", t, W, max_window,
                h->split_directed_max_cluster, kCtaWindow);
      if (wide)
        B2_FAIL(h, B2_ERR_UNSUPPORTED,
                "split: track %d: a window of %lld offsets is wider than %lld (a cluster of %d CTAs of %d offsets, "
                "the widest this device co-schedules)", t, W, max_window, h->split_max_cluster, kCtaWindow);
      B2_FAIL(h, B2_ERR_UNSUPPORTED,
              "split: track %d: a window of %lld offsets is wider than %d (b2_split_tracks_wide takes wider ones)", t,
              W, kMaxWindow);
    }
    long long kept = 0;
    for (long long c = cue_off[t]; c < cue_off[t + 1]; ++c) kept += cue_keep ? (cue_keep[c] != 0) : 1;
    if (kept > kMaxRuns)
      B2_FAIL(h, B2_ERR_UNSUPPORTED, "split: track %d: %lld kept cues may make more than %d runs", t, kept, kMaxRuns);
    if (vid_of[v] < 0) {
      vid_of[v] = (int)vids.size();
      vids.push_back(SplitVideo{(long long)ref_off[v], q_total, (int)R});
      q_total += runcorr::rc_ref_entries((int)R);
    }
    k.live = 1;
    k.vid = vid_of[v];
    k.q_off = vids[k.vid].q_off;
    k.R = (int)R;
    k.S = (int)len[t];
    k.o_lo = (int)p.o_lo;
    k.W = (int)W;
    k.nthr = (int)ceil_div64(W, per_thread);
    k.ratio = ratio[t];
    k.level = (float)std::min(1.0 / ratio[t], 1.0);
    k.unit_base = units;
    unit_bound[t] = std::max<long long>(kept, 1);
    units += unit_bound[t];
    max_runs = std::max<int>(max_runs, (int)kept);
    sig_words = std::max<long long>(sig_words, (len[t] >> 5) + 2);
    d_ratio_h[t] = ratio[t];
    len_h[t] = len[t];
  }
  for (int t = 0; t < T; ++t) trk[t].bits_off = (long long)t * sig_words;
  // track groups: the switch words of a group stay within kDecBudget words; within a group the tracks are launched
  // by cluster size C (cluster size is per launch), order[] listing each group's tracks by C.  Capped: N layers of
  // switch words per unit; directed: a switch word and a record word per unit; breaks: a switch word and a record
  // word per unit, each holding all layers' bits of the thread's 32 / (n + 1) offsets.
  const long long kDecBudget = 64LL << 20;
  const int words = capped ? N : (direction != 0 || broken) ? 2 : 1;
  std::vector<int> group_first{0};
  long long dec_max = 1, dec_at = 0;
  std::vector<int> ncta(T, 1), order(T);
  for (int t = 0; t < T; ++t) {
    SplitTrack& k = trk[t];
    const long long need = k.live ? unit_bound[t] * k.nthr * words : 0;
    if (dec_at > 0 && dec_at + need > kDecBudget) {
      group_first.push_back(t);
      dec_at = 0;
    }
    k.dec_base = dec_at;
    dec_at += need;
    dec_max = std::max(dec_max, dec_at);
    if (k.live) ncta[t] = (int)ceil_div64(k.W, cta_window);
    order[t] = t;
  }
  group_first.push_back(T);
  for (size_t g = 0; g + 1 < group_first.size(); ++g)
    std::stable_sort(order.begin() + group_first[g], order.begin() + group_first[g + 1],
                     [&](int a, int b) { return ncta[a] < ncta[b]; });

  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at = (at + bytes + 255) & ~size_t(255); return o; };
  const size_t nv = std::max<size_t>(vids.size(), 1), nunits = (size_t)std::max<long long>(units, 1);
  const size_t o_q = take((size_t)std::max<long long>(q_total, 1) * 8), o_lvl = take(nv * sizeof(SplitLevel)),
               o_bits = take((size_t)T * sig_words * 4), o_runs = take(nunits * 8), o_arg = take(nunits * N * 4),
               o_uo = take(nunits * 4), o_nu = take((size_t)T * 4), o_dec = take((size_t)dec_max * 4);
  void* d_ws;
  B2_TRY(b2i_ws(h, b2_ctx::WS_SPLIT, at + 256, &d_ws));
  char* base = (char*)d_ws;
  uint2* q = (uint2*)(base + o_q);
  SplitLevel* lvl = (SplitLevel*)(base + o_lvl);
  uint32_t* bits = (uint32_t*)(base + o_bits);
  int2* runs = (int2*)(base + o_runs);
  int* arg = (int*)(base + o_arg);
  int* uo = (int*)(base + o_uo);
  int* nu = (int*)(base + o_nu);
  uint32_t* dec = (uint32_t*)(base + o_dec);

  const long long nc = cue_off[T] - c_base;
  std::vector<long long> cue_rel(T + 1);
  for (int t = 0; t <= T; ++t) cue_rel[t] = cue_off[t] - c_base;
  MetaArena a;
  B2_TRY(b2i_meta_begin(h, &a, (size_t)nc * 17 + (size_t)(T + 1) * 8 + (size_t)T * (sizeof(SplitTrack) + 16) +
                                   vids.size() * sizeof(SplitVideo) + (size_t)T * 4 + 1024));
  B2CueDev cd;
  cd.start = (const double*)b2i_meta_put(&a, cue_start + c_base, (size_t)nc * 8);
  cd.end = (const double*)b2i_meta_put(&a, cue_end + c_base, (size_t)nc * 8);
  cd.keep = cue_keep ? (const uint8_t*)b2i_meta_put(&a, cue_keep + c_base, (size_t)nc) : nullptr;
  cd.cue_off = (const long long*)b2i_meta_put(&a, cue_rel.data(), (size_t)(T + 1) * 8);
  cd.sample_rate = sample_rate;
  cd.start_seconds = start_seconds;
  const SplitTrack* d_trk = (const SplitTrack*)b2i_meta_put(&a, trk.data(), (size_t)T * sizeof(SplitTrack));
  const double* d_ratio = (const double*)b2i_meta_put(&a, d_ratio_h.data(), (size_t)T * 8);
  const long long* d_len = (const long long*)b2i_meta_put(&a, len_h.data(), (size_t)T * 8);
  const int* d_order = (const int*)b2i_meta_put(&a, order.data(), (size_t)T * 4);
  const SplitVideo* d_vids =
      vids.empty() ? nullptr : (const SplitVideo*)b2i_meta_put(&a, vids.data(), vids.size() * sizeof(SplitVideo));
  B2_TRY(b2i_meta_commit(&a));

  if (!vids.empty()) {
    if (ref_f64)
      split_ref_kernel<double><<<(unsigned)vids.size(), 1024, 0, h->stream>>>((const double*)d_ref, d_vids, q, lvl);
    else
      split_ref_kernel<float><<<(unsigned)vids.size(), 1024, 0, h->stream>>>((const float*)d_ref, d_vids, q, lvl);
    B2_CHECK_LAUNCH(h, "split_ref_kernel");
    if (refuse_three_levels) {  // B2_HOST: a third level refuses the call before anything else runs
      std::vector<SplitLevel> lv(vids.size());
      B2_CUDA(h, cudaMemcpyAsync(lv.data(), lvl, vids.size() * sizeof(SplitLevel), cudaMemcpyDeviceToHost, h->stream));
      B2_CUDA(h, cudaStreamSynchronize(h->stream));
      for (int v = 0; v < V; ++v) {
        if (vid_of[v] < 0 || lv[vid_of[v]].bad < 0) continue;
        const long long f = lv[vid_of[v]].bad;
        B2_FAIL(h, B2_ERR_UNSUPPORTED,
                "split: video %d: frame %lld holds %g, a level other than 1.0 and %g (the reference must have two "
                "finite levels)", v, f, !h_ref ? NAN : h_ref_f64 ? ((const double*)h_ref)[ref_off[v] + f] : (double)((const float*)h_ref)[ref_off[v] + f], lv[vid_of[v]].beta);
      }
    }
  }
  B2_TRY(b2i_raster_bits_dev_launch(h, cd, T, max_cues, d_ratio, d_len, sig_words, bits));
  const size_t smem = (size_t)2 * max_runs * sizeof(int);
  B2_CUDA(h, cudaFuncSetAttribute(split_dp_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2_CUDA(h, cudaFuncSetAttribute(split_dp_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  B2_CUDA(h, cudaFuncSetAttribute(split_dp_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  const SplitCues sc{cd.start, cd.end, sample_rate, start_seconds};
  if (broken) {
    // cluster launches of split_breaks_dp_kernel<KM> by cluster size (C = 1: the bucket's widest track's threads)
    auto run = [&](auto offsets) -> int {
      constexpr int KM = decltype(offsets)::value;
      B2_CUDA(h, cudaFuncSetAttribute(split_breaks_dp_kernel<KM>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
      B2_CUDA(h, cudaFuncSetAttribute(split_breaks_dp_kernel<KM>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      for (size_t g = 0; g + 1 < group_first.size(); ++g) {
        const int g0 = group_first[g], n = group_first[g + 1] - g0;
        if (n <= 0) continue;
        for (int i = g0; i < g0 + n;) {
          const int C = ncta[order[i]];
          int e = i;
          while (e < g0 + n && ncta[order[e]] == C) ++e;
          int thr = kCtaThreads;
          if (C == 1) {
            thr = 32;
            for (int x = i; x < e; ++x) thr = std::max<int>(thr, (int)(32 * ceil_div64(trk[order[x]].nthr, 32)));
          }
          cudaLaunchConfig_t cfg = {};
          cfg.gridDim = dim3((unsigned)((e - i) * C));
          cfg.blockDim = dim3((unsigned)thr);
          cfg.dynamicSmemBytes = smem;
          cfg.stream = h->stream;
          cudaLaunchAttribute at[1];
          at[0].id = cudaLaunchAttributeClusterDimension;
          at[0].val.clusterDim.x = (unsigned)C;
          at[0].val.clusterDim.y = 1;
          at[0].val.clusterDim.z = 1;
          cfg.attrs = at;
          cfg.numAttrs = 1;
          B2_CUDA(h, cudaLaunchKernelEx(&cfg, split_breaks_dp_kernel<KM>, d_trk, (const int*)d_order, i,
                                        (const uint2*)q, (const SplitLevel*)lvl, (const uint32_t*)bits, max_runs,
                                        penalty, n_breaks, up, dec, arg, runs, nu, d_profile));
          B2_CHECK_LAUNCH(h, "split_breaks_dp_kernel");
          i = e;
        }
        split_breaks_backtrack_kernel<<<(unsigned)n, 256, 0, h->stream>>>(
            d_trk, g0, n_breaks, up, KM, q, lvl, dec, arg, d_profile, runs, nu, uo, sc, d_cue_offset + c_base,
            d_n_segments, d_split_score);
        B2_CHECK_LAUNCH(h, "split_breaks_backtrack_kernel");
      }
      return B2_OK;
    };
    switch (per_thread) {
      case 16: return run(std::integral_constant<int, 16>{});
      case 10: return run(std::integral_constant<int, 10>{});
      case 8: return run(std::integral_constant<int, 8>{});
      case 6: return run(std::integral_constant<int, 6>{});
      case 5: return run(std::integral_constant<int, 5>{});
      case 4: return run(std::integral_constant<int, 4>{});
      case 3: return run(std::integral_constant<int, 3>{});
      default: return run(std::integral_constant<int, 2>{});
    }
  }
  if (capped) {
    B2_CUDA(h, cudaFuncSetAttribute(split_capped_dp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    B2_CUDA(h, cudaFuncSetAttribute(split_capped_dp_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    for (size_t g = 0; g + 1 < group_first.size(); ++g) {
      const int g0 = group_first[g], n = group_first[g + 1] - g0;
      if (n <= 0) continue;
      for (int i = g0; i < g0 + n;) {
        const int C = ncta[order[i]];
        int e = i;
        while (e < g0 + n && ncta[order[e]] == C) ++e;
        int thr = kCtaThreads;  // C = 1: CTAs of the bucket's widest track's threads
        if (C == 1) {
          thr = 32;
          for (int x = i; x < e; ++x) thr = std::max<int>(thr, (int)(32 * ceil_div64(trk[order[x]].nthr, 32)));
        }
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)((e - i) * N * C));
        cfg.blockDim = dim3((unsigned)thr);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = h->stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)(N * C);
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        B2_CUDA(h, cudaLaunchKernelEx(&cfg, split_capped_dp_kernel, d_trk, (const int*)d_order, i, N, (const uint2*)q,
                                      (const SplitLevel*)lvl, (const uint32_t*)bits, max_runs, penalty, dec, arg, runs,
                                      nu, d_profile));
        B2_CHECK_LAUNCH(h, "split_capped_dp_kernel");
        i = e;
      }
      split_capped_backtrack_kernel<<<(unsigned)n, 256, 0, h->stream>>>(
          d_trk, g0, N, q, lvl, dec, arg, runs, nu, uo, sc, d_cue_offset + c_base, d_n_segments, d_split_score);
      B2_CHECK_LAUNCH(h, "split_capped_backtrack_kernel");
    }
    return B2_OK;
  }
  if (direction != 0) {
    // the launches of split_dp_kernel below with the directed kernel of direction D
    auto run = [&](auto dir) -> int {
      constexpr int D = decltype(dir)::value;
      B2_CUDA(h, cudaFuncSetAttribute(split_directed_dp_kernel<D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
      B2_CUDA(h, cudaFuncSetAttribute(split_directed_dp_kernel<D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
      B2_CUDA(h, cudaFuncSetAttribute(split_directed_dp_kernel<D, true>,
                                      cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
      for (size_t g = 0; g + 1 < group_first.size(); ++g) {
        const int g0 = group_first[g], n = group_first[g + 1] - g0;
        if (n <= 0) continue;
        for (int i = g0; i < g0 + n;) {
          const int C = ncta[order[i]];
          int e = i;
          while (e < g0 + n && ncta[order[e]] == C) ++e;
          if (C == 1) {  // one CTA of the bucket's widest track's threads
            int thr = 32;
            for (int x = i; x < e; ++x) thr = std::max<int>(thr, (int)(32 * ceil_div64(trk[order[x]].nthr, 32)));
            split_directed_dp_kernel<D, false><<<(unsigned)(e - i), (unsigned)thr, smem, h->stream>>>(
                d_trk, d_order, i, q, lvl, bits, max_runs, penalty, dec, arg, runs, nu);
          } else {
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)((e - i) * C));
            cfg.blockDim = dim3((unsigned)kCtaThreads);
            cfg.dynamicSmemBytes = smem;
            cfg.stream = h->stream;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = (unsigned)C;
            at[0].val.clusterDim.y = 1;
            at[0].val.clusterDim.z = 1;
            cfg.attrs = at;
            cfg.numAttrs = 1;
            B2_CUDA(h, cudaLaunchKernelEx(&cfg, split_directed_dp_kernel<D, true>, d_trk, (const int*)d_order, i,
                                          (const uint2*)q, (const SplitLevel*)lvl, (const uint32_t*)bits, max_runs,
                                          penalty, dec, arg, runs, nu));
          }
          B2_CHECK_LAUNCH(h, "split_directed_dp_kernel");
          i = e;
        }
        split_directed_backtrack_kernel<<<(unsigned)n, 256, 0, h->stream>>>(
            d_trk, g0, D, q, lvl, dec, arg, runs, nu, uo, sc, d_cue_offset + c_base, d_n_segments, d_split_score);
        B2_CHECK_LAUNCH(h, "split_directed_backtrack_kernel");
      }
      return B2_OK;
    };
    return direction > 0 ? run(std::integral_constant<int, 1>{}) : run(std::integral_constant<int, -1>{});
  }
  for (size_t g = 0; g + 1 < group_first.size(); ++g) {
    const int g0 = group_first[g], n = group_first[g + 1] - g0;
    if (n <= 0) continue;
    for (int i = g0; i < g0 + n;) {
      const int C = ncta[order[i]];
      int e = i;
      while (e < g0 + n && ncta[order[e]] == C) ++e;
      if (C == 1) {  // one CTA of the bucket's widest track's threads
        int thr = 32;
        for (int x = i; x < e; ++x) thr = std::max<int>(thr, (int)(32 * ceil_div64(trk[order[x]].nthr, 32)));
        split_dp_kernel<false><<<(unsigned)(e - i), (unsigned)thr, smem, h->stream>>>(
            d_trk, d_order, i, q, lvl, bits, max_runs, penalty, dec, arg, runs, nu);
      } else {  // CTAs of kCtaThreads threads: CTA r of a track owns its offsets r * kCtaWindow ..
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3((unsigned)((e - i) * C));
        cfg.blockDim = dim3((unsigned)kCtaThreads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = h->stream;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = (unsigned)C;
        at[0].val.clusterDim.y = 1;
        at[0].val.clusterDim.z = 1;
        cfg.attrs = at;
        cfg.numAttrs = 1;
        B2_CUDA(h, cudaLaunchKernelEx(&cfg, split_dp_kernel<true>, d_trk, (const int*)d_order, i, (const uint2*)q,
                                      (const SplitLevel*)lvl, (const uint32_t*)bits, max_runs, penalty, dec, arg, runs,
                                      nu));
      }
      B2_CHECK_LAUNCH(h, "split_dp_kernel");
      i = e;
    }
    // the kernel's cue indices are relative to c_base; d_cue_offset is indexed by absolute cue
    split_backtrack_kernel<<<(unsigned)n, 256, 0, h->stream>>>(d_trk, g0, q, lvl, dec, arg, runs, nu, uo, sc,
                                                              d_cue_offset + c_base, d_n_segments, d_split_score);
    B2_CHECK_LAUNCH(h, "split_backtrack_kernel");
  }
  return B2_OK;
}
