// K1: fused frame-energy / zero-crossing VAD over 10 ms windows of s16le PCM, and the
// counter-hash PCM synthesiser used by tests and bench.
//
// Replaces the per-window detector loop of the reference
// (ffsubsync/speech_transformers.py:155-183 called from :710-753): for every window of
// fpw = int(frame_rate/sample_rate + 0.5) samples emit 1.0 (speech) or non_speech_label.
// Rule (DESIGN.md, oracle/vad_oracle.py): E = sum x^2 (int64), Z = sign changes inside the
// window; speech <=> E >= fpw*energy_threshold and z_lo <= Z <= z_hi; a trailing partial
// window is non-speech.
//
// Roofline: pure HBM stream, 2*fpw bytes in -> 4 bytes out per window (320 B -> 4 B at 16 kHz).
// Persistent, warp-specialised CTAs: one producer warp moves tiles of TW windows HBM -> shared
// memory with 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx, SASS UBLKCP) into a
// ring of stages; eight consumer warps wait on the stage's "full" mbarrier, reduce their windows
// straight out of shared memory (conflict-free LDS.128) and release the stage through its
// "empty" mbarrier - no CTA-wide barrier on the steady-state path.
#include "common.cuh"
#include "vad_group.cuh"
#include "vad_layout.h"
#include "vad_lane.cuh"

namespace {

// lane-group kernel: 256 consumer threads per CTA (two such CTAs share an SM), a ring of up to
// kMaxStages stages
constexpr int kConsumerThreads = 256;
constexpr int kMaxStages = 10;
// lane-per-window kernel (vad_lane.cuh): tiles of 32 windows per consumer WARP, in a ring of up to
// kLaneMaxStages stages that fills the SM's shared memory; the producer warp claims and stages kLaneBatch
// tiles at a time, one per lane
constexpr int kLaneMaxStages = 24;
constexpr int kLaneBatch = 5;
constexpr int kLaneConsumers = 256;
constexpr int kLanePipes = 2;

struct TileDesc {
  long long out_base;   // index into out[] of the tile's first window
  long long n_left;     // samples of the signal from the tile's first sample to the signal end
  long long span_gbyte; // global byte offset of the staged span start
  int n_windows;        // windows in this tile (0 = no more tiles for this CTA)
  int sig;              // index of the signal the tile belongs to
  int head_bytes;       // offset of the first sample inside the 16 B-aligned staged span
  int tail_src_off;     // >=0: bytes [tail_src_off, tail_end) of the span must be copied by hand
  int tail_end;
  int seq;              // lane-per-window kernel: number of the tile in its CTA's staging order
};

struct VadParams {
  const unsigned char* pcm_bytes;
  float* out;
  const long long* pcm_off;   // [B+1] samples
  // [B] samples: signal b spans pcm_off[b] .. pcm_end[b] (signals need not abut: the sampled segments of
  // b2_sync_tracks_seg leave gaps and may overlap).  nullptr: pcm_off[b + 1].
  const long long* pcm_end;
  const long long* out_off;   // [B+1] windows
  const long long* tile_off;  // [B+1] tiles
  unsigned long long* tile_counter;  // zeroed before the launch
  long long total_tiles;
  long long pcm_total_bytes;
  long long e_min;            // smallest sum of squares of a full window that counts as speech
  // auditok contract (b2_vad_auditok): a trailing partial window of signal b is evaluated on the
  // samples it has, speech <=> sum x^2 >= tail_emin[b] (no zero-crossing band).  nullptr: the
  // webrtc contract - a partial window is non-speech.
  const long long* tail_emin;
  // lane-per-window kernel, packed output (b2i_vad_launch): the window bits m = (r == 1.0f) as words, signal b's
  // from bits + out_off[b] on; tiles then carry word offsets in out_base.  nullptr: float output to out.
  uint32_t* bits;
  int B, fpw, G, tw, z_lo, z_hi, fast, stage_bytes, cpl, stages, consumers, batch, evict_first;
  float label;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D TMA bulk copy global -> shared, completion signalled on an mbarrier.
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes,
                                             uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

// Sum (e, z) over the G lanes of a window (G a power of two <= 32, lanes contiguous).
template <int GT>
__device__ __forceinline__ void lane_group_sum(int G, long long& e, int& z) {
  if (GT > 0) {
#pragma unroll
    for (int off = GT >> 1; off > 0; off >>= 1) {
      e += __shfl_xor_sync(0xffffffffu, e, off);
      z += __shfl_xor_sync(0xffffffffu, z, off);
    }
  } else {
    for (int off = G >> 1; off > 0; off >>= 1) {
      e += __shfl_xor_sync(0xffffffffu, e, off);
      z += __shfl_xor_sync(0xffffffffu, z, off);
    }
  }
}

// All windows of one staged tile that belong to this thread's lane group (vector path: the window
// starts are 16-byte aligned inside the span).  CPL / GT are compile-time for the common rates.
template <int CPL, int GT>
__device__ __forceinline__ void consume_tile_fast(const VadParams& p, const TileDesc& d,
                                                  const unsigned char* span, int g, int wl0,
                                                  int wstep) {  // wstep = consumers / G
  const int fpw = p.fpw;
#pragma unroll 1
  for (int wl = wl0; wl < p.tw; wl += wstep) {  // uniform trip count: shuffles stay converged
    long long e = 0;
    int z = 0;
    const bool active = wl < d.n_windows;
    const long long avail = d.n_left - (long long)wl * fpw;
    const bool full = active && avail >= fpw;
    const bool tail = active && !full && avail > 0 && p.tail_emin != nullptr;
    if (full) {
      vadgroup::window_part_fast<CPL>(span + (size_t)wl * fpw * 2, g, p.cpl, e, z);
    } else if (tail) {  // at most one window per signal: plain 16-bit loop over the samples it has
      const short* xs = reinterpret_cast<const short*>(span + (size_t)wl * fpw * 2);
      for (int i = g; i < (int)avail; i += p.G) e += (long long)xs[i] * xs[i];
    }
    lane_group_sum<GT>(p.G, e, z);
    if (active && g == 0) {
      const bool speech = full ? (e >= p.e_min && z >= p.z_lo && z <= p.z_hi)
                               : (tail && e >= p.tail_emin[d.sig]);
      p.out[d.out_base + wl] = speech ? 1.0f : p.label;
    }
  }
}

// Descriptor of tile t (cur_b: signal index carried by the caller, tiles are claimed in ascending order);
// bulk = bytes the 1-D bulk copy moves from p.pcm_bytes + d.span_gbyte.
__device__ __forceinline__ TileDesc make_tile(const VadParams& p, long long t, int& cur_b, uint32_t& bulk) {
  TileDesc d;
  while (t >= p.tile_off[cur_b + 1]) ++cur_b;
  const long long w0 = (t - p.tile_off[cur_b]) * p.tw;
  const long long sig0 = p.pcm_off[cur_b], sig1 = p.pcm_end ? p.pcm_end[cur_b] : p.pcm_off[cur_b + 1];
  const long long nwin = p.out_off[cur_b + 1] - p.out_off[cur_b];
  const int nw = (int)min((long long)p.tw, nwin - w0);
  const long long s0 = sig0 + w0 * p.fpw;
  const long long s1 = min(s0 + (long long)nw * p.fpw, sig1);
  const long long b0 = 2 * s0, b1 = 2 * s1;
  const long long a0 = b0 & ~15LL;
  const long long a1 = (b1 + 15) & ~15LL;
  const long long limit = p.pcm_total_bytes & ~15LL;  // bulk copies stay inside the buffer
  const long long bulk_end = min(a1, limit);
  bulk = bulk_end > a0 ? (uint32_t)(bulk_end - a0) : 0u;
  d.n_windows = nw;
  d.sig = cur_b;
  d.out_base = p.out_off[cur_b] + w0;
  d.n_left = sig1 - s0;
  d.head_bytes = (int)(b0 - a0);
  d.span_gbyte = a0;
  if (bulk_end < b1) {  // ragged end of the whole buffer: < 16 bytes copied by hand
    d.tail_src_off = (int)(max(bulk_end, a0) - a0);
    d.tail_end = (int)(b1 - a0);
  } else {
    d.tail_src_off = -1;
    d.tail_end = 0;
  }
  return d;
}
__device__ __forceinline__ TileDesc end_tile() {
  TileDesc d;
  d.n_windows = 0;
  d.sig = 0;
  d.out_base = d.n_left = d.span_gbyte = 0;
  d.head_bytes = 0;
  d.tail_src_off = -1;
  d.tail_end = 0;
  return d;
}

__global__ void __launch_bounds__(kConsumerThreads + 32) vad_energy_zcr_kernel(VadParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* data = smem;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * p.stage_bytes);
  uint64_t* empty_bar = full_bar + kMaxStages;
  TileDesc* descs = reinterpret_cast<TileDesc*>(empty_bar + kMaxStages);

  const int nst = p.stages;
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < kMaxStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kConsumerThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (tid >= kConsumerThreads) {
    // ================================ producer warp ==========================================
    if (tid != kConsumerThreads) return;
    int cur_b = 0, stage = 0;
    uint32_t round = 0;  // how many times the ring wrapped
    for (;; ++stage) {
      if (stage == nst) {
        stage = 0;
        ++round;
      }
      if (round > 0) mbar_wait(&empty_bar[stage], (round - 1) & 1u);
      // dynamic tile hand-out: whichever CTAs are resident share the stream evenly, also when
      // this kernel co-runs with the correlation kernels and gets fewer than its 2 CTAs per SM
      const long long t = (long long)atomicAdd(p.tile_counter, 1ULL);
      TileDesc d;
      if (t >= p.total_tiles) {
        descs[stage] = end_tile();
        mbar_arrive(&full_bar[stage]);
        return;
      }
      uint32_t bulk;
      d = make_tile(p, t, cur_b, bulk);
      descs[stage] = d;
      if (bulk) {
        mbar_arrive_expect_tx(&full_bar[stage], bulk);
        tma_bulk_g2s(data + (size_t)stage * p.stage_bytes, p.pcm_bytes + d.span_gbyte, bulk, &full_bar[stage]);
      } else {
        mbar_arrive(&full_bar[stage]);
      }
    }
  }

  // ================================== consumer warps ==========================================
  const int G = p.G;
  const int g = tid % G;
  const int wl0 = tid / G;
  const int wstep = kConsumerThreads / G;
  const int fpw = p.fpw;
  int stage = 0;
  uint32_t phase = 0;
  for (;;) {
    mbar_wait(&full_bar[stage], phase);
    const TileDesc d = descs[stage];
    if (d.n_windows == 0) break;
    unsigned char* span = data + (size_t)stage * p.stage_bytes;
    if (d.tail_src_off >= 0) {  // rare: last < 16 bytes of the whole PCM buffer
      const int nb = d.tail_end - d.tail_src_off;
      if (tid < nb) span[d.tail_src_off + tid] = p.pcm_bytes[d.span_gbyte + d.tail_src_off + tid];
      asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
    }
    if (p.fast && d.head_bytes == 0) {
      if (p.cpl == 5 && G == 4) consume_tile_fast<5, 4>(p, d, span, g, wl0, wstep);         // 16 kHz
      else if (p.cpl == 15 && G == 4) consume_tile_fast<15, 4>(p, d, span, g, wl0, wstep);  // 48 kHz
      else consume_tile_fast<0, 0>(p, d, span, g, wl0, wstep);
    } else {
      for (int wl = wl0; wl < p.tw; wl += wstep) {
        long long e = 0;
        int z = 0;
        const bool active = wl < d.n_windows;
        const long long avail = d.n_left - (long long)wl * fpw;
        const bool full = active && avail >= fpw;
        const bool tail = active && !full && avail > 0 && p.tail_emin != nullptr;
        if (full || tail) {
          const short* xs = reinterpret_cast<const short*>(span + d.head_bytes + (size_t)wl * fpw * 2);
          const int n_use = full ? fpw : (int)avail;
          for (int i = g; i < n_use; i += G) {
            const int x = xs[i];
            const int px = i > 0 ? (int)xs[i - 1] : x;
            e += (long long)x * x;
            z += ((x < 0) != (px < 0));
          }
        }
        lane_group_sum<0>(G, e, z);
        if (active && g == 0) {
          const bool speech = full ? (e >= p.e_min && z >= p.z_lo && z <= p.z_hi)
                                   : (tail && e >= p.tail_emin[d.sig]);
          p.out[d.out_base + wl] = speech ? 1.0f : p.label;
        }
      }
    }
    __syncwarp();
    if ((tid & 31) == 0) mbar_arrive(&empty_bar[stage]);  // this warp is done with the stage
    if (++stage == nst) {
      stage = 0;
      phase ^= 1u;
    }
  }
}

// Bulk copy with an L2 evict-first policy: the PCM is read once; keeping it from displacing the reference
// spectra that the correlation kernels on the other SMs re-read K times (SM-partitioned pipeline).
__device__ __forceinline__ void tma_bulk_g2s_stream(void* dst, const void* src, uint32_t bytes, uint64_t* bar,
                                                    uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
          "r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

// ---- lane-per-window kernel ---------------------------------------------------------------------
// Same contract as above; tiles of 32 * WPL windows, tile number q of a CTA (in the order its producer
// stages them) goes to ring stage q mod nst and to consumer warp q mod 8; lane i of the warp reduces
// windows i, i + 32, ... with vadlane::lane_window (17 instructions per 16 bytes, no shuffles): 1.3
// instructions per byte and lane against 3.25 for the lane-group layout.  Launched for 8 and 16 kHz
// (C = 10, 20 chunks per window) and 16-byte aligned signals; everything else takes the kernel above.
//
// Producer.  One warp per SM has to stage a 10 KB tile every ~200 cycles to feed 100 GB/s per SM; a single
// thread needs ~600 (measured: 27-32 GB/s per SM).  So: the signal's table entries stay in registers
// (reloaded when a lane's tile sequence crosses into the next signal), interior tiles take a 20-instruction
// descriptor path, kLaneBatch lanes stage kLaneBatch tiles side by side (wait for the stage, descriptor,
// expect-tx, bulk copy: one pass of the instruction stream), and the next claim is requested one batch ahead.
//
// Consumers.  Bulk copies complete out of order, and a parity wait cannot tell "phase r complete" from
// "phase r - 2 complete": a warp that waits for tile q while the previous user of the stage (tile q - nst,
// consumed by a DIFFERENT warp) is still in flight would sail through.  The descriptor therefore carries the
// tile's sequence number: the producer writes it after the stage was released and before it arms the barrier,
// the consumer first polls it, then waits on the barrier (now at most one phase behind).
struct SigCache {
  int b;                    // signal index, -1 = nothing loaded
  long long tile_lo, tile_hi, sig0, sig1, nwin, out0;
};
__device__ __forceinline__ TileDesc make_tile_cached(const VadParams& p, long long t, SigCache& c, uint32_t& bulk) {
  if (c.b < 0 || t >= c.tile_hi) {
    int b = c.b < 0 ? 0 : c.b;
    while (t >= p.tile_off[b + 1]) ++b;
    c.b = b;
    c.tile_lo = p.tile_off[b];
    c.tile_hi = p.tile_off[b + 1];
    c.sig0 = p.pcm_off[b];
    c.sig1 = p.pcm_end ? p.pcm_end[b] : p.pcm_off[b + 1];
    c.out0 = p.out_off[b];
    c.nwin = p.out_off[b + 1] - c.out0;
  }
  TileDesc d;
  const long long w0 = (t - c.tile_lo) * p.tw;
  const long long s0 = c.sig0 + w0 * p.fpw;
  d.sig = c.b;
  d.out_base = c.out0 + (p.bits ? w0 >> 5 : w0);   // tiles start at multiples of 32 windows
  d.n_left = c.sig1 - s0;
  d.seq = 0;
  if (t + 1 < c.tile_hi) {
    // interior tile of a 16-byte aligned signal: whole windows, aligned at both ends, inside the buffer
    d.n_windows = p.tw;
    d.head_bytes = 0;
    d.span_gbyte = 2 * s0;
    d.tail_src_off = -1;
    d.tail_end = 0;
    bulk = (uint32_t)(p.tw * p.fpw * 2);
    return d;
  }
  const int nw = (int)min((long long)p.tw, c.nwin - w0);
  const long long s1 = min(s0 + (long long)nw * p.fpw, c.sig1);
  const long long b0 = 2 * s0, b1 = 2 * s1;
  const long long a0 = b0 & ~15LL;
  const long long a1 = (b1 + 15) & ~15LL;
  const long long limit = p.pcm_total_bytes & ~15LL;  // bulk copies stay inside the buffer
  const long long bulk_end = min(a1, limit);
  bulk = bulk_end > a0 ? (uint32_t)(bulk_end - a0) : 0u;
  d.n_windows = nw;
  d.head_bytes = (int)(b0 - a0);
  d.span_gbyte = a0;
  if (bulk_end < b1) {  // ragged end of the whole buffer: < 16 bytes copied by hand
    d.tail_src_off = (int)(max(bulk_end, a0) - a0);
    d.tail_end = (int)(b1 - a0);
  } else {
    d.tail_src_off = -1;
    d.tail_end = 0;
  }
  return d;
}

// Tile claim.  ptxas turns an atomic add on a provably uniform address into a warp-aggregated atomic whose
// result is shuffled out right away: the full round trip to L2 (~1300 cycles under load) then sits in front
// of every batch (measured: 1300 cycles + 140 per tile, for every batch size).  `skew` is a per-lane zero
// read from shared memory: the address is no longer provably uniform, the atomic stays a plain one and
// returns through the scoreboard - the warp stalls only where the value is used, one batch later.
__device__ __forceinline__ long long claim_tiles(unsigned long long* counter, int n, int skew) {
  unsigned long long r;
  asm volatile("atom.global.add.u64 %0, [%1], %2;" : "=l"(r) : "l"(counter + skew), "l"((unsigned long long)n) : "memory");
  return (long long)r;
}

template <int C, int WPL>
__global__ void __launch_bounds__(kLaneConsumers + 32 * kLanePipes) vad_lane_kernel(VadParams p) {
  constexpr int RMAX = vadlane::rotation_max(C);
  // kLanePipes independent pipelines per CTA: a producer warp, kLaneConsumers / 32 / kLanePipes consumer
  // warps and p.stages ring stages each (the producer's instruction stream is latency-bound: ~1200 cycles per
  // batch whatever the batch holds - two of them stage twice as much)
  constexpr int kWarps = kLaneConsumers / 32 / kLanePipes;   // consumer warps per pipeline
  extern __shared__ __align__(128) unsigned char smem[];
  const int nst = p.stages;   // per pipeline
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const bool is_producer = tid >= kLaneConsumers;
  const int pipe = is_producer ? warp - kLaneConsumers / 32 : warp / kWarps;
  uint64_t* bar0 = reinterpret_cast<uint64_t*>(smem + (size_t)kLanePipes * nst * p.stage_bytes);
  TileDesc* desc0 = reinterpret_cast<TileDesc*>(bar0 + 2 * kLaneMaxStages);
  unsigned char* data = smem + (size_t)pipe * nst * p.stage_bytes;
  uint64_t* full_bar = bar0 + pipe * nst;
  uint64_t* empty_bar = bar0 + kLaneMaxStages + pipe * nst;
  TileDesc* descs = desc0 + pipe * nst;
  volatile int* zeros = reinterpret_cast<volatile int*>(desc0 + kLaneMaxStages);   // 64 spare bytes
  if (tid == 0) {
    for (int s = 0; s < kLaneMaxStages; ++s) {
      mbar_init(&bar0[s], 1);
      mbar_init(&bar0[kLaneMaxStages + s], 1);   // released by the one warp that consumed the stage
      desc0[s].seq = -1;
    }
    for (int i = 0; i < 8; ++i) zeros[i] = 0;   // claim_tiles' skew
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (is_producer) {
    // ================================ producer warp ==========================================
    const int lane = tid & 31;
    SigCache sc;
    sc.b = -1;
    int q0 = 0;              // sequence number of the batch's first tile; it lives in stage0, ring pass `round`
    int stage0 = 0;
    uint32_t round = 0;
    int ends_left = kWarps;  // end markers still to post once the tiles are gone: one per consumer warp
    long long pending = 0;   // lane 0: first tile of the next claim, requested one batch ahead
    const int skew = zeros[lane & 7];   // 0, opaque to ptxas
    const uint64_t l2_policy = l2_evict_first_policy();
    if (lane == 0) pending = claim_tiles(p.tile_counter, p.batch, skew);
    for (;;) {
      const long long t0 = __shfl_sync(0xffffffffu, pending, 0);
      const int n = (int)max(0LL, min((long long)p.batch, p.total_tiles - t0));
      if (n > 0 && lane == 0) pending = claim_tiles(p.tile_counter, p.batch, skew);
      const int count = n > 0 ? n : min(ends_left, p.batch);   // slots staged by this batch
      if (lane < count) {
        TileDesc d = end_tile();
        uint32_t bulk = 0;
        if (n > 0) d = make_tile_cached(p, t0 + lane, sc, bulk);
        d.seq = q0 + lane;
        int stage = stage0 + lane;
        uint32_t rnd = round;
        if (stage >= nst) {
          stage -= nst;
          ++rnd;
        }
        if (rnd > 0) mbar_wait(&empty_bar[stage], (rnd - 1) & 1u);
        descs[stage] = d;
        if (bulk) {
          mbar_arrive_expect_tx(&full_bar[stage], bulk);
          if (p.evict_first)
            tma_bulk_g2s_stream(data + (size_t)stage * p.stage_bytes, p.pcm_bytes + d.span_gbyte, bulk,
                                &full_bar[stage], l2_policy);
          else
            tma_bulk_g2s(data + (size_t)stage * p.stage_bytes, p.pcm_bytes + d.span_gbyte, bulk, &full_bar[stage]);
        } else {
          mbar_arrive(&full_bar[stage]);
        }
      }
      __syncwarp();
      q0 += count;
      stage0 += count;
      if (stage0 >= nst) {
        stage0 -= nst;
        ++round;
      }
      if (n == 0) {
        ends_left -= count;
        if (ends_left == 0) return;
      }
    }
  }

  // ================================== consumer warps ==========================================
  const int lane = tid & 31;
  const int rot = vadlane::lane_rotation(C, lane);
  constexpr int fpw = 8 * C;
  int q = warp - pipe * kWarps;      // this warp's first tile
  int stage = q;                     // nst >= kWarps (launch condition)
  uint32_t phase = 0;
  for (;;) {
    // tile q staged?  (see above: only then is the parity wait unambiguous)
    while (*reinterpret_cast<volatile int*>(&descs[stage].seq) != q) {
    }
    mbar_wait(&full_bar[stage], phase);
    const TileDesc d = descs[stage];
    if (d.n_windows == 0) break;
    unsigned char* span = data + (size_t)stage * p.stage_bytes;
    if (d.tail_src_off >= 0) {  // rare: last < 16 bytes of the whole PCM buffer
      const int nb = d.tail_end - d.tail_src_off;
      if (lane < nb) span[d.tail_src_off + lane] = p.pcm_bytes[d.span_gbyte + d.tail_src_off + lane];
      __syncwarp();
    }
#pragma unroll 1
    for (int k = 0; k < WPL; ++k) {
      const int wl = lane + 32 * k;
      const bool active = wl < d.n_windows;
      const long long avail = d.n_left - (long long)wl * fpw;
      const bool full = active && avail >= fpw;
      long long e = 0;
      int z = 0;
      bool speech = false;
      if (full) {   // tiles start 16-byte aligned (launch condition): head_bytes == 0
        vadlane::lane_window<C, RMAX>(span + (size_t)wl * (fpw * 2), rot, e, z);
        speech = e >= p.e_min && z >= p.z_lo && z <= p.z_hi;
      } else if (active && avail > 0 && p.tail_emin != nullptr) {
        // auditok contract: the trailing partial window of a signal is judged on the samples it has
        const short* xs = reinterpret_cast<const short*>(span + (size_t)wl * (fpw * 2));
        for (int i = 0; i < (int)avail; ++i) e += (long long)xs[i] * xs[i];
        speech = e >= p.tail_emin[d.sig];
      }
      if (p.bits) {
        // packed: iteration k is word k of the tile (32 consecutive windows); m = (r == 1.0f) of the float below,
        // 0 past the last window.  A word wholly past it is not the signal's.
        const uint32_t m = __ballot_sync(0xffffffffu, active && (speech || p.label == 1.0f));
        if (lane == 0 && 32 * k < d.n_windows) p.bits[d.out_base + k] = m;
      } else if (active) {
        p.out[d.out_base + wl] = speech ? 1.0f : p.label;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    q += kWarps;
    stage += kWarps;
    if (stage >= nst) {
      stage -= nst;
      phase ^= 1u;
    }
  }
}

// ------------------------------------------------------------------------------ synthesiser
__device__ __forceinline__ uint32_t lowbias32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

__global__ void __launch_bounds__(256) synth_pcm_kernel(const uint8_t* __restrict__ cls,
                                                         long long n_windows, int fpw,
                                                         uint32_t seed, short* __restrict__ out) {
  const long long n = n_windows * (long long)fpw;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const long long w = i / fpw;
    const int pos = (int)(i - w * fpw);
    const uint32_t hsh = lowbias32(((uint32_t)i) ^ seed);
    const int c = cls[w];
    int v;
    if (c == 0)
      v = (int)((hsh >> 26) & 0x3fu) - 32;
    else if (c == 1)
      v = ((((pos / 40) & 1) == 0) ? 6000 : -6000) + (int)((hsh >> 14) & 0xfffu) - 2048;
    else
      v = (int)(hsh & 0x3fffu) - 8192;
    out[i] = (short)v;
  }
}

}  // namespace

int b2i_synth_launch(b2_ctx* h, const uint8_t* d_cls, int64_t n_windows, int fpw, uint32_t seed,
                     int16_t* d_out) {
  long long n = n_windows * (long long)fpw;
  int blocks = (int)std::min<long long>((n + 255) / 256, (long long)h->sm_count * 16);
  synth_pcm_kernel<<<blocks, 256, 0, h->stream>>>(d_cls, n_windows, fpw, seed, (short*)d_out);
  B2_CHECK_LAUNCH(h, "synth_pcm_kernel");
  return B2_OK;
}

// Would b2i_vad_launch take the lane-per-window kernel for these signals?  (b2_sync_batch pipelines
// sub-batches over an SM partition only then.)  An empty signal has no tiles, so where it starts does not
// matter (b2_sync_tracks_subs: a video with a subtitle reference has an empty PCM range).
bool b2i_vad_lane_eligible(const int64_t* pcm_off, int B, int fpw) {
  return vad_layout(pcm_off, nullptr, B, fpw, getenv("B2_VAD_LAYOUT")).kernel == kVadLane;
}

int b2i_vad_launch(b2_ctx* h, const int16_t* d_pcm, const int64_t* pcm_off, int B, int fpw,
                   float non_speech_label, int64_t e_min_full, int z_lo, int z_hi,
                   float* d_out, const int64_t* out_off, const int64_t* tail_emin, bool packed,
                   const int64_t* pcm_end) {
  B2Range range("b2:vad_energy_zcr");
  auto sig_end = [&](int b) { return pcm_end ? pcm_end[b] : pcm_off[b + 1]; };
  if (((uintptr_t)d_pcm & 15) != 0)
    B2_FAIL(h, B2_ERR_BAD_ARG, "vad: device PCM pointer must be 16-byte aligned");
  VadParams p;
  p.consumers = kConsumerThreads;
  // which kernel, and its lanes per window (vad_layout.h)
  const int C = fpw / 8;
  const VadLayout lay = vad_layout(pcm_off, pcm_end, B, fpw, getenv("B2_VAD_LAYOUT"));
  p.fast = lay.kernel != kVadGeneric ? 1 : 0;
  const int G = lay.G;
  p.G = G;
  p.cpl = p.fast ? C / G : 0;
  // tile = wpt rounds of (256 / G) windows: per-tile costs (mbarrier wait, descriptor, release)
  // are amortised over wpt windows per lane group
  int wpt = 1;
  if (const char* e = getenv("B2_VAD_WPT")) wpt = std::max(1, std::min(8, atoi(e)));  // tuning knob
  p.fpw = fpw;
  // Ring depth matters more than resident warps (tools/vad_tune.py sweeps stages x CTAs per SM),
  // so the ring is 4 deep when two such CTAs fit an SM.
  int stages = 4;
  if (const char* e = getenv("B2_VAD_STAGES")) stages = std::max(2, std::min(kMaxStages, atoi(e)));  // tuning knob
  for (;;) {
    p.tw = wpt * (kConsumerThreads / G);
    p.stage_bytes = ((p.tw * fpw * 2 + 32) + 127) & ~127;
    if ((size_t)stages * p.stage_bytes <= 200 * 1024) break;
    if (wpt > 1) --wpt;
    else if (stages > 2) --stages;
    else break;
  }
  p.stages = stages;
  size_t smem = (size_t)stages * p.stage_bytes + 2 * kMaxStages * sizeof(uint64_t) +
                kMaxStages * sizeof(TileDesc) + 64;
  if (smem > 227 * 1024) B2_FAIL(h, B2_ERR_UNSUPPORTED, "vad: window of %d samples too large", fpw);

  std::vector<long long> tile_off(B + 1);
  tile_off[0] = 0;
  for (int b = 0; b < B; ++b) {
    long long n = sig_end(b) - pcm_off[b];
    long long nwin = (n + fpw - 1) / fpw;
    tile_off[b + 1] = tile_off[b] + (nwin + p.tw - 1) / p.tw;
  }
  // lane-per-window kernel: 16-byte aligned signals and an instantiated chunk count (8 / 16 kHz at 100 windows
  // per second).  B2_VAD_LAYOUT=group keeps the lane-group kernel (A/B and test knob).
  const bool lane_layout = lay.kernel == kVadLane;
  // windows per lane and tile: stages of 10 KB
  int wpl = C == 10 ? 2 : 1;
  if (const char* e = getenv("B2_VAD_WPL")) wpl = (C == 10 ? 2 : 1) * (atoi(e) >= 2 ? 2 : 1);   // tuning knob
  if (lane_layout) {
    p.tw = 32 * wpl;
    p.stage_bytes = ((p.tw * fpw * 2 + 32) + 127) & ~127;
    // ring stages per pipeline (at least one per consumer warp of the pipeline)
    stages = std::min<int>(kLaneMaxStages, (int)((208 * 1024) / p.stage_bytes)) / kLanePipes;
    if (const char* e = getenv("B2_VAD_STAGES"))
      stages = std::max(kLaneConsumers / 32 / kLanePipes, std::min(stages, atoi(e)));
    p.consumers = kLaneConsumers;
    p.stages = stages;
    p.evict_first = 1;
    if (const char* e = getenv("B2_VAD_EVICT_FIRST")) p.evict_first = atoi(e) != 0;   // A/B knob
    p.batch = kLaneBatch;
    if (const char* e = getenv("B2_VAD_BATCH")) p.batch = std::max(1, std::min(16, atoi(e)));   // tuning knob
    // lane l of a producer pass stages into stage0 + l, wrapped once: a batch deeper than the ring would run
    // past the pipeline's stages (and two lanes of one pass would share a stage)
    p.batch = std::min(p.batch, stages);
    smem = (size_t)kLanePipes * stages * p.stage_bytes + 2 * kLaneMaxStages * sizeof(uint64_t) +
           kLaneMaxStages * sizeof(TileDesc) + 64;
    for (int b = 0; b < B; ++b) {
      const long long n = sig_end(b) - pcm_off[b];
      tile_off[b + 1] = tile_off[b] + ((n + fpw - 1) / fpw + p.tw - 1) / p.tw;
    }
  }
  if (packed && !lane_layout)
    B2_FAIL(h, B2_ERR_UNSUPPORTED, "vad: internal error: packed output asked of the lane-group kernel");
  p.bits = packed ? reinterpret_cast<uint32_t*>(d_out) : nullptr;
  p.total_tiles = tile_off[B];
  if (p.total_tiles == 0) return B2_OK;

  MetaArena a;
  size_t tbl = (size_t)(B + 1) * 8;
  B2_TRY(b2i_meta_begin(h, &a, (pcm_end ? 5 : 4) * tbl + 256));
  p.pcm_off = (const long long*)b2i_meta_put(&a, pcm_off, tbl);
  p.pcm_end = pcm_end ? (const long long*)b2i_meta_put(&a, pcm_end, (size_t)B * 8) : nullptr;
  p.out_off = (const long long*)b2i_meta_put(&a, out_off, tbl);
  p.tile_off = (const long long*)b2i_meta_put(&a, tile_off.data(), tbl);
  p.tail_emin = tail_emin ? (const long long*)b2i_meta_put(&a, tail_emin, (size_t)B * 8) : nullptr;
  B2_TRY(b2i_meta_commit(&a));

  p.pcm_bytes = (const unsigned char*)d_pcm;
  p.out = d_out;
  p.B = B;
  // bulk copies stay below the last sample any signal reads (with pcm_end: the largest end; the caller's buffer
  // holds at least that much)
  long long pcm_total = pcm_off[B];
  if (pcm_end) {
    pcm_total = 0;
    for (int b = 0; b < B; ++b)
      if (pcm_end[b] > pcm_off[b]) pcm_total = std::max<long long>(pcm_total, pcm_end[b]);
  }
  p.pcm_total_bytes = 2 * pcm_total;
  p.e_min = (long long)e_min_full;
  p.z_lo = z_lo;
  p.z_hi = z_hi;
  p.label = non_speech_label;

  void* d_counter;
  B2_TRY(b2i_ws(h, b2_ctx::WS_COUNTERS, 64, &d_counter));
  p.tile_counter = (unsigned long long*)d_counter;
  B2_CUDA(h, cudaMemsetAsync(d_counter, 0, 8, h->stream));
  if (lane_layout) {
    void (*lk)(VadParams) = C == 10 ? (wpl == 2 ? vad_lane_kernel<10, 2> : vad_lane_kernel<10, 4>)
                                    : (wpl == 1 ? vad_lane_kernel<20, 1> : vad_lane_kernel<20, 2>);
    if (smem < 116 * 1024) smem = 116 * 1024;   // one CTA per SM: the ring is sized for the whole SM
    B2_CUDA(h, cudaFuncSetAttribute(lk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // tiles are claimed kLaneBatch at a time: no point in more CTAs than claims
    long long grid = std::min<long long>((p.total_tiles + kLanePipes * p.batch - 1) / (kLanePipes * p.batch), (long long)h->sm_count);
    // b2_sync_batch's pipeline: this many SMs for the VAD, the rest for the correlation kernels
    if (h->vad_partition_sms > 0) grid = std::min<long long>(grid, h->vad_partition_sms);
    lk<<<(unsigned)grid, kLaneConsumers + 32 * kLanePipes, smem, h->stream>>>(p);
    B2_CHECK_LAUNCH(h, "vad_lane_kernel");
    return B2_OK;
  }
  B2_CUDA(h, cudaFuncSetAttribute(vad_energy_zcr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (220 * 1024) / smem));
  if (const char* f = getenv("B2_VAD_CTAS_FORCE")) per_sm = std::max(1, atoi(f));  // profiling knob
  const long long grid = std::min<long long>(p.total_tiles, (long long)h->sm_count * per_sm);
  vad_energy_zcr_kernel<<<(unsigned)grid, kConsumerThreads + 32, smem, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "vad_energy_zcr_kernel");
  return B2_OK;
}
