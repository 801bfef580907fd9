// C-ABI entry points (include/ffsubsync_b200.h): handle lifecycle, workspace management and
// the host<->device staging that turns B2_HOST calls into the device path.  All arithmetic
// lives in the kernels (vad.cu, tokenizer.cu, raster.cu, corr.cu, bigfft.cu); nothing here computes
// results on the CPU.  The batched sync calls are planned on the host by sync_plan.h (argument checks,
// tables, sub-batch cuts) and run by the pipeline at the end of this file.
#include <math.h>

#include <chrono>
#include <cmath>
#include <algorithm>
#include <atomic>
#include <thread>

#include "common.cuh"
#include "sync_plan.h"

// Entry guard: the handle's device is current for the duration of the call and the caller
// thread's previous device is restored on every return path.
struct DeviceScope {
  int prev = -1, want;
  bool ok = true;
  explicit DeviceScope(int dev) : want(dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != want) ok = cudaSetDevice(want) == cudaSuccess;
  }
  ~DeviceScope() {
    if (prev >= 0 && prev != want) cudaSetDevice(prev);
  }
};
extern "C" int b2_version(void) { return 200; }

static uint64_t compute_log2_quirk_mask() {
  // CPython: total_bits = math.log(n, 2) == log(n)/log(2) in double; ceil() of that is k+1 for
  // some exact powers of two (k = 29, 31, 39, ... with glibc).  Reproduced with the same libm.
  uint64_t mask = 0;
  for (int k = 0; k < 63; ++k) {
    double v = log((double)(1ULL << k)) / log(2.0);
    if (ceil(v) > (double)k) mask |= (1ULL << k);
  }
  return mask;
}

extern "C" int b2_create(int device, b2_handle* out) {
  if (!out) return B2_ERR_BAD_ARG;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count)
    return B2_ERR_CUDA;
  b2_ctx* h = new b2_ctx();
  h->device = device;
  DeviceScope scope(device);
  if (!scope.ok) { delete h; return B2_ERR_CUDA; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete h; return B2_ERR_CUDA; }
  h->sm_count = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) {  // built for sm_90a only: fail loudly instead of falling back
    delete h;
    return B2_ERR_UNSUPPORTED;
  }
  if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete h;
    return B2_ERR_CUDA;
  }
  h->own_stream = true;
  // internal second stream at the highest priority: when b2_sync_batch pipelines sub-batches, the VAD CTAs
  // queued on it take the SMs that the (lower-priority) correlation CTAs of the caller's stream give up
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
  if (cudaStreamCreateWithPriority(&h->stream2, cudaStreamNonBlocking, prio_hi) != cudaSuccess) {
    cudaStreamDestroy(h->stream);
    delete h;
    return B2_ERR_CUDA;
  }
  for (auto& e : h->ev_pool)
    if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) {
      delete h;
      return B2_ERR_CUDA;
    }
  if (cudaEventCreateWithFlags(&h->resident_fence, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&h->resident_done, cudaEventDisableTiming) != cudaSuccess) {
    delete h;
    return B2_ERR_CUDA;
  }
  h->log2_quirk_mask = compute_log2_quirk_mask();
  *out = h;
  return B2_OK;
}

extern "C" int b2_destroy(b2_handle h) {
  if (!h) return B2_OK;
  DeviceScope scope(h->device);
  if (h->stream2) cudaStreamSynchronize(h->stream2);
  cudaStreamSynchronize(h->stream);
  for (auto& w : h->ws)
    if (w.p) cudaFree(w.p);
  for (auto& p : h->pinned)
    if (p.p) cudaFreeHost(p.p);
  for (auto& e : h->pinned_ev)
    if (e) cudaEventDestroy(e);
  for (auto& b : h->bounce) {
    if (b.p) cudaFreeHost(b.p);
    if (b.ev) cudaEventDestroy(b.ev);
  }
  for (auto& sl : h->vs.slot) {
    if (sl.hp) cudaFreeHost(sl.hp);
    if (sl.hout) cudaFreeHost(sl.hout);
    if (sl.dp) cudaFree(sl.dp);
    if (sl.dout) cudaFree(sl.dout);
    if (sl.ev) cudaEventDestroy(sl.ev);
  }
  if (h->stream2) cudaStreamSynchronize(h->stream2);
  for (auto& ring : h->meta)
    for (auto& m : ring) {
      if (m.d) cudaFree(m.d);
      if (m.p) cudaFreeHost(m.p);
      if (m.ev) cudaEventDestroy(m.ev);
    }
  for (auto& e : h->ev_pool)
    if (e) cudaEventDestroy(e);
  if (h->resident_fence) cudaEventDestroy(h->resident_fence);
  if (h->resident_done) cudaEventDestroy(h->resident_done);
  if (h->stream2) cudaStreamDestroy(h->stream2);
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return B2_OK;
}

extern "C" int b2_set_stream(b2_handle h, void* s) {
  if (!h) return B2_ERR_BAD_ARG;
  DeviceScope scope(h->device);
  if (h->own_stream && h->stream) {
    cudaStreamSynchronize(h->stream);
    cudaStreamDestroy(h->stream);
  }
  if (s) {
    h->stream = (cudaStream_t)s;
    h->own_stream = false;
  } else {
    B2_CUDA(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    h->own_stream = true;
  }
  return B2_OK;
}

extern "C" int b2_synchronize(b2_handle h) {
  if (!h) return B2_ERR_BAD_ARG;
  DeviceScope scope(h->device);
  B2_CUDA(h, cudaStreamSynchronize(h->stream));
  return B2_OK;
}

extern "C" const char* b2_last_error(b2_handle h) { return h ? h->err.c_str() : "null handle"; }
extern "C" int64_t b2_launch_count(b2_handle h) { return h ? h->launches : 0; }

// ---- workspaces --------------------------------------------------------------------------
int b2i_ws(b2_ctx* h, int which, size_t bytes, void** out) {
  DeviceBuf& w = h->ws[which];
  if (bytes > w.cap) {
    // stream-ordered reuse: earlier kernels may still read the old block
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
    if (w.p) B2_CUDA(h, cudaFree(w.p));
    w.p = nullptr;
    w.cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&w.p, want);
    if (e != cudaSuccess) {
      cudaGetLastError();
      B2_FAIL(h, B2_ERR_NOMEM, "cudaMalloc(%zu) for workspace %d failed: %s", want, which,
              cudaGetErrorString(e));
    }
    w.cap = want;
  }
  *out = w.p;
  return B2_OK;
}

int b2i_pinned(b2_ctx* h, int which, size_t bytes, void** out) {
  HostBuf& w = h->pinned[which];
  if (bytes > w.cap) {
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
    if (w.p) B2_CUDA(h, cudaFreeHost(w.p));
    w.p = nullptr;
    w.cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    B2_CUDA(h, cudaMallocHost(&w.p, want));
    w.cap = want;
  }
  *out = w.p;
  return B2_OK;
}

// Metadata arena: host-side tables (offsets, per-job parameters) are packed into one pinned
// block and uploaded with a single async copy per call.
// Arenas come from a ring of kMetaSlots (pinned, device) buffer pairs so that the host can plan
// and upload several launches ahead of the GPU without synchronising the stream.  A slot is
// reused kMetaSlots arenas later; the event recorded at the commit of the arena that FOLLOWED its
// previous use guarantees (in-order stream) that both its upload and every kernel that read its
// device copy have finished.
int b2i_meta_begin(b2_ctx* h, MetaArena* a, size_t bytes) {
  a->h = h;
  bytes = (bytes + 255) & ~size_t(255);
  b2_ctx::MetaSlot* ring = h->meta[h->ring];
  uint64_t& seq = h->meta_seq[h->ring];
  const int slot = (int)(seq % b2_ctx::kMetaSlots);
  b2_ctx::MetaSlot& next = ring[(slot + 1) % b2_ctx::kMetaSlots];
  if (seq >= (uint64_t)b2_ctx::kMetaSlots && next.ev) B2_CUDA(h, cudaEventSynchronize(next.ev));
  b2_ctx::MetaSlot& s = ring[slot];
  if (!s.ev) B2_CUDA(h, cudaEventCreateWithFlags(&s.ev, cudaEventDisableTiming));
  if (bytes > s.cap) {
    // grow every slot of this ring at once (pinned allocations cost milliseconds): after the
    // first large call no later arena, whichever slot it lands on, allocates again
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
    const size_t want = bytes + bytes / 4 + 65536;
    for (int i = 0; i < b2_ctx::kMetaSlots; ++i) {
      b2_ctx::MetaSlot& m = ring[i];
      if (m.cap >= want) continue;
      if (m.d) B2_CUDA(h, cudaFree(m.d));
      if (m.p) B2_CUDA(h, cudaFreeHost(m.p));
      m.d = m.p = nullptr;
      m.cap = 0;
      B2_CUDA(h, cudaMalloc(&m.d, want));
      B2_CUDA(h, cudaMallocHost(&m.p, want));
      m.cap = want;
    }
  }
  a->slot = slot;
  a->ring = h->ring;
  a->dbase = (char*)s.d;
  a->hbase = (char*)s.p;
  a->cap = bytes;
  a->used = 0;
  seq++;
  return B2_OK;
}

void* b2i_meta_reserve(MetaArena* a, size_t bytes, void** host_view) {
  size_t at = (a->used + 15) & ~size_t(15);
  if (at + bytes > a->cap) return nullptr;
  a->used = at + bytes;
  if (host_view) *host_view = a->hbase + at;
  return a->dbase + at;
}

void* b2i_meta_put(MetaArena* a, const void* src, size_t bytes) {
  void* hv;
  void* d = b2i_meta_reserve(a, bytes, &hv);
  if (d && bytes) memcpy(hv, src, bytes);
  return d;
}

int b2i_meta_commit(MetaArena* a) {
  b2_ctx* h = a->h;
  if (a->used)
    B2_CUDA(h, cudaMemcpyAsync(a->dbase, a->hbase, a->used, cudaMemcpyHostToDevice, h->stream));
  B2_CUDA(h, cudaEventRecord(h->meta[a->ring][a->slot].ev, h->stream));
  return B2_OK;
}

// Run `body` with the handle temporarily launching on its internal second stream.
struct Stream2Scope {
  b2_ctx* h;
  cudaStream_t saved;
  int saved_ring;
  explicit Stream2Scope(b2_ctx* hh) : h(hh), saved(hh->stream), saved_ring(hh->ring) {
    h->stream = h->stream2;
    h->ring = 1;
  }
  ~Stream2Scope() {
    h->stream = saved;
    h->ring = saved_ring;
  }
};

static cudaEvent_t next_event(b2_ctx* h) {
  cudaEvent_t e = h->ev_pool[h->ev_next];
  h->ev_next = (h->ev_next + 1) % b2_ctx::kEvents;
  return e;
}

// ---- helpers for B2_HOST calls -------------------------------------------------------------
// Large PAGEABLE inputs (a numpy array of PCM: 230 MB per 2 h signal): cudaMemcpyAsync stages them
// through the driver's bounce buffer with one thread, several times slower than a copy from pinned
// memory.  Here the copy goes through two
// pinned 32 MB buffers filled by kCopyThreads host threads while the previous buffer is on the bus.
static const size_t kBounceBytes = (size_t)32 << 20;
static const int kCopyThreads = 6;

static bool is_pageable(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeUnregistered;
}

// Copy workers live for one staged transfer: worker t copies slice t of every chunk into the bounce
// buffer the main thread announces (`ready`), and reports through `done`; the main thread turns each
// filled buffer into an async H2D copy.  No thread is created per chunk; the only blocking wait is
// on the event of the H2D copy that last read the buffer.
struct CopyCrew {
  std::atomic<int> ready{-1};           // index of the chunk whose bounce buffer may be filled
  std::atomic<int> done{0};             // slices finished, over all chunks
  std::atomic<bool> abort{false};
};

static void copy_slice(char* dst, const char* src, size_t n, int t, int nthreads) {
  const size_t per = ((n / nthreads) + 4095) & ~(size_t)4095;
  const size_t lo = std::min(n, per * (size_t)t), hi = t == nthreads - 1 ? n : std::min(n, per * (size_t)(t + 1));
  if (hi > lo) memcpy(dst + lo, src + lo, hi - lo);
}

static int staged_h2d(b2_ctx* h, void* dev, const void* host, size_t bytes) {
  for (auto& b : h->bounce)
    if (!b.p) {
      B2_CUDA(h, cudaMallocHost(&b.p, kBounceBytes));
      B2_CUDA(h, cudaEventCreateWithFlags(&b.ev, cudaEventDisableTiming));
    }
  const int n_chunks = (int)((bytes + kBounceBytes - 1) / kBounceBytes);
  CopyCrew crew;
  std::thread workers[kCopyThreads];
  int n_workers = 0;   // helpers besides this thread (slice 0 is copied here)
  auto work = [&](int t, int nthreads) {
    for (int c = 0; c < n_chunks; ++c) {
      while (crew.ready.load(std::memory_order_acquire) < c) {
        if (crew.abort.load(std::memory_order_relaxed)) return;
        std::this_thread::yield();
      }
      const size_t off = (size_t)c * kBounceBytes, n = std::min(kBounceBytes, bytes - off);
      copy_slice((char*)h->bounce[c & 1].p, (const char*)host + off, n, t, nthreads);
      crew.done.fetch_add(1, std::memory_order_release);
    }
  };
  try {
    for (; n_workers < kCopyThreads - 1; ++n_workers) workers[n_workers] = std::thread(work, n_workers + 1, kCopyThreads);
  } catch (...) {   // no more threads to be had: nothing may escape through the C ABI
    crew.abort.store(true);
    for (int i = 0; i < n_workers; ++i) workers[i].join();
    n_workers = 0;
    crew.abort.store(false);
  }
  const int nthreads = n_workers == kCopyThreads - 1 ? kCopyThreads : 1;   // all helpers or none
  int status = B2_OK;
  for (int c = 0; c < n_chunks && status == B2_OK; ++c) {
    b2_ctx::Bounce& b = h->bounce[c & 1];
    const size_t off = (size_t)c * kBounceBytes, n = std::min(kBounceBytes, bytes - off);
    if (cudaEventSynchronize(b.ev) != cudaSuccess) {   // the copy that last read this buffer
      status = B2_ERR_CUDA;
      break;
    }
    crew.ready.store(c, std::memory_order_release);
    copy_slice((char*)b.p, (const char*)host + off, n, 0, nthreads);
    while (crew.done.load(std::memory_order_acquire) < (c + 1) * (nthreads - 1)) std::this_thread::yield();
    if (cudaMemcpyAsync((char*)dev + off, b.p, n, cudaMemcpyHostToDevice, h->stream) != cudaSuccess ||
        cudaEventRecord(b.ev, h->stream) != cudaSuccess)
      status = B2_ERR_CUDA;
  }
  if (status != B2_OK) crew.abort.store(true);
  crew.ready.store(n_chunks, std::memory_order_release);
  for (int i = 0; i < n_workers; ++i) workers[i].join();
  if (status != B2_OK) B2_FAIL(h, status, "staged host-to-device copy failed: %s", cudaGetErrorString(cudaGetLastError()));
  return B2_OK;
}

static int stage_in(b2_ctx* h, int which, const void* host, size_t bytes, void** dev) {
  B2_TRY(b2i_ws(h, which, bytes ? bytes : 16, dev));
  if (!bytes) return B2_OK;
  if (bytes >= kBounceBytes / 2 && is_pageable(host)) return staged_h2d(h, *dev, host, bytes);
  B2_CUDA(h, cudaMemcpyAsync(*dev, host, bytes, cudaMemcpyHostToDevice, h->stream));
  return B2_OK;
}

static int copy_out(b2_ctx* h, void* host, const void* dev, size_t bytes) {
  if (bytes)
    B2_CUDA(h, cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, h->stream));
  return B2_OK;
}

#define B2_ENTER(h)                                              \
  if (!(h)) return B2_ERR_BAD_ARG;                               \
  (h)->err.clear();                                              \
  const bool _b2_fence_was_valid = (h)->resident_fence_valid;    \
  (void)_b2_fence_was_valid;                                     \
  (h)->resident_fence_valid = false; /* any entry point breaks a chain of resident b2_sync_batch calls */ \
  DeviceScope _b2_scope((h)->device);                            \
  if (!_b2_scope.ok) return B2_ERR_CUDA;

// B2_DEVICE calls: a bulk pointer must be device (or managed) memory of the handle's device.
static int check_device_ptr(b2_ctx* h, const void* p, const char* what) {
  if (!p) return B2_OK;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    B2_FAIL(h, B2_ERR_BAD_ARG, "%s: not a CUDA pointer", what);
  }
  if (at.type == cudaMemoryTypeManaged) return B2_OK;
  if (at.type != cudaMemoryTypeDevice)
    B2_FAIL(h, B2_ERR_BAD_ARG, "%s: B2_DEVICE call with a host pointer", what);
  if (at.device != h->device)
    B2_FAIL(h, B2_ERR_BAD_ARG, "%s: pointer lives on device %d, the handle on device %d", what, at.device,
            h->device);
  return B2_OK;
}
#define B2_CHECK_DEV(h, memspace, p, what)                                                       \
  do {                                                                                           \
    if ((memspace) != B2_HOST && (memspace) != B2_DEVICE) /* b2_sync_batch maps RESIDENT first */ \
      B2_FAIL(h, B2_ERR_BAD_ARG, "%s: memspace must be B2_HOST or B2_DEVICE", what);             \
    if ((memspace) == B2_DEVICE) B2_TRY(check_device_ptr(h, p, what));                           \
  } while (0)

// ---- VAD -----------------------------------------------------------------------------------
extern "C" int b2_vad_frames_per_window(int frame_rate, int sample_rate) {
  return vad_frames_per_window(frame_rate, sample_rate);
}

extern "C" int64_t b2_vad_num_windows(int64_t n_samples, int frame_rate, int sample_rate) {
  int fpw = b2_vad_frames_per_window(frame_rate, sample_rate);
  if (fpw <= 0 || n_samples < 0) return -1;
  return (n_samples + fpw - 1) / fpw;  // len(range(0, n, fpw)), speech_transformers.py:169
}

extern "C" int b2_vad_energy_zcr(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int B,
                                 int frame_rate, int sample_rate, float non_speech_label,
                                 int64_t energy_threshold, int z_lo, int z_hi, float* out,
                                 const int64_t* out_off, int memspace) {
  B2_ENTER(h);
  if (B < 0 || !pcm_off || !out_off) B2_FAIL(h, B2_ERR_BAD_ARG, "vad: null offset table / B<0");
  int fpw = b2_vad_frames_per_window(frame_rate, sample_rate);
  if (fpw <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "vad: bad frame_rate/sample_rate");
  if (energy_threshold < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "vad: negative energy threshold");
  if (z_lo < 0) z_lo = 0;
  if (z_hi < 0) z_hi = (3 * fpw) / 8;
  for (int b = 0; b < B; ++b) {
    int64_t n = pcm_off[b + 1] - pcm_off[b];
    if (n < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "vad: pcm_off not monotone at %d", b);
    if (out_off[b + 1] - out_off[b] != (n + fpw - 1) / fpw)
      B2_FAIL(h, B2_ERR_BAD_ARG, "vad: out_off[%d] span must be ceil(n/fpw)", b);
  }
  if (B == 0) return B2_OK;
  int64_t n_total = pcm_off[B], w_total = out_off[B];
  if ((n_total && !pcm) || (w_total && !out)) B2_FAIL(h, B2_ERR_BAD_ARG, "vad: null data pointer");
  B2_CHECK_DEV(h, memspace, pcm, "vad: pcm");
  B2_CHECK_DEV(h, memspace, out, "vad: out");
  const int16_t* d_pcm = pcm;
  float* d_out = out;
  if (memspace == B2_HOST) {
    void *dp, *dq;
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, pcm, (size_t)n_total * 2, &dp));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)w_total * 4 + 16, &dq));
    d_pcm = (const int16_t*)dp;
    d_out = (float*)dq;
  }
  B2_TRY(b2i_vad_launch(h, d_pcm, pcm_off, B, fpw, non_speech_label, (int64_t)fpw * energy_threshold,
                        z_lo, z_hi, d_out, out_off));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, out, d_out, (size_t)w_total * 4));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- auditok detector (speech_transformers.py:101-152) ---------------------------------------
extern "C" int b2_auditok_block_size(int frame_rate, int sample_rate) {
  return auditok_block_size(frame_rate, sample_rate);
}

extern "C" int64_t b2_auditok_energy_floor(int n_samples, double energy_threshold_db) {
  return auditok_energy_floor(n_samples, energy_threshold_db);
}

extern "C" int b2_vad_auditok(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int B,
                              int frame_rate, int sample_rate, double non_speech_label,
                              double energy_threshold_db, double min_length, int64_t max_length,
                              double max_continuous_silence, int64_t chunk_samples, double* out,
                              const int64_t* out_off, int memspace) {
  B2_ENTER(h);
  if (B < 0 || !pcm_off || !out_off) B2_FAIL(h, B2_ERR_BAD_ARG, "auditok: null offset table / B<0");
  const int fpw = auditok_block_size(frame_rate, sample_rate);
  if (fpw <= 0)
    B2_FAIL(h, B2_ERR_UNSUPPORTED, "auditok: int(frame_rate/sample_rate) block size and frame_rate//sample_rate "
                                   "window size differ (or are 0) for %d / %d", frame_rate, sample_rate);
  if (!tokenizer_params_ok(min_length, max_length, max_continuous_silence, chunk_samples))
    B2_FAIL(h, B2_ERR_BAD_ARG, "auditok: bad tokenizer parameters");
  // one detector call per chunk: chunk c of signal b becomes "signal" n of the batched energy kernel
  ChunkTable ct;
  build_chunk_table(pcm_off, B, B ? pcm_off[0] : 0, fpw, chunk_samples, energy_threshold_db, nullptr, &ct);
  for (int b = 0; b < B; ++b) {
    if (pcm_off[b + 1] < pcm_off[b]) B2_FAIL(h, B2_ERR_BAD_ARG, "auditok: pcm_off not monotone at %d", b);
    if (out_off[b + 1] - out_off[b] != ct.out[ct.first[b + 1]] - ct.out[ct.first[b]])
      B2_FAIL(h, B2_ERR_BAD_ARG, "auditok: out_off[%d] span must be the sum of ceil(chunk/fpw)", b);
  }
  const int n_chunks = (int)ct.tail.size();
  if (n_chunks == 0) return B2_OK;
  const int64_t n_total = pcm_off[B] - pcm_off[0], w_total = ct.out.back();
  if ((n_total && !pcm) || (w_total && !out)) B2_FAIL(h, B2_ERR_BAD_ARG, "auditok: null data pointer");
  B2_CHECK_DEV(h, memspace, pcm, "auditok: pcm");
  B2_CHECK_DEV(h, memspace, out, "auditok: out");
  const int16_t* d_pcm = pcm + pcm_off[0];
  double* d_out = out + out_off[0];
  void *d_flags, *dp, *dq;
  if (memspace == B2_HOST) {
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, pcm + pcm_off[0], (size_t)n_total * 2, &dp));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)w_total * 8 + 16, &dq));
    d_pcm = (const int16_t*)dp;
    d_out = (double*)dq;
  }
  B2_TRY(b2i_ws(h, b2_ctx::WS_SIG_REF, (size_t)w_total * 4 + 64, &d_flags));
  B2_TRY(b2i_vad_launch(h, d_pcm, ct.pcm.data(), n_chunks, fpw, 0.0f, auditok_energy_floor(fpw, energy_threshold_db),
                        0, fpw, (float*)d_flags, ct.out.data(), ct.tail.data()));
  B2TokenizerParams tp{min_length, max_continuous_silence, non_speech_label, (long long)max_length};
  B2_TRY(b2i_tokenize_launch(h, (const float*)d_flags, ct.out.data(), n_chunks, tp, d_out));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, out + out_off[0], d_out, (size_t)w_total * 8));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- streaming VAD (chunk loop of speech_transformers.py:710-746) -----------------------------
static int vs_collect(b2_ctx* h, b2_ctx::VadStream::Slot& sl) {
  if (!sl.busy) return B2_OK;
  B2_CUDA(h, cudaEventSynchronize(sl.ev));
  h->vs.results.insert(h->vs.results.end(), sl.hout, sl.hout + sl.n_out);
  sl.busy = false;
  return B2_OK;
}

extern "C" int b2_vad_stream_begin(b2_handle h, int frame_rate, int sample_rate, float non_speech_label,
                                   int64_t energy_threshold, int z_lo, int z_hi) {
  B2_ENTER(h);
  auto& vs = h->vs;
  if (vs.active) B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: already open on this handle");
  const int fpw = b2_vad_frames_per_window(frame_rate, sample_rate);
  if (fpw <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: bad frame_rate/sample_rate");
  if (energy_threshold < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: negative energy threshold");
  vs.frame_rate = frame_rate;
  vs.sample_rate = sample_rate;
  vs.fpw = fpw;
  vs.label = non_speech_label;
  vs.thr = energy_threshold;
  vs.z_lo = z_lo < 0 ? 0 : z_lo;
  vs.z_hi = z_hi < 0 ? (3 * fpw) / 8 : z_hi;
  vs.windows = 0;
  vs.seq = 0;
  vs.results.clear();
  vs.active = true;
  return B2_OK;
}

extern "C" int b2_vad_stream_push(b2_handle h, const void* pcm_bytes, int64_t n_bytes) {
  B2_ENTER(h);
  auto& vs = h->vs;
  if (!vs.active) B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: not open");
  if (n_bytes < 0 || (n_bytes && !pcm_bytes)) B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: bad chunk");
  const int64_t n = n_bytes / 2;  // an odd trailing byte is ignored (speech_transformers.py:745)
  if (n == 0) return B2_OK;
  const int64_t nwin = (n + vs.fpw - 1) / vs.fpw;
  auto& sl = vs.slot[vs.seq % b2_ctx::VadStream::kSlots];
  B2_TRY(vs_collect(h, sl));  // the slot's previous chunk (kSlots pushes ago) must be done
  if ((size_t)n * 2 > sl.cap) {
    if (sl.hp) B2_CUDA(h, cudaFreeHost(sl.hp));
    if (sl.dp) B2_CUDA(h, cudaFree(sl.dp));
    sl.hp = sl.dp = nullptr;
    sl.cap = 0;
    const size_t want = (size_t)n * 2 + 256;
    B2_CUDA(h, cudaMallocHost(&sl.hp, want));
    B2_CUDA(h, cudaMalloc(&sl.dp, want));
    sl.cap = want;
  }
  if ((size_t)nwin * 4 > sl.out_cap) {
    if (sl.hout) B2_CUDA(h, cudaFreeHost(sl.hout));
    if (sl.dout) B2_CUDA(h, cudaFree(sl.dout));
    sl.hout = sl.dout = nullptr;
    sl.out_cap = 0;
    const size_t want = (size_t)nwin * 4 + 256;
    B2_CUDA(h, cudaMallocHost((void**)&sl.hout, want));
    B2_CUDA(h, cudaMalloc((void**)&sl.dout, want));
    sl.out_cap = want;
  }
  if (!sl.ev) B2_CUDA(h, cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming));
  memcpy(sl.hp, pcm_bytes, (size_t)n * 2);
  B2_CUDA(h, cudaMemcpyAsync(sl.dp, sl.hp, (size_t)n * 2, cudaMemcpyHostToDevice, h->stream));
  const int64_t pcm_off[2] = {0, n}, out_off[2] = {0, nwin};
  B2_TRY(b2i_vad_launch(h, (const int16_t*)sl.dp, pcm_off, 1, vs.fpw, vs.label, (int64_t)vs.fpw * vs.thr,
                        vs.z_lo, vs.z_hi, sl.dout, out_off));
  B2_CUDA(h, cudaMemcpyAsync(sl.hout, sl.dout, (size_t)nwin * 4, cudaMemcpyDeviceToHost, h->stream));
  B2_CUDA(h, cudaEventRecord(sl.ev, h->stream));
  sl.n_out = nwin;
  sl.busy = true;
  vs.windows += nwin;
  ++vs.seq;
  return B2_OK;
}

extern "C" int64_t b2_vad_stream_windows(b2_handle h) { return (h && h->vs.active) ? h->vs.windows : -1; }

extern "C" int b2_vad_stream_end(b2_handle h, float* out, int64_t capacity, int64_t* n_out) {
  B2_ENTER(h);
  auto& vs = h->vs;
  if (!vs.active) B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: not open");
  const int ns = b2_ctx::VadStream::kSlots;
  for (uint64_t i = vs.seq > (uint64_t)ns ? vs.seq - ns : 0; i < vs.seq; ++i)  // oldest first
    B2_TRY(vs_collect(h, vs.slot[i % ns]));
  vs.active = false;
  const int64_t total = (int64_t)vs.results.size();
  if (n_out) *n_out = total;
  if (total > capacity || (total && !out)) {
    vs.results.clear();
    B2_FAIL(h, B2_ERR_BAD_ARG, "vad stream: output holds %lld windows, capacity %lld", (long long)total,
            (long long)capacity);
  }
  if (total) memcpy(out, vs.results.data(), (size_t)total * 4);
  vs.results.clear();
  return B2_OK;
}

extern "C" int b2_synth_pcm(b2_handle h, const uint8_t* window_class, int64_t n_windows, int fpw,
                            uint32_t seed, int16_t* pcm_out, int memspace) {
  B2_ENTER(h);
  if (n_windows < 0 || fpw <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "synth: bad sizes");
  if (n_windows == 0) return B2_OK;
  if (!window_class || !pcm_out) B2_FAIL(h, B2_ERR_BAD_ARG, "synth: null pointer");
  const uint8_t* d_cls = window_class;
  int16_t* d_out = pcm_out;
  size_t out_bytes = (size_t)n_windows * fpw * 2;
  if (memspace == B2_HOST) {
    void *dp, *dq;
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, window_class, (size_t)n_windows, &dp));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, out_bytes, &dq));
    d_cls = (const uint8_t*)dp;
    d_out = (int16_t*)dq;
  }
  B2_TRY(b2i_synth_launch(h, d_cls, n_windows, fpw, seed, d_out));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, pcm_out, d_out, out_bytes));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- rasteriser ----------------------------------------------------------------------------
extern "C" int b2_rasterize_lengths(const double* cue_end_s, const int64_t* cue_off, int B,
                                    const double* ratios, int K, int per_pair_ratios,
                                    int sample_rate, int64_t* lengths) {
  return rasterize_lengths(nullptr, cue_end_s, cue_off, B, ratios, K, per_pair_ratios, sample_rate, lengths);
}

extern "C" int b2_rasterize(b2_handle h, const double* cue_start_s, const double* cue_end_s,
                            const uint8_t* cue_keep, const int64_t* cue_off, int B,
                            const double* ratios, int K, int per_pair_ratios,
                            const double* levels, int sample_rate, double start_seconds,
                            float* out, const int64_t* out_off, int memspace) {
  B2_ENTER(h);
  if (B < 0 || K < 0 || !cue_off || !out_off || sample_rate <= 0)
    B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize: bad arguments");
  if (B == 0 || K == 0) return B2_OK;
  if (!ratios || (cue_off[B] && (!cue_start_s || !cue_end_s)))
    B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize: null cue/ratio arrays");
  int64_t at;
  double val;
  if (const char* why = bad_cue_input(cue_start_s, cue_end_s, cue_off, B, ratios, K, per_pair_ratios,
                                      start_seconds, &at, &val))
    B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize: %s (index %lld: %g)", why, (long long)at, val);
  int64_t total = out_off[(size_t)B * K];
  if (total && !out) B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize: null output");
  float* d_out = out;
  if (memspace == B2_HOST) {
    void* dq;
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)total * 4 + 16, &dq));
    d_out = (float*)dq;
  }
  B2_TRY(b2i_raster_launch(h, cue_start_s, cue_end_s, cue_keep, cue_off, B, ratios, K,
                           per_pair_ratios, levels, sample_rate, start_seconds, d_out, out_off));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, out, d_out, (size_t)total * 4));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- fused-VAD blend -------------------------------------------------------------------------
extern "C" int b2_blend_signals(b2_handle h, const float* a, const float* b, int64_t n, int mode,
                                double wa, double wb, float* out, int memspace) {
  B2_ENTER(h);
  if (n < 0 || mode < 0 || mode > 2) B2_FAIL(h, B2_ERR_BAD_ARG, "blend: bad arguments");
  if (n == 0) return B2_OK;
  if (!a || !b || !out) B2_FAIL(h, B2_ERR_BAD_ARG, "blend: null pointer");
  const float *d_a = a, *d_b = b;
  float* d_out = out;
  if (memspace == B2_HOST) {
    void *da, *db, *dq;
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, a, (size_t)n * 4, &da));
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN1, b, (size_t)n * 4, &db));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)n * 4, &dq));
    d_a = (const float*)da;
    d_b = (const float*)db;
    d_out = (float*)dq;
  }
  B2_TRY(b2i_blend_launch(h, d_a, d_b, n, mode, wa, wb, d_out));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, out, d_out, (size_t)n * 4));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- boundaries ----------------------------------------------------------------------------
extern "C" int b2_first_last_nonzero(b2_handle h, const float* sig, const int64_t* sig_off, int n,
                                     int64_t* first, int64_t* last, int memspace) {
  B2_ENTER(h);
  if (n < 0 || !sig_off || !first || !last) B2_FAIL(h, B2_ERR_BAD_ARG, "boundaries: bad arguments");
  if (n == 0) return B2_OK;
  const float* d_sig = sig;
  int64_t *d_first = first, *d_last = last;
  if (memspace == B2_HOST) {
    void *dp, *dq;
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, sig, (size_t)sig_off[n] * 4, &dp));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)n * 16, &dq));
    d_sig = (const float*)dp;
    d_first = (int64_t*)dq;
    d_last = d_first + n;
  }
  B2_TRY(b2i_bounds_launch(h, d_sig, sig_off, n, d_first, d_last));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, first, d_first, (size_t)n * 8));
    B2_TRY(copy_out(h, last, d_last, (size_t)n * 8));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- aligner -------------------------------------------------------------------------------
extern "C" int b2_align_batch(b2_handle h, const float* ref, const int64_t* ref_off,
                              const float* sub, const int64_t* sub_off, int B, int K,
                              int64_t max_offset_samples, double* score, int32_t* offset,
                              int32_t* status, int memspace) {
  B2_ENTER(h);
  if (B < 0 || K < 0 || !ref_off || !sub_off) B2_FAIL(h, B2_ERR_BAD_ARG, "align: bad arguments");
  if (B == 0 || K == 0) return B2_OK;
  if (!score || !offset || !status) B2_FAIL(h, B2_ERR_BAD_ARG, "align: null output");
  size_t J = (size_t)B * K;
  B2_CHECK_DEV(h, memspace, ref, "align: ref");
  B2_CHECK_DEV(h, memspace, sub, "align: sub");
  B2_CHECK_DEV(h, memspace, score, "align: score");
  const float *d_ref = ref, *d_sub = sub;
  double* d_score = score;
  int32_t *d_offset = offset, *d_status = status;
  if (memspace == B2_HOST) {
    void *dr, *ds, *dq;
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, ref, (size_t)ref_off[B] * 4, &dr));
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN1, sub, (size_t)sub_off[J] * 4, &ds));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, J * 16 + 64, &dq));
    d_ref = (const float*)dr;
    d_sub = (const float*)ds;
    d_score = (double*)dq;
    d_offset = (int32_t*)(d_score + J);
    d_status = d_offset + J;
  }
  B2_TRY(b2i_align_launch(h, d_ref, ref_off, B, /*trk_off=*/nullptr, d_sub, sub_off, B, K, max_offset_samples,
                          d_score, d_offset, d_status, /*winner_only=*/0, /*cue_src=*/nullptr, /*capture_j0=*/0));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, score, d_score, J * 8));
    B2_TRY(copy_out(h, offset, d_offset, J * 4));
    B2_TRY(copy_out(h, status, d_status, J * 4));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

extern "C" int b2_capture_nominations(b2_handle h, float* scores, int64_t stride, int64_t* win, float* stat,
                                      int32_t* cand) {
  B2_ENTER(h);
  h->capture = B2Capture{};
  if (!scores) return B2_OK;
  if (stride <= 0 || !win || !stat || !cand) B2_FAIL(h, B2_ERR_BAD_ARG, "capture: bad arguments");
  B2_TRY(check_device_ptr(h, scores, "capture: scores"));
  B2_TRY(check_device_ptr(h, win, "capture: win"));
  B2_TRY(check_device_ptr(h, stat, "capture: stat"));
  B2_TRY(check_device_ptr(h, cand, "capture: cand"));
  h->capture = B2Capture{scores, (long long)stride, (long long*)win, stat, cand};
  return B2_OK;
}

extern "C" int b2_reduce_ratios(b2_handle h, const double* score, const int32_t* offset,
                                const int32_t* status, int B, int K, int64_t max_offset_samples,
                                double* best_score, int32_t* best_offset, int32_t* best_k,
                                int memspace) {
  B2_ENTER(h);
  if (B < 0 || K <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "reduce: bad arguments");
  if (B == 0) return B2_OK;
  if (!score || !offset || !best_score || !best_offset || !best_k)
    B2_FAIL(h, B2_ERR_BAD_ARG, "reduce: null pointer");
  size_t J = (size_t)B * K;
  const double* d_score = score;
  const int32_t *d_offset = offset, *d_status = status;
  double* d_bs = best_score;
  int32_t *d_bo = best_offset, *d_bk = best_k;
  if (memspace == B2_HOST) {
    void *d0, *dq;
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_IN0, J * 16 + 64, &d0));
    B2_CUDA(h, cudaMemcpyAsync(d0, score, J * 8, cudaMemcpyHostToDevice, h->stream));
    int32_t* doff = (int32_t*)((char*)d0 + J * 8);
    B2_CUDA(h, cudaMemcpyAsync(doff, offset, J * 4, cudaMemcpyHostToDevice, h->stream));
    int32_t* dst = doff + J;
    if (status)
      B2_CUDA(h, cudaMemcpyAsync(dst, status, J * 4, cudaMemcpyHostToDevice, h->stream));
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)B * 16 + 64, &dq));
    d_score = (const double*)d0;
    d_offset = doff;
    d_status = status ? dst : nullptr;
    d_bs = (double*)dq;
    d_bo = (int32_t*)(d_bs + B);
    d_bk = d_bo + B;
  }
  B2_TRY(b2i_reduce_launch(h, d_score, d_offset, d_status, B, K, max_offset_samples, d_bs, d_bo,
                           d_bk));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, best_score, d_bs, (size_t)B * 8));
    B2_TRY(copy_out(h, best_offset, d_bo, (size_t)B * 4));
    B2_TRY(copy_out(h, best_k, d_bk, (size_t)B * 4));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return B2_OK;
}

// ---- whole hot path --------------------------------------------------------------------------
// VideoSpeechTransformer.fit (VAD) -> K x (SubtitleScaler + SubtitleSpeechTransformer) ->
// MaxScoreAligner(FFTAligner).fit_transform (ffsubsync/ffsubsync.py:637,196-235), for V videos and T
// subtitle tracks: track t is synced against video track_video[t] (non-decreasing; NULL: V == T, track t
// against video t - b2_sync_batch).  Each video's PCM goes through the VAD once; its reference spectra
// serve the K ratio jobs t*K + k of every one of its tracks.
// The detector is this package's energy / zero-crossing VAD, or the reference's auditok detector
// (b2_vad_auditok's arguments; its float64 signal rounded once to float32 is the reference signal).  With
// subtitle references (b2_sync_tracks_subs) the videos that have one take it instead.  Each entry point fills
// one SyncRequest; plan_sync (sync_plan.h) checks it and builds the host tables, and sync_run below runs the
// plan.

// The device buffers one call reads and writes
struct SyncBufs {
  const int16_t* pcm;
  float* refsig;
  float* subsig;           // float subtitle signals (unfused raster only)
  double* score;           // [T*K] per-ratio results: the caller's all_* on B2_DEVICE without the search
  int32_t* offset;
  int32_t* status;
  double* bs;              // [T] reduced results: the caller's on B2_DEVICE
  int32_t* bo;
  int32_t* bk;
  double* g_all_score;     // GSS outputs: the caller's on B2_DEVICE, staged otherwise
  int32_t* g_all_offset;
  double* g_ratio;
  double* g_evals;
  bool fused;
  int winner_only;
};

// rasterise (float signals only if !fused) -> align -> reduce the tracks of the videos [v0, v1) on the
// caller's stream, then the GSS rounds with the search
static int enqueue_chain(b2_ctx* h, const SyncRequest& r, const SyncPlan& p, const SyncBufs& b, int v0, int v1,
                         bool ref_packed) {
  const int K = r.K, t0 = p.trk_off[v0], nt = p.trk_off[v1] - t0;
  const size_t j0 = (size_t)t0 * K;
  std::vector<int> chain_trk(v1 - v0 + 1);
  for (int v = v0; v <= v1; ++v) chain_trk[v - v0] = p.trk_off[v] - t0;
  if (!b.fused)
    B2_TRY(b2i_raster_launch(h, r.cue_start_s, r.cue_end_s, r.cue_keep, r.cue_off + t0, nt, r.ratios, K, 0, nullptr,
                             r.sample_rate, r.start_seconds, b.subsig, p.sub_off.data() + j0));
  const B2CueSource src{r.cue_start_s, r.cue_end_s, r.cue_keep, r.cue_off + t0, r.ratios, r.sample_rate,
                        r.start_seconds, p.ref_label, p.two_level, ref_packed};
  B2_TRY(b2i_align_launch(h, b.refsig, p.ref_off.data() + v0, v1 - v0, chain_trk.data(), b.subsig,
                          p.sub_off.data() + j0, nt, K, r.max_offset_samples, b.score + j0, b.offset + j0,
                          b.status + j0, b.winner_only, b.fused ? &src : nullptr, (long long)j0));
  B2_TRY(b2i_reduce_launch(h, b.score + j0, b.offset + j0, b.status + j0, nt, K, r.max_offset_samples, b.bs + t0,
                           b.bo + t0, b.bk + t0));
  if (!p.gss || nt == 0) return B2_OK;
  const size_t a0 = (size_t)t0 * (K + 1);
  const B2GssOut go{b.bs + t0, b.bo + t0, b.bk + t0, b.score + j0, b.offset + j0,
                    b.g_all_score ? b.g_all_score + a0 : nullptr, b.g_all_offset ? b.g_all_offset + a0 : nullptr,
                    b.g_ratio + t0, b.g_evals ? b.g_evals + (size_t)t0 * kGssEvals : nullptr};
  return b2i_gss_launch(h, b.refsig, p.ref_off.data() + v0, v1 - v0, chain_trk.data(), K, src,
                        p.max_end.data() + t0, r.max_offset_samples, go);
}

// The detector step of the videos [v0, v1), on whichever stream the handle launches on: the energy / ZCR VAD
// into the reference-signal buffer, or for auditok the energy pass over the videos' chunks (label 0, every
// crossing count accepted, a short last block judged on its own samples) writing its 0/1 flags there, then
// the tokenizer turning each chunk's flags into its float32 signal in place.  Both auditok launches take a
// metadata arena from the ring of the stream they run on; on the pipeline's internal stream that ring is its
// own, so the GSS invariant (no later arena of a chain recycles the chain's arena, runcorr.cu b2i_gss_launch)
// holds as before: the chains' arenas come from the caller-facing ring, and with one sub-batch the detector's
// arenas there precede the chain's.
// With subtitle references (b2_sync_tracks_subs) the step also rasterises those of the videos [v0, v1) into
// their ranges, on the same stream: the detector never writes there (no PCM: no tiles, no tokenizer chunk), and
// the step stays the buffer's only writer, so the pipeline and resident chaining need nothing new.
static int detect(b2_ctx* h, const SyncRequest& r, const SyncPlan& p, const SyncBufs& b, int v0, int v1,
                  bool ref_packed) {
  if (!p.auditok) {
    B2_TRY(b2i_vad_launch(h, b.pcm, r.pcm_off + v0, v1 - v0, p.fpw, r.energy.non_speech_label,
                          (int64_t)p.fpw * r.energy.energy_threshold, p.z_lo, p.z_hi, b.refsig, p.ref_off.data() + v0,
                          nullptr, ref_packed));
  } else {
    const ChunkTable& ch = p.ch;
    const int c0 = ch.first[v0], nc = ch.first[v1] - c0;
    B2_TRY(b2i_vad_launch(h, b.pcm, ch.pcm.data() + c0, nc, p.fpw, 0.0f, p.auditok_e_min, 0, p.fpw, b.refsig,
                          ch.out.data() + c0, ch.tail.data() + c0));
    if (!p.any_subs) return b2i_tokenize_inplace_launch(h, b.refsig, ch.out.data() + c0, nc, p.tok);
    const int k0 = ch.tok_first[v0];
    B2_TRY(b2i_tokenize_inplace_launch(h, b.refsig, ch.tok_off.data() + k0, ch.tok_first[v1] - k0, p.tok,
                                       ch.tok_end.data() + k0));
  }
  if (!p.any_subs) return B2_OK;
  const auto& sv = p.sub_video;
  const int s0 = (int)(std::lower_bound(sv.begin(), sv.end(), v0) - sv.begin());
  const int s1 = (int)(std::lower_bound(sv.begin(), sv.end(), v1) - sv.begin());
  if (s1 == s0) return B2_OK;
  std::vector<int> rel(sv.begin() + s0, sv.begin() + s1);
  for (int& v : rel) v -= v0;
  return b2i_raster_ref_launch(h, r.refs.cue_start_s, r.refs.cue_end_s, r.refs.cue_keep, r.refs.cue_off + v0,
                               p.ref_off.data() + v0, v1 - v0, rel.data(), (int)rel.size(), r.sample_rate,
                               r.start_seconds, b.refsig);
}

// Software pipeline over the plan's sub-batches of videos (sync_plan.h plan_cuts).  The VAD (HBM-bound) of every
// sub-batch is queued on the internal high-priority stream: sub-batch 0 on the whole GPU, the later ones on
// `vad_sms` SMs only (one lane-per-window CTA per SM, csrc/vad.cu); the rasterisation / correlation / reduction
// of the tracks of sub-batch i (FP32- and shared-memory bound) follows on the caller's stream as soon as its VAD
// is done and runs on the SMs the VAD leaves free - a VAD CTA owns its SM's shared memory, so the block scheduler
// keeps the two apart.  Needs the lane-per-window kernel (1.3 instructions per byte: ~80 GB/s per SM); the
// lane-group kernel needs every SM's issue slots to reach the HBM roofline, so partitioning never paid with it.
// B2_DEVICE_RESIDENT, previous entry point on this handle = a pipelined resident b2_sync_batch or b2_sync_tracks
// (`chained`): the VAD starts behind that call's fence (everything on the caller's stream up to, not including,
// its last correlation chain) and overlaps that chain like a further sub-batch - on vad_sms SMs if it is still
// running.  It writes the other reference-signal buffer (the chain still reads the previous one); the chains of
// the call before that, which read this buffer, precede the fence.
static int run_pipeline(b2_ctx* h, const SyncRequest& r, const SyncPlan& p, const SyncBufs& b, bool resident,
                        bool chained, int refsig_slot) {
  const int n_sub = p.n_sub;
  const std::vector<int>& cut = p.cut;
  if (n_sub == 1) {
    B2_TRY(detect(h, r, p, b, 0, r.V, p.ref_packed[0]));
    return enqueue_chain(h, r, p, b, 0, r.V, p.ref_packed[0]);
  }
  std::vector<cudaEvent_t> vad_done(n_sub);
  cudaEvent_t inputs_ready = next_event(h);
  B2_CUDA(h, cudaEventRecord(inputs_ready, h->stream));
  // B2_PIPE_TRACE=1 (diagnostic; synchronises): device timeline of the sub-batches and host enqueue times
  const bool trace = getenv("B2_PIPE_TRACE") != nullptr;
  std::vector<cudaEvent_t> tev;   // t0, then per sub-batch: VAD start, VAD end, chain start, chain end
  std::vector<double> host_ms(n_sub + 1, 0.0);
  const auto host_t0 = std::chrono::steady_clock::now();
  auto host_now = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count(); };
  if (trace) {
    tev.resize(1 + 4 * (size_t)n_sub);
    for (auto& e : tev) B2_CUDA(h, cudaEventCreate(&e));
    B2_CUDA(h, cudaEventRecord(tev[0], h->stream));
  }
  bool prev_busy = false;
  if (chained) {
    prev_busy = cudaEventQuery(h->resident_done) == cudaErrorNotReady;
    cudaGetLastError();
  }
  {
    Stream2Scope on2(h);
    B2_CUDA(h, cudaStreamWaitEvent(h->stream, chained ? h->resident_fence : inputs_ready, 0));
    for (int i = 0; i < n_sub; ++i) {
      h->vad_partition_sms = (i > 0 || prev_busy) ? p.vad_sms : 0;
      if (trace) B2_CUDA(h, cudaEventRecord(tev[1 + 4 * i], h->stream));
      const int st = detect(h, r, p, b, cut[i], cut[i + 1], p.ref_packed[i]);
      h->vad_partition_sms = 0;
      if (st != B2_OK) return st;
      vad_done[i] = next_event(h);
      B2_CUDA(h, cudaEventRecord(vad_done[i], h->stream));
      if (trace) B2_CUDA(h, cudaEventRecord(tev[2 + 4 * i], h->stream));
    }
  }
  host_ms[0] = host_now();
  for (int i = 0; i < n_sub; ++i) {
    if (resident && i == n_sub - 1) B2_CUDA(h, cudaEventRecord(h->resident_fence, h->stream));
    B2_CUDA(h, cudaStreamWaitEvent(h->stream, vad_done[i], 0));
    if (trace) B2_CUDA(h, cudaEventRecord(tev[3 + 4 * i], h->stream));
    B2_TRY(enqueue_chain(h, r, p, b, cut[i], cut[i + 1], p.ref_packed[i]));
    if (trace) B2_CUDA(h, cudaEventRecord(tev[4 + 4 * i], h->stream));
    host_ms[i + 1] = host_now();
  }
  if (resident) {
    B2_CUDA(h, cudaEventRecord(h->resident_done, h->stream));
    h->refsig_parity = refsig_slot == b2_ctx::WS_SIG_REF2 ? 1 : 0;
    h->resident_fence_valid = true;
  }
  if (trace) {
    B2_CUDA(h, cudaStreamSynchronize(h->stream2));
    B2_CUDA(h, cudaStreamSynchronize(h->stream));
    auto at = [&](size_t k) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, tev[0], tev[k]);
      return ms;
    };
    fprintf(stderr, "[b2 pipe] V=%d T=%d n_sub=%d vad_sms=%d chained=%d prev_busy=%d; host: VADs enqueued at %.3f ms\n",
            r.V, r.T, n_sub, p.vad_sms, (int)chained, (int)prev_busy, host_ms[0]);
    for (int i = 0; i < n_sub; ++i)
      fprintf(stderr, "[b2 pipe]  sub %d videos %4d..%4d  VAD %7.3f -> %7.3f ms   chain %7.3f -> %7.3f ms   host enqueued chain at %.3f ms\n",
              i, cut[i], cut[i + 1], at(1 + 4 * i), at(2 + 4 * i), at(3 + 4 * i), at(4 + 4 * i), host_ms[i + 1]);
    for (auto& e : tev) cudaEventDestroy(e);
  }
  return B2_OK;
}

static int sync_run(b2_ctx* h, bool fence_was_valid, const SyncRequest& r) {
  SyncPlan p;
  SyncPipeEnv env{h->sm_count, b2_ctx::kEvents - 2, getenv("B2_SUBBATCHES"), getenv("B2_VAD_SMS"),
                  b2i_vad_lane_eligible};
  env.quirk_mask = h->log2_quirk_mask;
  env.capture = h->capture.scores != nullptr;
  env.align_path = getenv("B2_ALIGN_PATH");
  env.fused = true;
  if (const char* e = getenv("B2_FUSED_RASTER")) env.fused = atoi(e) != 0;
  env.ref_packed = getenv("B2_REF_PACKED");
  if (const int st = plan_sync(r, env, &p)) {
    h->err = p.err;
    return st;
  }
  const int T = r.T, K = r.K;
  if (T == 0) return B2_OK;
  const bool resident = r.memspace == B2_DEVICE_RESIDENT;
  const int memspace = resident ? B2_DEVICE : r.memspace;
  // every bulk pointer of a B2_DEVICE call, before anything is launched
  const char* prefix = r.track_video ? "sync_tracks" : "sync_batch";
  const std::pair<const void*, const char*> bulk[] = {{r.pcm, "pcm"}, {r.best_score, "best_score"},
                                                      {r.best_offset, "best_offset"}, {r.best_k, "best_k"},
                                                      {r.all_score, "all_score"}, {r.all_offset, "all_offset"}};
  for (const auto& [ptr, name] : bulk) {
    char what[64];
    snprintf(what, sizeof(what), "%s: %s", prefix, name);
    B2_CHECK_DEV(h, memspace, ptr, what);
  }
  if (p.gss) {
    B2_CHECK_DEV(h, memspace, r.gss_ratio, "sync_tracks_gss: gss_ratio");
    B2_CHECK_DEV(h, memspace, r.gss_evals, "sync_tracks_gss: gss_evals");
  }
  // Default: the K subtitle signals of a track are never materialised as floats - the cue list is
  // rasterised into bit masks (1 bit per frame) that the correlation kernel and the exact re-score
  // read.  B2_FUSED_RASTER=0 (A/B and test knob): raster_cues_kernel writes float signals to HBM and
  // the generic aligner (the b2_align_batch path) reads them back.
  SyncBufs b{};
  b.fused = env.fused;
  const size_t J = (size_t)T * K, JG = (size_t)T * (K + 1);
  void *d_refsig, *d_subsig = nullptr, *d_res;
  // a chained resident call writes the buffer the previous call is not reading any more
  const bool chained = resident && fence_was_valid;
  const int refsig_slot = chained && h->refsig_parity == 0 ? b2_ctx::WS_SIG_REF2 : b2_ctx::WS_SIG_REF;
  B2_TRY(b2i_ws(h, refsig_slot, (size_t)p.ref_off[r.V] * 4 + 64, &d_refsig));
  if (!b.fused) B2_TRY(b2i_ws(h, b2_ctx::WS_SIG_SUB, (size_t)p.sub_off[J] * 4 + 64, &d_subsig));
  B2_TRY(b2i_ws(h, b2_ctx::WS_MISC, J * 16 + (size_t)T * 16 + 256, &d_res));
  double* d_score = (double*)d_res;
  double* d_bs = d_score + J;
  int32_t* d_offset = (int32_t*)(d_bs + T);
  int32_t* d_status = d_offset + J;
  int32_t* d_bo = d_status + J;
  int32_t* d_bk = d_bo + T;
  b.refsig = (float*)d_refsig;
  b.subsig = (float*)d_subsig;
  b.status = d_status;
  // GSS: the grid's per-ratio results stay in the workspace (all_* then hold K + 1 columns, written by the
  // combine); host calls stage the GSS outputs in a second workspace
  b.g_ratio = r.gss_ratio;
  b.g_evals = r.gss_evals;
  if (p.gss) {
    void* d_go;
    B2_TRY(b2i_ws(h, b2_ctx::WS_GSS_OUT, JG * 12 + (size_t)T * 8 * (1 + kGssEvals) + 256, &d_go));
    double* hs = (double*)d_go;
    double* hr = hs + JG;
    double* he = hr + T;
    int32_t* ho = (int32_t*)(he + (size_t)T * kGssEvals);
    b.g_all_score = r.all_score ? (memspace == B2_DEVICE ? r.all_score : hs) : nullptr;
    b.g_all_offset = r.all_offset ? (memspace == B2_DEVICE ? r.all_offset : ho) : nullptr;
    if (memspace != B2_DEVICE) {
      b.g_ratio = hr;
      b.g_evals = r.gss_evals ? he : nullptr;
    }
  }
  b.pcm = r.pcm;
  if (memspace == B2_HOST) {   // a call without audio samples reads no PCM (b2_sync_tracks_subs may pass none)
    void* dp = nullptr;
    if (p.audio_samples > 0) B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, r.pcm, (size_t)r.pcm_off[r.V] * 2, &dp));
    b.pcm = (const int16_t*)dp;
  }
  const bool dev = memspace == B2_DEVICE;
  b.score = (dev && r.all_score && !p.gss) ? r.all_score : d_score;
  b.offset = (dev && r.all_offset && !p.gss) ? r.all_offset : d_offset;
  b.bs = dev ? r.best_score : d_bs;
  b.bo = dev ? r.best_offset : d_bo;
  b.bk = dev ? r.best_k : d_bk;
  // only the best ratio of each track is reported unless the per-ratio arrays are requested:
  // ratios that cannot win even after the round-off bound tau are then not re-scored exactly (B2_ALIGN_APPROX)
  b.winner_only = (!r.all_score && !r.all_offset) ? 1 : 0;
  B2_TRY(run_pipeline(h, r, p, b, resident, chained, refsig_slot));
  if (dev) return B2_OK;
  B2_TRY(copy_out(h, r.best_score, d_bs, (size_t)T * 8));
  B2_TRY(copy_out(h, r.best_offset, d_bo, (size_t)T * 4));
  B2_TRY(copy_out(h, r.best_k, d_bk, (size_t)T * 4));
  if (p.gss) {
    if (r.all_score) B2_TRY(copy_out(h, r.all_score, b.g_all_score, JG * 8));
    if (r.all_offset) B2_TRY(copy_out(h, r.all_offset, b.g_all_offset, JG * 4));
    B2_TRY(copy_out(h, r.gss_ratio, b.g_ratio, (size_t)T * 8));
    if (r.gss_evals) B2_TRY(copy_out(h, r.gss_evals, b.g_evals, (size_t)T * kGssEvals * 8));
  } else {
    if (r.all_score) B2_TRY(copy_out(h, r.all_score, d_score, J * 8));
    if (r.all_offset) B2_TRY(copy_out(h, r.all_offset, d_offset, J * 4));
  }
  B2_CUDA(h, cudaStreamSynchronize(h->stream));
  return B2_OK;
}

extern "C" int b2_sync_batch(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int B,
                             int frame_rate, int sample_rate, float non_speech_label,
                             int64_t energy_threshold, int z_lo, int z_hi,
                             const double* cue_start_s, const double* cue_end_s,
                             const uint8_t* cue_keep, const int64_t* cue_off, const double* ratios,
                             int K, double start_seconds, int64_t max_offset_samples,
                             double* best_score, int32_t* best_offset, int32_t* best_k,
                             double* all_score, int32_t* all_offset, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_batch");
  const SyncRequest r{"sync_batch", pcm, pcm_off, B, nullptr, B, frame_rate, sample_rate, B2_DETECTOR_ENERGY_ZCR,
                      {non_speech_label, energy_threshold, z_lo, z_hi}, {}, {},
                      cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                      best_score, best_offset, best_k, all_score, all_offset, false, nullptr, nullptr, memspace};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_sync_tracks(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                              const int32_t* track_video, int T, int frame_rate, int sample_rate,
                              float non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                              const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                              const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                              int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                              int32_t* best_k, double* all_score, int32_t* all_offset, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks: null track_video");
  const SyncRequest r{"sync_tracks", pcm, pcm_off, V, track_video, T, frame_rate, sample_rate, B2_DETECTOR_ENERGY_ZCR,
                      {non_speech_label, energy_threshold, z_lo, z_hi}, {}, {},
                      cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                      best_score, best_offset, best_k, all_score, all_offset, false, nullptr, nullptr, memspace};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_sync_tracks_gss(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                                  const int32_t* track_video, int T, int frame_rate, int sample_rate,
                                  float non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                                  const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                                  const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                                  int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                                  int32_t* best_k, double* all_score, int32_t* all_offset, double* gss_ratio,
                                  double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks_gss");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_gss: null track_video");
  const SyncRequest r{"sync_tracks_gss", pcm, pcm_off, V, track_video, T, frame_rate, sample_rate,
                      B2_DETECTOR_ENERGY_ZCR, {non_speech_label, energy_threshold, z_lo, z_hi}, {}, {},
                      cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                      best_score, best_offset, best_k, all_score, all_offset, true, gss_ratio, gss_evals, memspace};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_sync_tracks_auditok(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                                      const int32_t* track_video, int T, int frame_rate, int sample_rate,
                                      double non_speech_label, double energy_threshold_db, double min_length,
                                      int64_t max_length, double max_continuous_silence, int64_t chunk_samples,
                                      const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                                      const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                                      int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                                      int32_t* best_k, double* all_score, int32_t* all_offset, double* gss_ratio,
                                      double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks_auditok");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_auditok: null track_video");
  if (!gss_ratio && gss_evals) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_auditok: gss_evals without gss_ratio");
  const SyncRequest r{gss_ratio ? "sync_tracks_auditok (search)" : "sync_tracks_auditok", pcm, pcm_off, V, track_video,
                      T, frame_rate, sample_rate, B2_DETECTOR_AUDITOK, {},
                      {non_speech_label, energy_threshold_db, min_length, max_continuous_silence, max_length,
                       chunk_samples},
                      {}, cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                      best_score, best_offset, best_k, all_score, all_offset, gss_ratio != nullptr, gss_ratio, gss_evals,
                      memspace};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_sync_tracks_subs(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                                   const int32_t* track_video, int T, int frame_rate, int sample_rate, int detector,
                                   double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                                   double energy_threshold_db, double min_length, int64_t max_length,
                                   double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs,
                                   const double* ref_cue_start_s, const double* ref_cue_end_s,
                                   const uint8_t* ref_cue_keep, const int64_t* ref_cue_off,
                                   const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                                   const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                                   int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                                   int32_t* best_k, double* all_score, int32_t* all_offset, double* gss_ratio,
                                   double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks_subs");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_subs: null track_video");
  if (!gss_ratio && gss_evals) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_subs: gss_evals without gss_ratio");
  if (V > 0 && (!pcm_off || !ref_cue_off)) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_subs: null pcm_off / ref_cue_off");
  if (detector != B2_DETECTOR_ENERGY_ZCR && detector != B2_DETECTOR_AUDITOK)
    B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_subs: detector must be B2_DETECTOR_ENERGY_ZCR or B2_DETECTOR_AUDITOK, "
            "not %d", detector);
  static const int64_t no_cues[1] = {0};
  const SyncRequest r{gss_ratio ? "sync_tracks_subs (search)" : "sync_tracks_subs", pcm, pcm_off, V, track_video, T,
                      frame_rate, sample_rate, detector, {(float)non_speech_label, energy_threshold, z_lo, z_hi},
                      {non_speech_label, energy_threshold_db, min_length, max_continuous_silence, max_length,
                       chunk_samples},
                      {ref_is_subs, ref_cue_start_s, ref_cue_end_s, ref_cue_keep, V > 0 ? ref_cue_off : no_cues},
                      cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                      best_score, best_offset, best_k, all_score, all_offset, gss_ratio != nullptr, gss_ratio, gss_evals,
                      memspace};
  return sync_run(h, _b2_fence_was_valid, r);
}
