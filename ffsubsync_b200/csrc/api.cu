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
#include "ingest_plan.h"
#include "sync_plan.h"
#include "sync_output.cuh"
#include "speech_out.cuh"

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

static void ingest_free(b2_ctx* h);

extern "C" int b2_destroy(b2_handle h) {
  if (!h) return B2_OK;
  DeviceScope scope(h->device);
  if (h->stream2) cudaStreamSynchronize(h->stream2);
  cudaStreamSynchronize(h->stream);
  ingest_free(h);
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

// The bytes [at[i], at[i] + len[i]) of host and device buffers, ascending and disjoint, read as one stream: stream byte
// s lies in range i where sum(len[0 .. i-1]) <= s < sum(len[0 .. i]) (pre[i] = that sum).
struct ByteRanges {
  std::vector<size_t> at, len, pre;
  void add(size_t a, size_t n) {
    if (!n) return;
    pre.push_back(pre.empty() ? 0 : pre.back() + len.back());
    at.push_back(a);
    len.push_back(n);
  }
  size_t total() const { return pre.empty() ? 0 : pre.back() + len.back(); }
  size_t find(size_t s) const { return (size_t)(std::upper_bound(pre.begin(), pre.end(), s) - pre.begin()) - 1; }
};

// Copy stream bytes [s0, s0 + n) of `host` (ranges rg) to dst
static void gather(char* dst, const char* host, const ByteRanges& rg, size_t s0, size_t n) {
  for (size_t i = n ? rg.find(s0) : 0, done = 0; done < n; ++i) {
    const size_t off = s0 + done - rg.pre[i], m = std::min(n - done, rg.len[i] - off);
    memcpy(dst + done, host + rg.at[i] + off, m);
    done += m;
  }
}

static void copy_slice(char* dst, const char* host, const ByteRanges& rg, size_t s0, size_t n, int t, int nthreads) {
  const size_t per = ((n / nthreads) + 4095) & ~(size_t)4095;
  const size_t lo = std::min(n, per * (size_t)t), hi = t == nthreads - 1 ? n : std::min(n, per * (size_t)(t + 1));
  if (hi > lo) gather(dst + lo, host, rg, s0 + lo, hi - lo);
}

// The ranges rg of host to the same positions of dev (one range [0, bytes): the whole buffer)
static int staged_h2d(b2_ctx* h, void* dev, const void* host, const ByteRanges& rg) {
  const size_t bytes = rg.total();
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
      copy_slice((char*)h->bounce[c & 1].p, (const char*)host, rg, off, n, t, nthreads);
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
    copy_slice((char*)b.p, (const char*)host, rg, off, n, 0, nthreads);
    while (crew.done.load(std::memory_order_acquire) < (c + 1) * (nthreads - 1)) std::this_thread::yield();
    for (size_t i = rg.find(off), done = 0; done < n && status == B2_OK; ++i) {   // one copy per range piece
      const size_t o = off + done - rg.pre[i], m = std::min(n - done, rg.len[i] - o);
      if (cudaMemcpyAsync((char*)dev + rg.at[i] + o, (char*)b.p + done, m, cudaMemcpyHostToDevice, h->stream) !=
          cudaSuccess)
        status = B2_ERR_CUDA;
      done += m;
    }
    if (status == B2_OK && cudaEventRecord(b.ev, h->stream) != cudaSuccess) status = B2_ERR_CUDA;
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
  if (bytes >= kBounceBytes / 2 && is_pageable(host)) {
    ByteRanges rg;
    rg.add(0, bytes);
    return staged_h2d(h, *dev, host, rg);
  }
  B2_CUDA(h, cudaMemcpyAsync(*dev, host, bytes, cudaMemcpyHostToDevice, h->stream));
  return B2_OK;
}

// stage_in of the int16 sample ranges [lo[i], hi[i]) (ascending, disjoint) of a buffer of `bytes` bytes: the device
// workspace spans the whole buffer, and only those ranges are copied, to their own positions (b2_sync_tracks_seg: the
// sampled segments and the audio videos, not the samples between segments).
static int stage_ranges(b2_ctx* h, int which, const void* host, size_t bytes, const std::vector<int64_t>& lo,
                        const std::vector<int64_t>& hi, void** dev) {
  B2_TRY(b2i_ws(h, which, bytes ? bytes : 16, dev));
  ByteRanges rg;
  for (size_t i = 0; i < lo.size(); ++i) rg.add((size_t)lo[i] * 2, (size_t)(hi[i] - lo[i]) * 2);
  if (rg.total() >= kBounceBytes / 2 && is_pageable(host)) return staged_h2d(h, *dev, host, rg);
  for (size_t i = 0; i < rg.at.size(); ++i)
    B2_CUDA(h, cudaMemcpyAsync((char*)*dev + rg.at[i], (const char*)host + rg.at[i], rg.len[i], cudaMemcpyHostToDevice,
                               h->stream));
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

extern "C" int64_t b2_vad_call_samples(int frame_rate, int sample_rate) {
  return energy_call_samples(frame_rate, sample_rate);
}

extern "C" int64_t b2_vad_num_windows(int64_t n_samples, int frame_rate, int sample_rate) {
  int fpw = b2_vad_frames_per_window(frame_rate, sample_rate);
  if (fpw <= 0 || n_samples < 0) return -1;
  // len(range(0, len, fpw)) per detector call (speech_transformers.py:169), summed over the chunk loop's calls
  return chunked_num_windows(n_samples, fpw, energy_call_samples(frame_rate, sample_rate));
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

// ---- PGS rasteriser (PGSSpeechTransformer.fit) ------------------------------------------------
extern "C" int b2_rasterize_pgs_lengths(const double* end_s, const int64_t* off, int B, int sample_rate,
                                        int64_t* lengths) {
  if (B < 0 || !off || !lengths) return B2_ERR_BAD_ARG;
  std::string err;
  return pgs_lengths(&err, "rasterize_pgs_lengths", "", nullptr, end_s, off, B, sample_rate, false, 0.0, nullptr,
                     lengths);
}

extern "C" int b2_rasterize_pgs(b2_handle h, const double* start_s, const double* end_s, const int64_t* off, int B,
                                int sample_rate, double start_seconds, float* out, const int64_t* out_off,
                                int memspace) {
  B2_ENTER(h);
  if (B < 0 || !off || !out_off) B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize_pgs: bad arguments");
  if (B == 0) return B2_OK;
  std::vector<int64_t> lengths(B);
  if (const int st = pgs_lengths(&h->err, "rasterize_pgs", "", start_s, end_s, off, B, sample_rate, true,
                                 start_seconds, nullptr, lengths.data()))
    return st;
  for (int b = 0; b < B; ++b)
    if (out_off[b + 1] < out_off[b]) B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize_pgs: out_off not monotone at %d", b);
  const int64_t base = out_off[0], total = out_off[B] - base;
  if (total && !out) B2_FAIL(h, B2_ERR_BAD_ARG, "rasterize_pgs: null output");
  if (total) B2_CHECK_DEV(h, memspace, out, "rasterize_pgs: out");
  // signal b goes to out + out_off[b]; a host call stages the signals from offset 0
  float* d_out = out;
  std::vector<int64_t> staged_off;
  const int64_t* d_off = out_off;
  if (memspace == B2_HOST) {
    void* dq;
    B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)total * 4 + 16, &dq));
    d_out = (float*)dq;
    staged_off.resize(B + 1);
    for (int b = 0; b <= B; ++b) staged_off[b] = out_off[b] - base;
    d_off = staged_off.data();
  }
  std::vector<int> all(B);
  for (int b = 0; b < B; ++b) all[b] = b;
  B2_TRY(b2i_raster_ref_launch(h, start_s, end_s, nullptr, off, d_off, B, all.data(), B, sample_rate, start_seconds,
                               d_out, true));
  if (memspace == B2_HOST) {
    B2_TRY(copy_out(h, out + base, d_out, (size_t)total * 4));
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

extern "C" int b2_capture_reference(b2_handle h, float* ref, int64_t capacity, int64_t* ref_off, uint8_t* packed,
                                    int64_t max_videos) {
  B2_ENTER(h);
  h->ref_capture = B2RefCapture{};
  if (!ref) return B2_OK;
  if (capacity < 0 || max_videos < 0 || !ref_off || !packed)
    B2_FAIL(h, B2_ERR_BAD_ARG, "capture_reference: bad arguments");
  B2_TRY(check_device_ptr(h, ref, "capture_reference: ref"));
  h->ref_capture = B2RefCapture{ref, (long long)capacity, ref_off, packed, (long long)max_videos};
  return B2_OK;
}

extern "C" int b2_speech_output(b2_handle h, double* speech, int64_t capacity, const int32_t* videos, int n_videos,
                                int64_t* speech_off, int memspace) {
  // Not B2_ENTER: this call enqueues nothing and is read only after a sync call's plan, so a chain of resident sync
  // calls stays valid across it (as across b2_apply_sync).
  if (!h) return B2_ERR_BAD_ARG;
  h->err.clear();
  DeviceScope scope(h->device);
  if (!scope.ok) return B2_ERR_CUDA;
  h->speech_out = B2SpeechOut{};
  if (!speech) return B2_OK;
  if (capacity < 0 || n_videos < 0 || !speech_off || (n_videos > 0 && !videos))
    B2_FAIL(h, B2_ERR_BAD_ARG, "speech_output: bad arguments (capacity %lld, %d videos)", (long long)capacity,
            n_videos);
  if (memspace != B2_HOST && memspace != B2_DEVICE)
    B2_FAIL(h, B2_ERR_BAD_ARG, "speech_output: memspace must be B2_HOST or B2_DEVICE");
  for (int i = 0; i < n_videos; ++i)
    if (videos[i] < 0 || (i > 0 && videos[i] <= videos[i - 1]))
      B2_FAIL(h, B2_ERR_BAD_ARG, "speech_output: videos[%d] = %d is negative or not increasing", i, (int)videos[i]);
  if (memspace == B2_DEVICE) B2_TRY(check_device_ptr(h, speech, "speech_output: speech"));
  B2SpeechOut sout;
  sout.speech = speech;
  sout.capacity = capacity;
  sout.videos.assign(videos, videos + n_videos);
  sout.speech_off = speech_off;
  sout.memspace = memspace;
  h->speech_out = std::move(sout);
  return B2_OK;
}

extern "C" int64_t b2_segment_length(double total_seconds, int sample_rate) {
  return seg_ref_length(total_seconds, sample_rate);
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
  const double* sigx;                 // signal references' stored values (absolute sig_off indices), on the device
  unsigned long long* first_bad;      // [V]: per video, its first out-of-domain frame (sig_ref_kernel)
  float* seg_scratch;                 // the sampled segments' detector output (plan: seg_frames floats)
  unsigned long long* speech;         // [V]: per segment video, its first frame > 0 (seg_ref_kernel)
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

// The references of the videos [v0, v1) that no detector writes and no PCM feeds, from the call's host tables: the
// signal videos' (sig_ref_kernel: floats, or in a packed sub-batch the bits the VAD would write; it also resets and
// sets their flags) and the text and PGS videos' (rasterised into their ranges).  The last part of the detector step
// of the whole calls and of the ingest session's sync alike.
static int written_refs(b2_ctx* h, const SyncRequest& r, const SyncPlan& p, const SyncBufs& b, int v0, int v1,
                        bool ref_packed) {
  // the videos of `list` in [v0, v1), relative to v0
  auto in_range = [&](const std::vector<int>& list) {
    std::vector<int> rel(std::lower_bound(list.begin(), list.end(), v0), std::lower_bound(list.begin(), list.end(), v1));
    for (int& v : rel) v -= v0;
    return rel;
  };
  const std::vector<int> sig(std::lower_bound(p.sig_video.begin(), p.sig_video.end(), v0),
                             std::lower_bound(p.sig_video.begin(), p.sig_video.end(), v1));
  if (!sig.empty())
    B2_TRY(b2i_sig_ref_launch(h, b.sigx, r.sig.off, p.ref_off.data(), r.V, sig.data(), (int)sig.size(), p.label,
                              ref_packed, b.refsig, b.first_bad));
  if (!p.any_subs) return B2_OK;
  const std::vector<int> subs = in_range(p.sub_video), pgs = in_range(p.pgs_video);
  if (!subs.empty())
    B2_TRY(b2i_raster_ref_launch(h, r.refs.cue_start_s, r.refs.cue_end_s, r.refs.cue_keep, r.refs.cue_off + v0,
                                 p.ref_off.data() + v0, v1 - v0, subs.data(), (int)subs.size(), r.sample_rate,
                                 r.start_seconds, b.refsig));
  if (!pgs.empty())
    B2_TRY(b2i_raster_ref_launch(h, r.pgs.start_s, r.pgs.end_s, nullptr, r.pgs.off + v0, p.ref_off.data() + v0,
                                 v1 - v0, pgs.data(), (int)pgs.size(), r.sample_rate, r.start_seconds, b.refsig,
                                 true));
  return B2_OK;
}

// The detector step of the videos [v0, v1), on whichever stream the handle launches on: the energy / ZCR VAD
// into the reference-signal buffer, or for auditok the energy pass over the videos' chunks (label 0, every
// crossing count accepted, a short last block judged on its own samples) writing its 0/1 flags there, then
// the tokenizer turning each chunk's flags into its float32 signal in place.  Both auditok launches take a
// metadata arena from the ring of the stream they run on; on the pipeline's internal stream that ring is its
// own, so the GSS invariant (no later arena of a chain recycles the chain's arena, runcorr.cu b2i_gss_launch)
// holds as before: the chains' arenas come from the caller-facing ring, and with one sub-batch the detector's
// arenas there precede the chain's.
// With subtitle references (b2_sync_tracks_subs; text and PGS ones with b2_sync_tracks_pgs) the step also
// rasterises those of the videos [v0, v1) into
// their ranges, on the same stream: the detector never writes there (no PCM: no tiles, no tokenizer chunk), and
// the step stays the buffer's only writer, so the pipeline and resident chaining need nothing new.
// With signal references (b2_sync_tracks_sig) sig_ref_kernel writes those of the videos [v0, v1) the same way, as
// floats or, in a packed sub-batch, as the bits the VAD would write; it also resets and sets their flags.
// With sampled segments (b2_sync_tracks_seg) a segment video is empty in the main launch (plan det_end); a second
// detector launch reads only its segments' samples into the scratch (floats), and seg_ref_kernel writes its reference
// from there, floats or bits, and resets and sets its speech flag.
// With ingested references (b2_ingest_sync_tracks / _refs) the detector already ran as the PCM arrived: the step copies
// the audio videos' references from the session's buffer to their ranges, one copy per run of videos stored back to
// back, seg_ref_kernel assembles the segment videos' ones from their segments' frames there, and the signal, text and
// PGS videos' ones are written from the call's tables as in the whole call (written_refs).
static int detect(b2_ctx* h, const SyncRequest& r, const SyncPlan& p, const SyncBufs& b, int v0, int v1,
                  bool ref_packed) {
  // the segment videos [s0, s1) of p.seg_video lie in [v0, v1)
  const int s0 = (int)(std::lower_bound(p.seg_video.begin(), p.seg_video.end(), v0) - p.seg_video.begin());
  const int s1 = (int)(std::lower_bound(p.seg_video.begin(), p.seg_video.end(), v1) - p.seg_video.begin());
  if (r.ready.len) {
    // a video whose reference is not its pushes' (segments, text, PGS, signal): none of its frames is copied
    auto not_audio = [&](int v) {
      auto has = [v](const std::vector<int>& list) { return std::binary_search(list.begin(), list.end(), v); };
      return (!p.seg_of.empty() && p.seg_of[v] >= 0) || has(p.sub_video) || has(p.pgs_video) || has(p.sig_video);
    };
    for (int v = v0; v < v1;) {
      if (not_audio(v)) {
        ++v;
        continue;
      }
      int w = v + 1;
      while (w < v1 && !not_audio(w) && r.ready.at[w] == r.ready.at[w - 1] + r.ready.len[w - 1]) ++w;
      const int64_t n = p.ref_off[w] - p.ref_off[v];
      if (n > 0)
        B2_CUDA(h, cudaMemcpyAsync(b.refsig + p.ref_off[v], r.ready.ref + r.ready.at[v], (size_t)n * 4,
                                   cudaMemcpyDeviceToDevice, h->stream));
      v = w;
    }
    // segment videos: their sparse references from the segments' frames in the session's buffer (run_src points there)
    if (s1 > s0)
      B2_TRY(b2i_seg_ref_launch(h, r.ready.ref, p.ref_off.data(), p.seg_video.data() + s0, s1 - s0,
                                p.run_first.data() + s0, p.run_lo.data(), p.run_src.data(), ref_packed, b.refsig,
                                b.speech));
    return p.any_ref ? written_refs(h, r, p, b, v0, v1, ref_packed) : B2_OK;
  }
  const bool seg = !p.det_end.empty();
  if (!p.auditok && p.chunked) {   // energy / ZCR over the detector calls (never packed: plan_ref_format)
    const ChunkTable& ch = p.ch;
    const int c0 = ch.first[v0];
    B2_TRY(b2i_vad_launch(h, b.pcm, ch.pcm.data() + c0, ch.first[v1] - c0, p.fpw, r.energy.non_speech_label,
                          (int64_t)p.fpw * r.energy.energy_threshold, p.z_lo, p.z_hi, b.refsig, ch.out.data() + c0,
                          nullptr, false, seg ? p.det_end.data() + c0 : nullptr));
  } else if (!p.auditok) {
    // a packed sub-batch of signal (or segment) videos alone has no audio: the VAD has no tiles and is not asked
    // for bits
    bool audio = r.pcm_off[v1] > r.pcm_off[v0];
    if (seg) {
      audio = false;
      for (int v = v0; v < v1; ++v) audio = audio || p.det_end[v] > r.pcm_off[v];
    }
    B2_TRY(b2i_vad_launch(h, b.pcm, r.pcm_off + v0, v1 - v0, p.fpw, r.energy.non_speech_label,
                          (int64_t)p.fpw * r.energy.energy_threshold, p.z_lo, p.z_hi, b.refsig, p.ref_off.data() + v0,
                          nullptr, ref_packed && audio, seg ? p.det_end.data() + v0 : nullptr));
  } else {
    const ChunkTable& ch = p.ch;
    const int c0 = ch.first[v0], nc = ch.first[v1] - c0;
    B2_TRY(b2i_vad_launch(h, b.pcm, ch.pcm.data() + c0, nc, p.fpw, 0.0f, p.auditok_e_min, 0, p.fpw, b.refsig,
                          ch.out.data() + c0, ch.tail.data() + c0, false, seg ? p.det_end.data() + c0 : nullptr));
    if (!p.any_ref) return b2i_tokenize_inplace_launch(h, b.refsig, ch.out.data() + c0, nc, p.tok);
    const int k0 = ch.tok_first[v0];
    B2_TRY(b2i_tokenize_inplace_launch(h, b.refsig, ch.tok_off.data() + k0, ch.tok_first[v1] - k0, p.tok,
                                       ch.tok_end.data() + k0));
  }
  if (!p.any_ref) return B2_OK;
  if (s1 > s0) {
    const int k0 = p.item_first[v0], nk = p.item_first[v1] - k0;
    if (nk > 0 && !p.auditok) {
      B2_TRY(b2i_vad_launch(h, b.pcm, p.item_start.data() + k0, nk, p.fpw, r.energy.non_speech_label,
                            (int64_t)p.fpw * r.energy.energy_threshold, p.z_lo, p.z_hi, b.seg_scratch,
                            p.item_out.data() + k0, nullptr, false, p.item_end.data() + k0));
    } else if (nk > 0) {   // auditok: the energy pass, then the tokenizer restarting in every item
      B2_TRY(b2i_vad_launch(h, b.pcm, p.item_start.data() + k0, nk, p.fpw, 0.0f, p.auditok_e_min, 0, p.fpw,
                            b.seg_scratch, p.item_out.data() + k0, p.item_tail.data() + k0, false,
                            p.item_end.data() + k0));
      B2_TRY(b2i_tokenize_inplace_launch(h, b.seg_scratch, p.item_out.data() + k0, nk, p.tok));
    }
    B2_TRY(b2i_seg_ref_launch(h, b.seg_scratch, p.ref_off.data(), p.seg_video.data() + s0, s1 - s0,
                              p.run_first.data() + s0, p.run_lo.data(), p.run_src.data(), ref_packed, b.refsig,
                              b.speech));
  }
  return written_refs(h, r, p, b, v0, v1, ref_packed);
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
  const B2SpeechOut& sout = h->speech_out;
  env.speech_out = sout.speech != nullptr;
  if (const int st = plan_sync(r, env, &p)) {
    h->err = p.err;
    return st;
  }
  const int T = r.T, K = r.K;
  if (T == 0 && !sout.speech) return B2_OK;
  const B2RefCapture rc = h->ref_capture;
  if (rc.ref && (p.ref_off[r.V] > rc.capacity || r.V > rc.max_videos))
    B2_FAIL(h, B2_ERR_BAD_ARG, "%s: the reference capture holds %lld frames of %lld videos, the call has %lld of %d",
            r.who, rc.capacity, rc.max_videos, (long long)p.ref_off[r.V], r.V);
  const bool resident = r.memspace == B2_DEVICE_RESIDENT;
  const int memspace = resident ? B2_DEVICE : r.memspace;
  // The speech output: its offsets and its checks, before anything is enqueued
  const int n_speech = (int)sout.videos.size();
  std::vector<int64_t> speech_off;
  if (sout.speech) {
    if ((sout.memspace == B2_HOST) != (memspace == B2_HOST))
      B2_FAIL(h, B2_ERR_BAD_ARG, "%s: the speech output was set for %s memory, the call is a %s call", r.who,
              sout.memspace == B2_HOST ? "host" : "device", memspace == B2_HOST ? "B2_HOST" : "B2_DEVICE");
    if (n_speech > 0 && sout.videos.back() >= r.V)
      B2_FAIL(h, B2_ERR_BAD_ARG, "%s: the speech output lists video %d, the call has %d videos", r.who,
              sout.videos.back(), r.V);
    speech_off.assign(n_speech + 1, 0);
    for (int i = 0; i < n_speech; ++i)
      speech_off[i + 1] = speech_off[i] + p.ref_off[sout.videos[i] + 1] - p.ref_off[sout.videos[i]];
    if (speech_off[n_speech] > sout.capacity)
      B2_FAIL(h, B2_ERR_BAD_ARG, "%s: the speech output holds %lld frames, the listed videos need %lld", r.who,
              sout.capacity, (long long)speech_off[n_speech]);
    std::copy(speech_off.begin(), speech_off.end(), sout.speech_off);
  }
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
  const bool any_sig = !p.sig_video.empty();
  const int64_t sig0 = any_sig ? r.sig.off[0] : 0, n_sig_values = any_sig ? r.sig.off[r.V] - sig0 : 0;
  if (n_sig_values > 0) {
    char what[64];
    snprintf(what, sizeof(what), "%s: x", r.who);
    B2_CHECK_DEV(h, memspace, r.sig.x, what);
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
  // signal references: the per-video flags of sig_ref_kernel follow the reference in the same buffer, so a chained
  // resident call's flags alternate with its reference and live exactly as long
  // (and so do the speech flags of seg_ref_kernel, then the segments' detector scratch)
  const bool any_seg = !p.seg_video.empty();
  const size_t ref_bytes = any_sig || any_seg ? (((size_t)p.ref_off[r.V] * 4 + 64 + 7) & ~(size_t)7)
                                              : (size_t)p.ref_off[r.V] * 4 + 64;
  const size_t flag_bytes = (any_sig ? (size_t)r.V * 8 : 0) + (any_seg ? (size_t)r.V * 8 : 0);
  const size_t scr_at = (ref_bytes + flag_bytes + 15) & ~(size_t)15;
  B2_TRY(b2i_ws(h, refsig_slot, any_seg ? scr_at + (size_t)p.seg_frames * 4 + 64 : ref_bytes + flag_bytes,
                &d_refsig));
  b.first_bad = any_sig ? (unsigned long long*)((char*)d_refsig + ref_bytes) : nullptr;
  b.speech = any_seg ? (unsigned long long*)((char*)d_refsig + ref_bytes + (any_sig ? (size_t)r.V * 8 : 0)) : nullptr;
  b.seg_scratch = any_seg ? (float*)((char*)d_refsig + scr_at) : nullptr;
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
    if (T == 0 && !r.ready.len) {   // serialize-only: the samples the listed videos' detector step reads
      std::vector<std::pair<int64_t, int64_t>> rg;
      for (int v : sout.videos) {
        if (any_seg && p.seg_of[v] >= 0) {
          for (int k = p.item_first[v]; k < p.item_first[v + 1]; ++k) rg.push_back({p.item_start[k], p.item_end[k]});
        } else if (r.pcm_off[v + 1] > r.pcm_off[v]) {
          rg.push_back({r.pcm_off[v], r.pcm_off[v + 1]});
        }
      }
      std::sort(rg.begin(), rg.end());
      std::vector<int64_t> lo, hi;
      for (const auto& [a0, b0] : rg) {
        if (!hi.empty() && a0 <= hi.back()) hi.back() = std::max(hi.back(), b0);
        else {
          lo.push_back(a0);
          hi.push_back(b0);
        }
      }
      if (!lo.empty()) B2_TRY(stage_ranges(h, b2_ctx::WS_STAGE_IN0, r.pcm, (size_t)r.pcm_off[r.V] * 2, lo, hi, &dp));
    } else if (p.audio_samples > 0 && any_seg)   // the ranges the detector reads, at their own positions
      B2_TRY(stage_ranges(h, b2_ctx::WS_STAGE_IN0, r.pcm, (size_t)r.pcm_off[r.V] * 2, p.stage_lo, p.stage_hi, &dp));
    else if (p.audio_samples > 0)
      B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, r.pcm, (size_t)r.pcm_off[r.V] * 2, &dp));
    b.pcm = (const int16_t*)dp;
  }
  b.sigx = r.sig.x;
  if (memspace == B2_HOST && n_sig_values > 0) {   // the values [sig_off[0], sig_off[V]), read with their indices
    void* dx;
    B2_TRY(stage_in(h, b2_ctx::WS_STAGE_SIG, r.sig.x + sig0, (size_t)n_sig_values * 8, &dx));
    b.sigx = (const double*)dx - sig0;
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
  if (T > 0) {
    B2_TRY(run_pipeline(h, r, p, b, resident, chained, refsig_slot));
  } else {
    // no tracks, speech output set (the reference's serialize-only run): the detector step of the listed videos,
    // one launch sequence per run of consecutive indices, on the caller's stream
    for (int i = 0; i < n_speech;) {
      int j = i + 1;
      while (j < n_speech && sout.videos[j] == sout.videos[j - 1] + 1) ++j;
      B2_TRY(detect(h, r, p, b, sout.videos[i], sout.videos[j - 1] + 1, false));
      i = j;
    }
  }
  // Signal videos with out-of-domain values and segment videos without speech: their tracks' outputs are overwritten
  // behind every chain, on the caller's stream, before the host copies (the flags stay valid as the reference buffer
  // does, below)
  if (T > 0 && (any_sig || any_seg)) {
    B2SigBadOut so{b.bs, b.bo, b.bk, nullptr, nullptr, K, nullptr, nullptr, kGssEvals};
    if (p.gss) {
      so.a_score = b.g_all_score;
      so.a_offset = b.g_all_offset;
      so.cols = K + 1;
      so.ratio = b.g_ratio;
      so.evals = b.g_evals;
    } else {
      so.a_score = r.all_score ? b.score : nullptr;
      so.a_offset = r.all_offset ? b.offset : nullptr;
    }
    B2_TRY(b2i_sentinel_launch(h, b.first_bad, p.sig_video.data(), (int)p.sig_video.size(), p.trk_off.data(), so,
                               B2_BEST_K_BAD_SIGNAL, true));
    // segment videos without a frame > 0
    B2_TRY(b2i_sentinel_launch(h, b.speech, p.seg_video.data(), (int)p.seg_video.size(), p.trk_off.data(), so,
                               B2_BEST_K_NO_SPEECH, false));
  }
  // The reference capture: one copy behind every chain on the caller's stream, when every detector step is done.
  // The buffer stays valid until then: no chain kernel writes it (they read it as const), the next chained
  // resident call writes the other buffer, and the call after that starts its detector behind a fence recorded
  // on this stream after the copy.
  if (rc.ref) {
    for (int v = 0; v <= r.V; ++v) rc.ref_off[v] = p.ref_off[v];
    for (int i = 0; i < p.n_sub; ++i)
      for (int v = p.cut[i]; v < p.cut[i + 1]; ++v) rc.packed[v] = p.ref_packed[i];
    if (p.ref_off[r.V] > 0)
      B2_CUDA(h, cudaMemcpyAsync(rc.ref, b.refsig, (size_t)p.ref_off[r.V] * 4, cudaMemcpyDeviceToDevice, h->stream));
  }
  // The speech output (K1o): one kernel at the capture's spot, behind every chain on the caller's stream, so the same
  // argument keeps the buffer valid.  There it reads a buffer no kernel writes any more and adds no ordering beyond
  // the stream's; beside the later sub-batches' detector it would take HBM bandwidth from that bandwidth-bound step.
  // B2_HOST: written to a workspace and copied out with the results below.
  double* d_speech = sout.speech;
  if (sout.speech && speech_off[n_speech] > 0) {
    std::vector<B2SpeechVideo> sv(n_speech);
    for (int i = 0; i < n_speech; ++i) {
      const int v = sout.videos[i];
      const int sb = (int)(std::upper_bound(p.cut.begin(), p.cut.end(), v) - p.cut.begin()) - 1;
      auto has = [v](const std::vector<int>& list) { return std::binary_search(list.begin(), list.end(), v); };
      // a clear bit is the label for detector and signal videos, 0.0 for text, PGS and segment videos
      const bool zero_low = has(p.sub_video) || has(p.pgs_video) || has(p.seg_video);
      sv[i] = B2SpeechVideo{(long long)p.ref_off[v], zero_low ? 0.0f : p.label, p.ref_packed[sb] ? 1 : 0};
    }
    if (!dev) {
      void* ds;
      B2_TRY(b2i_ws(h, b2_ctx::WS_SPEECH, (size_t)speech_off[n_speech] * 8 + 64, &ds));
      d_speech = (double*)ds;
    }
    B2_TRY(b2i_speech_out_launch(h, b.refsig, speech_off.data(), sv.data(), n_speech, d_speech));
  }
  if (dev) return B2_OK;
  if (sout.speech) B2_TRY(copy_out(h, sout.speech, d_speech, (size_t)speech_off[n_speech] * 8));
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

extern "C" int b2_sync_tracks_pgs(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                                  const int32_t* track_video, int T, int frame_rate, int sample_rate, int detector,
                                  double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                                  double energy_threshold_db, double min_length, int64_t max_length,
                                  double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs,
                                  const double* ref_cue_start_s, const double* ref_cue_end_s,
                                  const uint8_t* ref_cue_keep, const int64_t* ref_cue_off, const uint8_t* ref_is_pgs,
                                  const double* pgs_start_s, const double* pgs_end_s, const int64_t* pgs_off,
                                  const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                                  const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                                  int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                                  int32_t* best_k, double* all_score, int32_t* all_offset, double* gss_ratio,
                                  double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks_pgs");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_pgs: null track_video");
  if (!gss_ratio && gss_evals) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_pgs: gss_evals without gss_ratio");
  if (V > 0 && (!pcm_off || !pgs_off)) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_pgs: null pcm_off / pgs_off");
  if (ref_is_subs && !ref_cue_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_pgs: ref_is_subs without ref_cue_off");
  if (detector != B2_DETECTOR_ENERGY_ZCR && detector != B2_DETECTOR_AUDITOK)
    B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_pgs: detector must be B2_DETECTOR_ENERGY_ZCR or B2_DETECTOR_AUDITOK, "
            "not %d", detector);
  static const int64_t no_intervals[1] = {0};
  SyncRequest r{gss_ratio ? "sync_tracks_pgs (search)" : "sync_tracks_pgs", pcm, pcm_off, V, track_video, T,
                frame_rate, sample_rate, detector, {(float)non_speech_label, energy_threshold, z_lo, z_hi},
                {non_speech_label, energy_threshold_db, min_length, max_continuous_silence, max_length, chunk_samples},
                {ref_is_subs, ref_cue_start_s, ref_cue_end_s, ref_cue_keep, V > 0 ? ref_cue_off : nullptr},
                cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                best_score, best_offset, best_k, all_score, all_offset, gss_ratio != nullptr, gss_ratio, gss_evals,
                memspace};
  r.pgs = {ref_is_pgs, pgs_start_s, pgs_end_s, V > 0 ? pgs_off : no_intervals};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_sync_tracks_sig(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                                  const int32_t* track_video, int T, int frame_rate, int sample_rate, int detector,
                                  double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                                  double energy_threshold_db, double min_length, int64_t max_length,
                                  double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs,
                                  const double* ref_cue_start_s, const double* ref_cue_end_s,
                                  const uint8_t* ref_cue_keep, const int64_t* ref_cue_off, const uint8_t* ref_is_pgs,
                                  const double* pgs_start_s, const double* pgs_end_s, const int64_t* pgs_off,
                                  const uint8_t* ref_is_sig, const double* x, const int64_t* sig_off,
                                  const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                                  const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                                  int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                                  int32_t* best_k, double* all_score, int32_t* all_offset, double* gss_ratio,
                                  double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks_sig");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_sig: null track_video");
  if (!gss_ratio && gss_evals) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_sig: gss_evals without gss_ratio");
  if (V > 0 && (!pcm_off || !sig_off)) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_sig: null pcm_off / sig_off");
  if (ref_is_subs && !ref_cue_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_sig: ref_is_subs without ref_cue_off");
  if (ref_is_pgs && !pgs_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_sig: ref_is_pgs without pgs_off");
  if (detector != B2_DETECTOR_ENERGY_ZCR && detector != B2_DETECTOR_AUDITOK)
    B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_sig: detector must be B2_DETECTOR_ENERGY_ZCR or B2_DETECTOR_AUDITOK, "
            "not %d", detector);
  static const int64_t no_values[1] = {0};
  SyncRequest r{gss_ratio ? "sync_tracks_sig (search)" : "sync_tracks_sig", pcm, pcm_off, V, track_video, T,
                frame_rate, sample_rate, detector, {(float)non_speech_label, energy_threshold, z_lo, z_hi},
                {non_speech_label, energy_threshold_db, min_length, max_continuous_silence, max_length, chunk_samples},
                {ref_is_subs, ref_cue_start_s, ref_cue_end_s, ref_cue_keep, V > 0 ? ref_cue_off : nullptr},
                cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                best_score, best_offset, best_k, all_score, all_offset, gss_ratio != nullptr, gss_ratio, gss_evals,
                memspace};
  r.pgs = {ref_is_pgs, pgs_start_s, pgs_end_s, V > 0 ? pgs_off : nullptr};
  r.sig = {ref_is_sig, x, V > 0 ? sig_off : no_values};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_sync_tracks_seg(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int V,
                                  const int32_t* track_video, int T, int frame_rate, int sample_rate, int detector,
                                  double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                                  double energy_threshold_db, double min_length, int64_t max_length,
                                  double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs,
                                  const double* ref_cue_start_s, const double* ref_cue_end_s,
                                  const uint8_t* ref_cue_keep, const int64_t* ref_cue_off, const uint8_t* ref_is_pgs,
                                  const double* pgs_start_s, const double* pgs_end_s, const int64_t* pgs_off,
                                  const uint8_t* ref_is_sig, const double* x, const int64_t* sig_off, int n_seg_videos,
                                  const int32_t* seg_video, const double* seg_total, const int64_t* seg_off,
                                  const int64_t* seg_start, const int64_t* seg_lo, const int64_t* seg_hi,
                                  const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                                  const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                                  int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                                  int32_t* best_k, double* all_score, int32_t* all_offset, double* gss_ratio,
                                  double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_sync_tracks_seg");
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: null track_video");
  if (!gss_ratio && gss_evals) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: gss_evals without gss_ratio");
  if (V > 0 && !pcm_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: null pcm_off");
  if (n_seg_videos < 0 || (n_seg_videos > 0 && !seg_off))
    B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: %d segment videos without seg_off", n_seg_videos);
  if (ref_is_subs && !ref_cue_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: ref_is_subs without ref_cue_off");
  if (ref_is_pgs && !pgs_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: ref_is_pgs without pgs_off");
  if (ref_is_sig && !sig_off) B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: ref_is_sig without sig_off");
  if (detector != B2_DETECTOR_ENERGY_ZCR && detector != B2_DETECTOR_AUDITOK)
    B2_FAIL(h, B2_ERR_BAD_ARG, "sync_tracks_seg: detector must be B2_DETECTOR_ENERGY_ZCR or B2_DETECTOR_AUDITOK, "
            "not %d", detector);
  static const int64_t no_segments[1] = {0};
  SyncRequest r{gss_ratio ? "sync_tracks_seg (search)" : "sync_tracks_seg", pcm, pcm_off, V, track_video, T,
                frame_rate, sample_rate, detector, {(float)non_speech_label, energy_threshold, z_lo, z_hi},
                {non_speech_label, energy_threshold_db, min_length, max_continuous_silence, max_length, chunk_samples},
                {ref_is_subs, ref_cue_start_s, ref_cue_end_s, ref_cue_keep, V > 0 ? ref_cue_off : nullptr},
                cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K, start_seconds, max_offset_samples,
                best_score, best_offset, best_k, all_score, all_offset, gss_ratio != nullptr, gss_ratio, gss_evals,
                memspace};
  r.pgs = {ref_is_pgs, pgs_start_s, pgs_end_s, V > 0 ? pgs_off : nullptr};
  r.sig = {ref_is_sig, x, V > 0 ? sig_off : nullptr};
  r.seg = {n_seg_videos, seg_video, seg_total, n_seg_videos > 0 ? seg_off : no_segments, seg_start, seg_lo, seg_hi};
  return sync_run(h, _b2_fence_was_valid, r);
}

// ---- batched ingest session (b2_ingest_*, DESIGN.md section 4 "K1i") ---------------------------------------------
// The reference's chunk loop (speech_transformers.py:680-753) for V videos at once: each push is cut by the span
// planner (ingest_plan.h), its spans staged in a ring slot of pinned host and device memory, copied to the device
// and run through the detector in one b2i_vad_launch over a table of (staging offset, samples, destination frame);
// for auditok the tokenizer then runs over every detector call the push completed.  Only the detector's output stays
// on the device, stream k's (an audio video's, or a sampled segment's: IngestStreams) at frames [at[k], at[k] + cap[k])
// of one buffer; b2_ingest_sync_tracks hands them to the batched sync calls' chain as ingested references
// (SyncRequest::ready), the segments' ones to be assembled into their videos' sparse references there.
struct IngestSession {
  static const int kSlots = 3;
  struct Slot {
    void* hp = nullptr;   // pinned staging
    void* dp = nullptr;   // device staging
    size_t cap = 0;
    cudaEvent_t ev = nullptr;
    bool busy = false;
  } slot[kSlots];
  uint64_t seq = 0;
  bool active = false;
  SyncRequest req{};                  // the detector arguments, as the sync call passes them
  SyncPlan det;                       // fpw, z_lo, z_hi, auditok_e_min, tok of those arguments
  int V = 0;
  IngestStreams streams;              // which stream each push feeds
  IngestPlanner plan;                 // per stream
  std::vector<std::vector<uint8_t>> held;   // stream k's bytes [2 * plan.base[k], plan.bytes[k])
  std::vector<int64_t> hint;          // [V] frames expected per stream of video v (expect_samples), 0: none
  float* ref = nullptr;               // cudaMallocAsync on the handle's stream
  std::vector<int64_t> at, cap;       // per stream
};

static void ingest_release_ref(b2_ctx* h, IngestSession* s) {
  if (s->ref) cudaFreeAsync(s->ref, h->stream);   // behind every kernel and copy that reads or writes it
  s->ref = nullptr;
  s->active = false;
  s->held.clear();
}

static void ingest_free(b2_ctx* h) {
  IngestSession* s = h->ingest;
  if (!s) return;
  ingest_release_ref(h, s);
  cudaStreamSynchronize(h->stream);
  for (auto& sl : s->slot) {
    if (sl.hp) cudaFreeHost(sl.hp);
    if (sl.dp) cudaFree(sl.dp);
    if (sl.ev) cudaEventDestroy(sl.ev);
  }
  delete s;
  h->ingest = nullptr;
}

// The streams' regions become cap[k] frames each, back to back in a new buffer: the frames written so far (at most
// written[k]) are copied over on the stream, and the old buffer is freed behind them.
static int ingest_relayout(b2_ctx* h, IngestSession* s, const std::vector<int64_t>& cap,
                           const std::vector<int64_t>& written) {
  const int n = (int)cap.size();
  std::vector<int64_t> at(n);
  int64_t total = 0;
  for (int k = 0; k < n; ++k) {
    at[k] = total;
    total += cap[k];
  }
  float* ref = nullptr;
  const cudaError_t e = cudaMallocAsync((void**)&ref, (size_t)total * 4 + 16, h->stream);
  if (e != cudaSuccess) {
    cudaGetLastError();
    B2_FAIL(h, B2_ERR_NOMEM, "ingest: cudaMallocAsync(%lld frames) for the references failed: %s", (long long)total,
            cudaGetErrorString(e));
  }
  for (int k = 0; k < n; ++k) {   // every frame written so far lies in the old region
    const int64_t m = k < (int)s->cap.size() ? std::min(std::min(s->cap[k], written[k]), cap[k]) : 0;
    if (m > 0)
      B2_CUDA(h, cudaMemcpyAsync(ref + at[k], s->ref + s->at[k], (size_t)m * 4, cudaMemcpyDeviceToDevice, h->stream));
  }
  if (s->ref) B2_CUDA(h, cudaFreeAsync(s->ref, h->stream));
  s->ref = ref;
  s->at.swap(at);
  s->cap = cap;
  return B2_OK;
}

// Room for frames [at[k], at[k] + need[k]) of every stream.  On overflow every live region grows to at least twice
// what its stream needs and to what the longest stream of its kind needs (videos decoded side by side grow alike, and
// so do their segments; a segment never grows to a whole video's length because a video did).  Streams that take no
// pushes (a segment video's own, a dropped segment's) keep their regions.
static int ingest_reserve(b2_ctx* h, IngestSession* s, const std::vector<int64_t>& need) {
  const int n = (int)need.size();
  bool grow = false;
  int64_t longest[2] = {0, 0};
  for (int k = 0; k < n; ++k) {
    grow = grow || need[k] > s->cap[k];
    longest[k >= s->V] = std::max(longest[k >= s->V], need[k]);
  }
  if (!grow) return B2_OK;
  std::vector<int64_t> cap(n);
  for (int k = 0; k < n; ++k)
    cap[k] = s->streams.live(k) ? std::max(s->cap[k], std::max(2 * need[k], longest[k >= s->V])) : s->cap[k];
  return ingest_relayout(h, s, cap, need);
}

// Appends the bytes [b0, b1) of the concatenation a ++ b (lengths na, nb) to dst
static void concat_bytes(uint8_t* dst, const uint8_t* a, int64_t na, const uint8_t* b, int64_t b0, int64_t b1) {
  if (b0 < na) {
    const int64_t m = std::min(b1, na) - b0;
    memcpy(dst, a + b0, (size_t)m);
    dst += m;
    b0 += m;
  }
  if (b1 > b0) memcpy(dst, b + (b0 - na), (size_t)(b1 - b0));
}

// Streams grew by the chunks (stream[i], bytes[i], n_bytes[i]) (n = 0 and final: every live stream's end): plans the
// spans, stages them in the next ring slot, and enqueues the copy, the detector launch and the tokenizer launch.
static int ingest_enqueue(b2_ctx* h, IngestSession* s, int n, const int32_t* video, const void* const* bytes,
                          const int64_t* n_bytes, bool final) {
  IngestPlanner& pl = s->plan;
  const int NS = (int)pl.bytes.size(), fpw = pl.fpw;
  // staging bound: every chunk with a held-back window and an odd byte in front, 16 bytes of alignment per span
  size_t bound = 0;
  auto spans_bound = [&](int64_t nb) { return 2 + (pl.chunk > 0 ? (nb / 2 + fpw) / pl.chunk : 0); };
  for (int i = 0; i < n; ++i) bound += (size_t)n_bytes[i] + 2 * fpw + 2 + 16 * spans_bound(n_bytes[i] + 2 * fpw);
  if (final)
    for (int k = 0; k < NS; ++k) bound += s->held[k].size() + 16 * 2;
  IngestSession::Slot& sl = s->slot[s->seq % IngestSession::kSlots];
  if (sl.busy) B2_CUDA(h, cudaEventSynchronize(sl.ev));   // the push kSlots ago has read this slot
  sl.busy = false;
  if (bound > sl.cap) {
    if (sl.hp) B2_CUDA(h, cudaFreeHost(sl.hp));
    if (sl.dp) B2_CUDA(h, cudaFree(sl.dp));
    sl.hp = sl.dp = nullptr;
    sl.cap = 0;
    const size_t want = bound + bound / 4 + 4096;
    B2_CUDA(h, cudaMallocHost(&sl.hp, want));
    B2_CUDA(h, cudaMalloc(&sl.dp, want));
    sl.cap = want;
  }
  if (!sl.ev) B2_CUDA(h, cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming));
  std::vector<IngestSpan> spans;
  std::vector<IngestChunk> chunks;
  std::vector<int64_t> stage;   // per span: its first sample in the slot (a multiple of 8)
  int64_t used = 0;             // samples
  auto add = [&](int v, const uint8_t* src, int64_t nsrc, int64_t base0, size_t from) {
    // the spans from index `from` on read video v's bytes [2 * base0, ...) = held ++ src
    const std::vector<uint8_t>& hv = s->held[v];
    for (size_t j = from; j < spans.size(); ++j) {
      const IngestSpan& sp = spans[j];
      stage.push_back(used);
      concat_bytes((uint8_t*)sl.hp + used * 2, hv.data(), (int64_t)hv.size(), src, 2 * (sp.s0 - base0),
                   2 * (sp.s1 - base0));
      used += (sp.s1 - sp.s0 + 7) & ~(int64_t)7;
    }
    // the new held-back bytes
    const int64_t keep0 = 2 * (pl.base[v] - base0), total = (int64_t)hv.size() + nsrc;
    std::vector<uint8_t> rest((size_t)(total - keep0));
    concat_bytes(rest.data(), hv.data(), (int64_t)hv.size(), src, keep0, total);
    s->held[v].swap(rest);
  };
  for (int i = 0; i < n; ++i) {
    const int v = video[i];
    const int64_t base0 = pl.base[v];
    const size_t from = spans.size();
    pl.push(v, n_bytes[i], &spans, &chunks);
    add(v, (const uint8_t*)bytes[i], n_bytes[i], base0, from);
  }
  if (final)
    for (int v = 0; v < NS; ++v) {
      if (!s->streams.live(v)) continue;   // a segment video's own stream, a dropped segment
      const int64_t base0 = pl.base[v];
      const size_t from = spans.size();
      pl.finish(v, &spans, &chunks);
      add(v, nullptr, 0, base0, from);
    }
  ++s->seq;
  const SyncPlan& dp = s->det;
  if (!spans.empty()) {
    B2_TRY(ingest_reserve(h, s, pl.frames));
    B2_CUDA(h, cudaMemcpyAsync(sl.dp, sl.hp, (size_t)used * 2, cudaMemcpyHostToDevice, h->stream));
    // the launch table: span j is entry 2j; entry 2j + 1 is an empty gap up to span j + 1's first frame, so that
    // out_off[2j + 1] - out_off[2j] is span j's window count while destinations need not be ordered
    const int S = (int)spans.size(), B = 2 * S - 1;
    std::vector<int64_t> off(B + 1), end(B), out(B + 1), tail(B, 0);
    for (int j = 0; j < S; ++j) {
      const IngestSpan& sp = spans[j];
      const int64_t d = s->at[sp.video] + sp.frame;
      off[2 * j] = stage[j];
      end[2 * j] = stage[j] + (sp.s1 - sp.s0);
      out[2 * j] = d;
      out[2 * j + 1] = d + (sp.s1 - sp.s0 + fpw - 1) / fpw;
      tail[2 * j] = sp.tail;
      if (j + 1 < S) off[2 * j + 1] = end[2 * j + 1] = end[2 * j];
    }
    off[B] = end[B - 1];
    if (!pl.auditok)
      B2_TRY(b2i_vad_launch(h, (const int16_t*)sl.dp, off.data(), B, fpw, s->req.energy.non_speech_label,
                            (int64_t)fpw * s->req.energy.energy_threshold, dp.z_lo, dp.z_hi, s->ref, out.data(),
                            nullptr, false, end.data()));
    else   // the energy pass (label 0, every crossing count, a closed call's short last block on its own samples)
      B2_TRY(b2i_vad_launch(h, (const int16_t*)sl.dp, off.data(), B, fpw, 0.0f, dp.auditok_e_min, 0, fpw, s->ref,
                            out.data(), tail.data(), false, end.data()));
    B2_CUDA(h, cudaEventRecord(sl.ev, h->stream));
    sl.busy = true;
  }
  // auditok: the tokenizer over every detector call this step completed.  A call can complete without a span of its
  // own here: the flush closes a video's last call even when its length ends on a window boundary (nothing held back).
  if (!chunks.empty()) {
    std::vector<int64_t> c0(chunks.size() + 1), c1(chunks.size());
    for (size_t k = 0; k < chunks.size(); ++k) {
      c0[k] = s->at[chunks[k].video] + chunks[k].f0;
      c1[k] = s->at[chunks[k].video] + chunks[k].f1;
    }
    c0.back() = c1.back();
    B2_TRY(b2i_tokenize_inplace_launch(h, s->ref, c0.data(), (int)chunks.size(), dp.tok, c1.data()));
  }
  return B2_OK;
}

extern "C" int b2_ingest_begin(b2_handle h, int V, int frame_rate, int sample_rate, int detector,
                               double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                               double energy_threshold_db, double min_length, int64_t max_length,
                               double max_continuous_silence, int64_t chunk_samples, const int64_t* expect_samples) {
  B2_ENTER(h);
  if (h->ingest && h->ingest->active) B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_begin: a session is already open on this handle");
  if (V < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_begin: V = %d < 0", V);
  if (detector != B2_DETECTOR_ENERGY_ZCR && detector != B2_DETECTOR_AUDITOK)
    B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_begin: detector must be B2_DETECTOR_ENERGY_ZCR or B2_DETECTOR_AUDITOK, not %d",
            detector);
  for (int v = 0; expect_samples && v < V; ++v)
    if (expect_samples[v] < 0)
      B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_begin: expect_samples[%d] = %lld < 0", v, (long long)expect_samples[v]);
  // the detector arguments and their checks: the sync calls' own (plan_references), on a call without videos
  static const int64_t no_pcm[1] = {0};
  SyncRequest r{};
  r.who = "ingest_begin";
  r.pcm_off = no_pcm;
  r.frame_rate = frame_rate;
  r.sample_rate = sample_rate;
  r.detector = detector;
  r.energy = {(float)non_speech_label, energy_threshold, z_lo, z_hi};
  r.auditok = {non_speech_label, energy_threshold_db, min_length, max_continuous_silence, max_length, chunk_samples};
  SyncPlan det;
  det.auditok = detector == B2_DETECTOR_AUDITOK;
  if (const int st = plan_references(r, &det)) {
    h->err = det.err;
    return st;
  }
  if (!h->ingest) h->ingest = new IngestSession();
  IngestSession* s = h->ingest;
  s->req = r;
  s->det = det;
  s->V = V;
  s->streams.begin(V);
  s->plan.begin(V, det.fpw, det.auditok, det.call, energy_threshold_db);
  s->held.assign(V, {});
  s->at.assign(V, 0);
  s->cap.assign(V, 0);
  std::vector<int64_t> need(V, 0);
  for (int v = 0; expect_samples && v < V; ++v) need[v] = s->plan.length(expect_samples[v]);
  s->hint = need;
  // sized to the hint exactly (regions back to back: the sync step then copies them in one piece)
  int64_t total = 0;
  for (int v = 0; v < V; ++v) {
    s->at[v] = total;
    s->cap[v] = need[v];
    total += need[v];
  }
  if (total > 0) {
    const cudaError_t e = cudaMallocAsync((void**)&s->ref, (size_t)total * 4 + 16, h->stream);
    if (e != cudaSuccess) {
      cudaGetLastError();
      s->ref = nullptr;
      B2_FAIL(h, B2_ERR_NOMEM, "ingest_begin: cudaMallocAsync(%lld frames) for the references failed: %s",
              (long long)total, cudaGetErrorString(e));
    }
  }
  s->active = true;
  return B2_OK;
}

// Routes chunk i to its stream: video[i]'s own, or with `segmented` its segment segment[i].  A refused chunk refuses
// the whole call before anything is pushed.  The chunks' videos then count as pushed to.
static int ingest_push_any(b2_ctx* h, const char* who, int n, const int32_t* video, bool segmented,
                           const int64_t* segment, const void* const* bytes, const int64_t* n_bytes) {
  IngestSession* s = h->ingest;
  if (!s || !s->active) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: no open session on this handle", who);
  if (n < 0 || (n > 0 && (!video || !bytes || !n_bytes || (segmented && !segment))))
    B2_FAIL(h, B2_ERR_BAD_ARG, "%s: bad chunk table (n = %d)", who, n);
  std::vector<int32_t> stream(n);
  for (int i = 0; i < n; ++i) {
    const int k = s->streams.route(who, i, video[i], segmented, segmented ? segment[i] : 0);
    if (k < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "%s", s->streams.err.c_str());
    stream[i] = k;
    if (n_bytes[i] < 0)
      B2_FAIL(h, B2_ERR_BAD_ARG, "%s: chunk %d: n_bytes = %lld < 0", who, i, (long long)n_bytes[i]);
    if (n_bytes[i] > 0 && !bytes[i])
      B2_FAIL(h, B2_ERR_BAD_ARG, "%s: chunk %d: null bytes with n_bytes = %lld", who, i, (long long)n_bytes[i]);
  }
  for (int i = 0; i < n; ++i) s->streams.touched[video[i]] = 1;
  if (const int st = ingest_enqueue(h, s, n, stream.data(), bytes, n_bytes, false)) {
    ingest_release_ref(h, s);   // the planner ran ahead of what reached the device: the session cannot go on
    return st;
  }
  return B2_OK;
}

extern "C" int b2_ingest_push(b2_handle h, int n, const int32_t* video, const void* const* bytes,
                              const int64_t* n_bytes) {
  B2_ENTER(h);
  B2Range range("b2_ingest_push");
  return ingest_push_any(h, "ingest_push", n, video, false, nullptr, bytes, n_bytes);
}

extern "C" int b2_ingest_push_segments(b2_handle h, int n, const int32_t* video, const int64_t* segment,
                                       const void* const* bytes, const int64_t* n_bytes) {
  B2_ENTER(h);
  B2Range range("b2_ingest_push_segments");
  return ingest_push_any(h, "ingest_push_segments", n, video, true, segment, bytes, n_bytes);
}

extern "C" int b2_ingest_segments(b2_handle h, int P, const int32_t* seg_video, const double* seg_total,
                                  const int64_t* seg_off, const int64_t* seg_start) {
  B2_ENTER(h);
  IngestSession* s = h->ingest;
  if (!s || !s->active) B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_segments: no open session on this handle");
  if (const int st = s->streams.declare(s->req, P, seg_video, seg_total, seg_off, seg_start))
    B2_FAIL(h, st, "%s", s->streams.err.c_str());
  // one stream per segment, its region sized from its video's hint; a segment video's own region is released
  const int V = s->V, NS = s->streams.streams();
  s->plan.add_streams(NS - V);
  s->held.resize(NS);
  std::vector<int64_t> cap(s->cap), written(s->plan.frames);
  cap.resize(NS, 0);
  for (int i = 0; i < P; ++i) {
    const int v = seg_video[i];
    cap[v] = 0;
    for (int64_t k = V + s->streams.first[i]; k < V + s->streams.first[i + 1]; ++k) cap[k] = s->hint[v];
  }
  if (const int st = ingest_relayout(h, s, cap, written)) {
    ingest_release_ref(h, s);
    return st;
  }
  return B2_OK;
}

extern "C" int b2_ingest_drop_segment(b2_handle h, int video, int64_t segment) {
  B2_ENTER(h);
  IngestSession* s = h->ingest;
  if (!s || !s->active) B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_drop_segment: no open session on this handle");
  const int k = s->streams.segment("ingest_drop_segment", -1, video, segment);
  if (k < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "%s", s->streams.err.c_str());
  s->streams.dropped[k - s->V] = 1;   // its frames stay where they are; the sync reads none of them
  s->held[k].clear();
  s->held[k].shrink_to_fit();
  return B2_OK;
}

extern "C" int b2_ingest_windows(b2_handle h, int64_t* windows) {
  B2_ENTER(h);
  IngestSession* s = h->ingest;
  if (!s || !s->active) B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_windows: no open session on this handle");
  if (!windows && s->V > 0) B2_FAIL(h, B2_ERR_BAD_ARG, "ingest_windows: null windows");
  for (int v = 0; v < s->V; ++v) windows[v] = s->streams.windows(s->plan, v);
  return B2_OK;
}

extern "C" int b2_ingest_abort(b2_handle h) {
  B2_ENTER(h);
  if (h->ingest) ingest_release_ref(h, h->ingest);
  return B2_OK;
}

// b2_ingest_sync_refs: the reference tables in the order b2_sync_tracks_sig takes them (any group may be NULL), then
// b2_ingest_sync_tracks' arguments; b2_ingest_sync_tracks is this call with every table NULL.
extern "C" int b2_ingest_sync_refs(b2_handle h, const uint8_t* ref_is_subs, const double* ref_cue_start_s,
                                   const double* ref_cue_end_s, const uint8_t* ref_cue_keep, const int64_t* ref_cue_off,
                                   const uint8_t* ref_is_pgs, const double* pgs_start_s, const double* pgs_end_s,
                                   const int64_t* pgs_off, const uint8_t* ref_is_sig, const double* x,
                                   const int64_t* sig_off, const int32_t* track_video, int T, const double* cue_start_s,
                                   const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off,
                                   const double* ratios, int K, double start_seconds, int64_t max_offset_samples,
                                   double* best_score, int32_t* best_offset, int32_t* best_k, double* all_score,
                                   int32_t* all_offset, double* gss_ratio, double* gss_evals, int memspace) {
  B2_ENTER(h);
  B2Range range("b2_ingest_sync_refs");
  const bool tables = ref_is_subs || ref_cue_off || ref_is_pgs || pgs_off || ref_is_sig || sig_off;
  // b2_ingest_sync_tracks keeps its own name in its messages
  const char* who = tables ? "ingest_sync_refs" : "ingest_sync_tracks";
  IngestSession* s = h->ingest;
  if (!s || !s->active) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: no open session on this handle", who);
  // the session closes whatever the outcome
  struct Close {
    b2_ctx* h;
    IngestSession* s;
    ~Close() { ingest_release_ref(h, s); }
  } close{h, s};
  if (T > 0 && !track_video) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: null track_video", who);
  if (!gss_ratio && gss_evals) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: gss_evals without gss_ratio", who);
  if (memspace != B2_HOST && memspace != B2_DEVICE)
    B2_FAIL(h, B2_ERR_BAD_ARG, "%s: memspace must be B2_HOST or B2_DEVICE", who);
  if (ref_is_subs && !ref_cue_off) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: ref_is_subs without ref_cue_off", who);
  if (ref_is_pgs && !pgs_off) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: ref_is_pgs without pgs_off", who);
  if (ref_is_sig && !sig_off) B2_FAIL(h, B2_ERR_BAD_ARG, "%s: ref_is_sig without sig_off", who);
  const int V = s->V;
  SyncRequest r = s->req;
  r.who = gss_ratio ? (tables ? "ingest_sync_refs (search)" : "ingest_sync_tracks (search)") : who;
  r.refs = {ref_is_subs, ref_cue_start_s, ref_cue_end_s, ref_cue_keep, V > 0 ? ref_cue_off : nullptr};
  r.pgs = {ref_is_pgs, pgs_start_s, pgs_end_s, V > 0 ? pgs_off : nullptr};
  r.sig = {ref_is_sig, x, V > 0 ? sig_off : nullptr};
  // a reference video has no audio: P_v must be empty (plan_refs_check compares pcm_off, all equal in a session)
  r.V = V;
  if (const int st = ingest_refs_check(r, &s->streams, s->plan)) B2_FAIL(h, st, "%s", s->streams.err.c_str());
  B2_TRY(ingest_enqueue(h, s, 0, nullptr, nullptr, nullptr, true));
  std::vector<int64_t> pcm_off(V + 1, 0);
  // the live segments' table: b2_sync_tracks_seg's, its sample ranges empty (the detector's output is on the
  // device), each segment's frames in the session's buffer
  const IngestStreams& ss = s->streams;
  const int P = (int)ss.video.size();
  std::vector<int64_t> seg_off(1, 0), seg_start, seg_at, seg_len;
  for (int i = 0; i < P; ++i) {
    for (int64_t j = ss.first[i]; j < ss.first[i + 1]; ++j)
      if (!ss.dropped[j]) {
        seg_start.push_back(ss.start[j]);
        seg_at.push_back(s->at[V + j]);
        seg_len.push_back(s->plan.frames[V + j]);
      }
    seg_off.push_back((int64_t)seg_start.size());
  }
  const std::vector<int64_t> no_range(seg_start.size() + 1, 0);
  r.pcm = nullptr;
  r.pcm_off = pcm_off.data();
  r.V = V;
  r.track_video = track_video;
  r.T = T;
  r.cue_start_s = cue_start_s;
  r.cue_end_s = cue_end_s;
  r.cue_keep = cue_keep;
  r.cue_off = cue_off;
  r.ratios = ratios;
  r.K = K;
  r.start_seconds = start_seconds;
  r.max_offset_samples = max_offset_samples;
  r.best_score = best_score;
  r.best_offset = best_offset;
  r.best_k = best_k;
  r.all_score = all_score;
  r.all_offset = all_offset;
  r.search = gss_ratio != nullptr;
  r.gss_ratio = gss_ratio;
  r.gss_evals = gss_evals;
  r.memspace = memspace;
  r.ready = {s->ref, s->at.data(), s->plan.frames.data(), seg_at.data(), seg_len.data()};
  if (ss.declared)
    r.seg = {P, ss.video.data(), ss.total.data(), seg_off.data(), seg_start.data(), no_range.data(), no_range.data()};
  return sync_run(h, _b2_fence_was_valid, r);
}

extern "C" int b2_ingest_sync_tracks(b2_handle h, const int32_t* track_video, int T, const double* cue_start_s,
                                     const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off,
                                     const double* ratios, int K, double start_seconds, int64_t max_offset_samples,
                                     double* best_score, int32_t* best_offset, int32_t* best_k, double* all_score,
                                     int32_t* all_offset, double* gss_ratio, double* gss_evals, int memspace) {
  return b2_ingest_sync_refs(h, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                             nullptr, nullptr, nullptr, track_video, T, cue_start_s, cue_end_s, cue_keep, cue_off,
                             ratios, K, start_seconds, max_offset_samples, best_score, best_offset, best_k, all_score,
                             all_offset, gss_ratio, gss_evals, memspace);
}

// ---- try_sync's epilogue (sync_output.cu) ----------------------------------------------------------------------
extern "C" int b2_apply_sync(b2_handle h, const double* best_score, const int32_t* best_offset, const int32_t* best_k,
                             const double* gss_ratio, int T, const double* cue_start_s, const double* cue_end_s,
                             const int64_t* cue_off, const double* ratios, int K, int sample_rate,
                             double apply_offset_seconds, int gate_enabled, double min_score,
                             double quality_max_offset_seconds, double max_framerate_deviation, int has_suppress,
                             double suppress_output_if_offset_less_than, int64_t* synced_start_us,
                             int64_t* synced_end_us, double* offset_seconds, double* scale, int32_t* status,
                             int memspace) {
  // Not B2_ENTER: this call only reads outputs already ordered on the handle's stream and writes none of the
  // buffers a sync call keeps between calls, so a chain of resident sync calls stays valid across it.
  if (!h) return B2_ERR_BAD_ARG;
  h->err.clear();
  DeviceScope scope(h->device);
  if (!scope.ok) return B2_ERR_CUDA;
  if (T < 0 || K < 0 || !cue_off) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: bad arguments (T %d, K %d)", T, K);
  if (sample_rate <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: sample_rate %d <= 0", sample_rate);
  if (!std::isfinite(apply_offset_seconds))
    B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: apply_offset_seconds %g is not finite", apply_offset_seconds);
  if (T == 0) return B2_OK;
  if (!best_score || !best_offset || !best_k) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: null best_score / offset / k");
  if (!offset_seconds || !scale || !status) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: null offset_seconds / scale / status");
  if (K && !ratios) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: null ratios");
  if (cue_off[0] < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: cue_off[0] %lld < 0", (long long)cue_off[0]);
  for (int t = 0; t < T; ++t)
    if (cue_off[t + 1] < cue_off[t]) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: cue_off not monotone at track %d", t);
  const int64_t c0 = cue_off[0], n = cue_off[T] - c0;
  if (n && (!cue_start_s || !cue_end_s)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: null cue times");
  if (n && (!synced_start_us || !synced_end_us)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: null synced_start_us / end_us");
  double smax = gss_ratio ? 1.1 : 1.0;
  for (int k = 0; k < K; ++k) {
    if (!std::isfinite(ratios[k])) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_sync: ratio %d (%g) is not finite", k, ratios[k]);
    smax = std::max(smax, fabs(ratios[k]));
  }
  // every output time is at most |t| * smax + |shift| in magnitude, |shift| <= 2^31 / sample_rate + |apply|: cue
  // times below this bound stay where the microsecond arithmetic is exact (checked while they are uploaded)
  const double t_max = (B2_MAX_CUE_SECONDS - 2147483648.0 / sample_rate - fabs(apply_offset_seconds)) / smax;
  B2_CHECK_DEV(h, memspace, best_score, "apply_sync: best_score");
  B2_CHECK_DEV(h, memspace, best_offset, "apply_sync: best_offset");
  B2_CHECK_DEV(h, memspace, best_k, "apply_sync: best_k");
  B2_CHECK_DEV(h, memspace, gss_ratio, "apply_sync: gss_ratio");
  B2_CHECK_DEV(h, memspace, offset_seconds, "apply_sync: offset_seconds");
  B2_CHECK_DEV(h, memspace, scale, "apply_sync: scale");
  B2_CHECK_DEV(h, memspace, status, "apply_sync: status");
  if (n) {
    B2_CHECK_DEV(h, memspace, synced_start_us, "apply_sync: synced_start_us");
    B2_CHECK_DEV(h, memspace, synced_end_us, "apply_sync: synced_end_us");
  }
  const B2SyncRule rule = b2_sync_rule(sample_rate, apply_offset_seconds, gate_enabled, min_score,
                                       quality_max_offset_seconds, max_framerate_deviation, has_suppress,
                                       suppress_output_if_offset_less_than);
  if (memspace == B2_DEVICE)
    return b2i_apply_sync_launch(h, best_score, best_offset, best_k, gss_ratio, T, cue_start_s, cue_end_s, cue_off,
                                 t_max, ratios, K, rule, synced_start_us, synced_end_us, offset_seconds, scale, status);
  // B2_HOST: inputs and outputs staged through the workspaces; cue outputs at their absolute indices
  void *din, *dout;
  const size_t Ts = (size_t)T;
  B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_IN0, Ts * 24 + 64, &din));
  B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)n * 16 + Ts * 20 + 64, &dout));
  double* d_bs = (double*)din;
  double* d_gss = gss_ratio ? d_bs + Ts : nullptr;
  int32_t* d_bo = (int32_t*)(d_bs + 2 * Ts);
  int32_t* d_bk = d_bo + Ts;
  B2_CUDA(h, cudaMemcpyAsync(d_bs, best_score, Ts * 8, cudaMemcpyHostToDevice, h->stream));
  if (gss_ratio) B2_CUDA(h, cudaMemcpyAsync(d_gss, gss_ratio, Ts * 8, cudaMemcpyHostToDevice, h->stream));
  B2_CUDA(h, cudaMemcpyAsync(d_bo, best_offset, Ts * 4, cudaMemcpyHostToDevice, h->stream));
  B2_CUDA(h, cudaMemcpyAsync(d_bk, best_k, Ts * 4, cudaMemcpyHostToDevice, h->stream));
  int64_t* d_su = (int64_t*)dout;
  int64_t* d_eu = d_su + n;
  double* d_off = (double*)(d_eu + n);
  double* d_sc = d_off + Ts;
  int32_t* d_st = (int32_t*)(d_sc + Ts);
  B2_TRY(b2i_apply_sync_launch(h, d_bs, d_bo, d_bk, d_gss, T, cue_start_s, cue_end_s, cue_off, t_max, ratios, K, rule,
                               d_su - c0, d_eu - c0, d_off, d_sc, d_st));
  B2_TRY(copy_out(h, synced_start_us + c0, d_su, (size_t)n * 8));
  B2_TRY(copy_out(h, synced_end_us + c0, d_eu, (size_t)n * 8));
  B2_TRY(copy_out(h, offset_seconds, d_off, Ts * 8));
  B2_TRY(copy_out(h, scale, d_sc, Ts * 8));
  B2_TRY(copy_out(h, status, d_st, Ts * 4));
  B2_CUDA(h, cudaStreamSynchronize(h->stream));
  return B2_OK;
}

// ---- per-segment offsets with a split penalty (split.cu, sync_output.cu) ---------------------------------------
// b2_split_tracks, b2_split_tracks_wide, b2_split_tracks_capped, b2_split_tracks_directed and b2_split_tracks_breaks:
// the same checks and outputs, wide: the wider envelope; max_segments > 0 (capped, wide set): at most that many segments and
// split_profile [T x max_segments]; directed (wide set): offsets monotone in direction +1 or -1; broken (wide set):
// at most n_breaks breaks in the stated directions and split_profile [T x (n_breaks + 1)]
static int split_tracks(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off, int V,
                        const int32_t* track_video, int T, const double* cue_start_s, const double* cue_end_s,
                        const uint8_t* cue_keep, const int64_t* cue_off, const double* ratio, int sample_rate,
                        double start_seconds, int64_t max_offset_samples, double split_penalty, int32_t* cue_offset,
                        int32_t* n_segments, double* split_score, int memspace, bool wide, bool capped = false,
                        int max_segments = 0, double* split_profile = nullptr, bool directed = false,
                        int direction = 0, bool broken = false, const int32_t* breaks = nullptr, int n_breaks = 0) {
  B2_ENTER(h);
  if (V < 0 || T < 0 || !ref_off || !cue_off || (T && (!track_video || !ratio)))
    B2_FAIL(h, B2_ERR_BAD_ARG, "split: bad arguments (V %d, T %d, null table)", V, T);
  if (memspace != B2_HOST && memspace != B2_DEVICE) B2_FAIL(h, B2_ERR_BAD_ARG, "split: memspace must be B2_HOST or B2_DEVICE");
  if (std::isnan(split_penalty) || split_penalty < 0)
    B2_FAIL(h, B2_ERR_BAD_ARG, "split: split_penalty %g must be >= 0 (+inf: no splits)", split_penalty);
  if (capped && max_segments < 1) B2_FAIL(h, B2_ERR_BAD_ARG, "split: max_segments %d must be >= 1", max_segments);
  if (directed && direction != 1 && direction != -1)
    B2_FAIL(h, B2_ERR_BAD_ARG, "split: direction %d must be +1 (offsets only grow) or -1 (only shrink)", direction);
  if (broken) {
    if (n_breaks < 1 || !breaks)
      B2_FAIL(h, B2_ERR_BAD_ARG, "split: n_breaks %d must be >= 1 (with a breaks list)", n_breaks);
    for (int i = 0; i < n_breaks; ++i)
      if (breaks[i] != 1 && breaks[i] != -1)
        B2_FAIL(h, B2_ERR_BAD_ARG, "split: breaks[%d] = %d must be +1 (the offset grows) or -1 (it shrinks)", i,
                breaks[i]);
    if (n_breaks > 15)  // split::kMaxBreaks: 16 layers of split_breaks_dp_kernel
      B2_FAIL(h, B2_ERR_UNSUPPORTED, "split: %d breaks is more than 15", n_breaks);
  }
  if (sample_rate <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "split: sample_rate %d <= 0", sample_rate);
  if (ref_off[0] < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "split: ref_off[0] %lld < 0", (long long)ref_off[0]);
  for (int v = 0; v < V; ++v) {
    if (ref_off[v + 1] < ref_off[v]) B2_FAIL(h, B2_ERR_BAD_ARG, "split: ref_off not monotone at video %d", v);
    if (ref_off[v + 1] - ref_off[v] > 0x3fffffff)
      B2_FAIL(h, B2_ERR_BAD_ARG, "split: video %d: reference of %lld frames (at most 2^30 - 1)", v,
              (long long)(ref_off[v + 1] - ref_off[v]));
  }
  if (cue_off[0] < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "split: cue_off[0] %lld < 0", (long long)cue_off[0]);
  for (int t = 0; t < T; ++t) {
    if (cue_off[t + 1] < cue_off[t]) B2_FAIL(h, B2_ERR_BAD_ARG, "split: cue_off not monotone at track %d", t);
    if (track_video[t] < 0 || track_video[t] >= V)
      B2_FAIL(h, B2_ERR_BAD_ARG, "split: track %d: video %d is outside [0, %d)", t, track_video[t], V);
    if (!std::isnan(ratio[t]) && !ratio_ok(ratio[t]))
      B2_FAIL(h, B2_ERR_BAD_ARG, "split: track %d: ratio %g is not a finite positive number (NaN skips)", t, ratio[t]);
  }
  if (T == 0) return B2_OK;
  const int64_t c0 = cue_off[0], n = cue_off[T] - c0;
  if (n && (!cue_start_s || !cue_end_s)) B2_FAIL(h, B2_ERR_BAD_ARG, "split: null cue times");
  if (!n_segments || !split_score || (n && !cue_offset)) B2_FAIL(h, B2_ERR_BAD_ARG, "split: null output");
  if ((capped || broken) && !split_profile) B2_FAIL(h, B2_ERR_BAD_ARG, "split: null split_profile");
  if (ref_off[V] > ref_off[0] && !ref) B2_FAIL(h, B2_ERR_BAD_ARG, "split: null ref");
  // the masks' lengths at each track's ratio (skipped tracks at 1.0), every cue time checked as b2_rasterize does
  std::vector<double> r1(T);
  for (int t = 0; t < T; ++t) r1[t] = std::isnan(ratio[t]) ? 1.0 : ratio[t];
  std::vector<int64_t> len(T);
  if (!(fabs(start_seconds) < B2_MAX_CUE_SECONDS) ||
      rasterize_lengths(cue_start_s, cue_end_s, cue_off, T, r1.data(), 1, 1, sample_rate, len.data()) != B2_OK) {
    int64_t at;
    double val;
    const char* why = bad_cue_input(cue_start_s, cue_end_s, cue_off, T, r1.data(), 1, 1, start_seconds, &at, &val);
    B2_FAIL(h, B2_ERR_BAD_ARG, "split: %s (index %lld: %g)", why ? why : "bad cue list", (long long)at, val);
  }
  for (int t = 0; t < T; ++t)
    if (len[t] > 0x3fffffff) B2_FAIL(h, B2_ERR_BAD_ARG, "split: track %d: mask of %lld frames", t, (long long)len[t]);
  B2_CHECK_DEV(h, memspace, ref, "split: ref");
  B2_CHECK_DEV(h, memspace, cue_offset, "split: cue_offset");
  B2_CHECK_DEV(h, memspace, n_segments, "split: n_segments");
  B2_CHECK_DEV(h, memspace, split_score, "split: split_score");
  if (capped || broken) B2_CHECK_DEV(h, memspace, split_profile, "split: split_profile");
  const int N = capped ? max_segments : broken ? n_breaks + 1 : 0;  // profile columns
  const size_t esz = ref_is_f64 ? 8 : 4;
  if (memspace == B2_DEVICE)
    return b2i_split_launch(h, ref, ref_is_f64 != 0, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep,
                            cue_off, ratio, len.data(), sample_rate, start_seconds, max_offset_samples, split_penalty,
                            false, nullptr, false, wide, cue_offset, n_segments, split_score, capped ? N : 0,
                            split_profile, directed ? direction : 0, breaks, broken ? n_breaks : 0);
  // B2_HOST: the reference staged in, outputs through the staging workspace (cue outputs at their absolute indices)
  void *d_ref, *dout;
  B2_TRY(stage_in(h, b2_ctx::WS_STAGE_IN0, ref, (size_t)ref_off[V] * esz, &d_ref));
  const size_t Ts = (size_t)T;
  B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, Ts * 12 + Ts * N * 8 + (size_t)n * 4 + 64, &dout));
  double* d_sc = (double*)dout;
  double* d_pr = d_sc + Ts;  // [T x N] (capped, breaks)
  int32_t* d_ns = (int32_t*)(d_pr + Ts * N);
  int32_t* d_co = d_ns + Ts;
  B2_TRY(b2i_split_launch(h, d_ref, ref_is_f64 != 0, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep,
                          cue_off, ratio, len.data(), sample_rate, start_seconds, max_offset_samples, split_penalty,
                          true, ref, ref_is_f64 != 0, wide, d_co - c0, d_ns, d_sc, capped ? N : 0, d_pr,
                          directed ? direction : 0, breaks, broken ? n_breaks : 0));
  B2_TRY(copy_out(h, cue_offset + c0, d_co, (size_t)n * 4));
  B2_TRY(copy_out(h, n_segments, d_ns, Ts * 4));
  B2_TRY(copy_out(h, split_score, d_sc, Ts * 8));
  if (capped || broken) B2_TRY(copy_out(h, split_profile, d_pr, Ts * N * 8));
  B2_CUDA(h, cudaStreamSynchronize(h->stream));
  return B2_OK;
}

extern "C" int b2_split_tracks(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off, int V,
                               const int32_t* track_video, int T, const double* cue_start_s, const double* cue_end_s,
                               const uint8_t* cue_keep, const int64_t* cue_off, const double* ratio, int sample_rate,
                               double start_seconds, int64_t max_offset_samples, double split_penalty,
                               int32_t* cue_offset, int32_t* n_segments, double* split_score, int memspace) {
  return split_tracks(h, ref, ref_is_f64, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep, cue_off, ratio,
                      sample_rate, start_seconds, max_offset_samples, split_penalty, cue_offset, n_segments,
                      split_score, memspace, false);
}

extern "C" int b2_split_tracks_wide(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off, int V,
                                    const int32_t* track_video, int T, const double* cue_start_s,
                                    const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off,
                                    const double* ratio, int sample_rate, double start_seconds,
                                    int64_t max_offset_samples, double split_penalty, int32_t* cue_offset,
                                    int32_t* n_segments, double* split_score, int memspace) {
  return split_tracks(h, ref, ref_is_f64, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep, cue_off, ratio,
                      sample_rate, start_seconds, max_offset_samples, split_penalty, cue_offset, n_segments,
                      split_score, memspace, true);
}

extern "C" int b2_split_tracks_capped(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off, int V,
                                      const int32_t* track_video, int T, const double* cue_start_s,
                                      const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off,
                                      const double* ratio, int sample_rate, double start_seconds,
                                      int64_t max_offset_samples, double split_penalty, int max_segments,
                                      int32_t* cue_offset, int32_t* n_segments, double* split_score,
                                      double* split_profile, int memspace) {
  return split_tracks(h, ref, ref_is_f64, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep, cue_off, ratio,
                      sample_rate, start_seconds, max_offset_samples, split_penalty, cue_offset, n_segments,
                      split_score, memspace, true, true, max_segments, split_profile);
}

extern "C" int b2_split_tracks_directed(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off, int V,
                                        const int32_t* track_video, int T, const double* cue_start_s,
                                        const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off,
                                        const double* ratio, int sample_rate, double start_seconds,
                                        int64_t max_offset_samples, double split_penalty, int direction,
                                        int32_t* cue_offset, int32_t* n_segments, double* split_score, int memspace) {
  return split_tracks(h, ref, ref_is_f64, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep, cue_off, ratio,
                      sample_rate, start_seconds, max_offset_samples, split_penalty, cue_offset, n_segments,
                      split_score, memspace, true, false, 0, nullptr, true, direction);
}

extern "C" int b2_split_tracks_breaks(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off, int V,
                                      const int32_t* track_video, int T, const double* cue_start_s,
                                      const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off,
                                      const double* ratio, int sample_rate, double start_seconds,
                                      int64_t max_offset_samples, double split_penalty, const int32_t* breaks,
                                      int n_breaks, int32_t* cue_offset, int32_t* n_segments, double* split_score,
                                      double* split_profile, int memspace) {
  return split_tracks(h, ref, ref_is_f64, ref_off, V, track_video, T, cue_start_s, cue_end_s, cue_keep, cue_off, ratio,
                      sample_rate, start_seconds, max_offset_samples, split_penalty, cue_offset, n_segments,
                      split_score, memspace, true, false, 0, split_profile, false, 0, true, breaks, n_breaks);
}

extern "C" int b2_apply_split(b2_handle h, const double* ratio, const int32_t* n_segments, const int32_t* cue_offset,
                              int T, const double* cue_start_s, const double* cue_end_s, const int64_t* cue_off,
                              int sample_rate, double apply_offset_seconds, int64_t* synced_start_us,
                              int64_t* synced_end_us, int32_t* status, int memspace) {
  // Not B2_ENTER, as b2_apply_sync: a chain of resident sync calls stays valid across it
  if (!h) return B2_ERR_BAD_ARG;
  h->err.clear();
  DeviceScope scope(h->device);
  if (!scope.ok) return B2_ERR_CUDA;
  if (T < 0 || !cue_off || (T && !ratio)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: bad arguments (T %d)", T);
  if (sample_rate <= 0) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: sample_rate %d <= 0", sample_rate);
  if (!std::isfinite(apply_offset_seconds))
    B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: apply_offset_seconds %g is not finite", apply_offset_seconds);
  if (T == 0) return B2_OK;
  if (!n_segments || !status) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: null n_segments / status");
  if (cue_off[0] < 0) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: cue_off[0] %lld < 0", (long long)cue_off[0]);
  double smax = 1.0;
  for (int t = 0; t < T; ++t) {
    if (cue_off[t + 1] < cue_off[t]) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: cue_off not monotone at track %d", t);
    if (!std::isnan(ratio[t]) && !ratio_ok(ratio[t]))
      B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: track %d: ratio %g is not a finite positive number", t, ratio[t]);
    if (!std::isnan(ratio[t])) smax = std::max(smax, ratio[t]);
  }
  const int64_t c0 = cue_off[0], n = cue_off[T] - c0;
  if (n && (!cue_start_s || !cue_end_s || !cue_offset)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: null cue input");
  if (n && (!synced_start_us || !synced_end_us)) B2_FAIL(h, B2_ERR_BAD_ARG, "apply_split: null synced_start_us / end_us");
  // as b2_apply_sync: every output time is at most |t| * smax + 2^31 / sample_rate + |apply| in magnitude
  const double t_max = (B2_MAX_CUE_SECONDS - 2147483648.0 / sample_rate - fabs(apply_offset_seconds)) / smax;
  B2_CHECK_DEV(h, memspace, n_segments, "apply_split: n_segments");
  B2_CHECK_DEV(h, memspace, status, "apply_split: status");
  if (n) {
    B2_CHECK_DEV(h, memspace, cue_offset, "apply_split: cue_offset");
    B2_CHECK_DEV(h, memspace, synced_start_us, "apply_split: synced_start_us");
    B2_CHECK_DEV(h, memspace, synced_end_us, "apply_split: synced_end_us");
  }
  const B2SyncRule rule = b2_sync_rule(sample_rate, apply_offset_seconds, 0, 0.0, 0.0, 0.0, 0, 0.0);
  if (memspace == B2_DEVICE)
    return b2i_apply_split_launch(h, ratio, n_segments, cue_offset, T, cue_start_s, cue_end_s, cue_off, t_max, rule,
                                  synced_start_us, synced_end_us, status);
  void *din, *dout;
  const size_t Ts = (size_t)T;
  B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_IN0, Ts * 4 + (size_t)n * 4 + 64, &din));
  B2_TRY(b2i_ws(h, b2_ctx::WS_STAGE_OUT, (size_t)n * 16 + Ts * 4 + 64, &dout));
  int32_t* d_ns = (int32_t*)din;
  int32_t* d_co = d_ns + Ts;
  B2_CUDA(h, cudaMemcpyAsync(d_ns, n_segments, Ts * 4, cudaMemcpyHostToDevice, h->stream));
  if (n) B2_CUDA(h, cudaMemcpyAsync(d_co, cue_offset + c0, (size_t)n * 4, cudaMemcpyHostToDevice, h->stream));
  int64_t* d_su = (int64_t*)dout;
  int64_t* d_eu = d_su + n;
  int32_t* d_st = (int32_t*)(d_eu + n);
  B2_TRY(b2i_apply_split_launch(h, ratio, d_ns, d_co - c0, T, cue_start_s, cue_end_s, cue_off, t_max, rule, d_su - c0,
                                d_eu - c0, d_st));
  B2_TRY(copy_out(h, synced_start_us + c0, d_su, (size_t)n * 8));
  B2_TRY(copy_out(h, synced_end_us + c0, d_eu, (size_t)n * 8));
  B2_TRY(copy_out(h, status, d_st, Ts * 4));
  B2_CUDA(h, cudaStreamSynchronize(h->stream));
  return B2_OK;
}
