// Shared plumbing for the ffsubsync hot-path library (internal; the ABI is
// include/ffsubsync_b200.h).  sm_90a (H100) only.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "../../include/ffsubsync_b200.h"

// NVTX range per stage (header-only nvtx3: a no-op costing one pointer test unless a profiler is
// attached).  Shows up in ncu / nsys timelines as vad / raster_bits / ref_spectra+correlate / ...
struct B2Range {
  explicit B2Range(const char* name) { nvtxRangePushA(name); }
  ~B2Range() { nvtxRangePop(); }
};

struct DeviceBuf {
  void* p = nullptr;
  size_t cap = 0;
};

struct HostBuf {  // pinned
  void* p = nullptr;
  size_t cap = 0;
};

// b2_capture_nominations: caller-owned device arrays the aligner copies its nomination stage into
struct B2Capture {
  float* scores = nullptr;  // nullptr: capture off
  long long stride = 0;
  long long* win = nullptr;
  float* stat = nullptr;
  int* cand = nullptr;
};

// b2_capture_reference: where the batched sync calls copy their reference-signal buffer.  Unlike B2Capture it
// is read only after the call's plan is made and its launches are enqueued, so it changes neither.
struct B2RefCapture {
  float* ref = nullptr;       // device, `capacity` floats; nullptr: capture off
  long long capacity = 0;
  int64_t* ref_off = nullptr; // host, max_videos + 1 entries
  uint8_t* packed = nullptr;  // host, max_videos entries
  long long max_videos = 0;
};

// b2_speech_output: where the batched sync calls write the listed videos' reference signals as float64.  Like
// B2RefCapture it is read after the call's plan is made; setting or clearing it enqueues nothing.
struct B2SpeechOut {
  double* speech = nullptr;      // `capacity` doubles in `memspace`; nullptr: output off
  long long capacity = 0;
  std::vector<int> videos;       // increasing
  int64_t* speech_off = nullptr; // host, videos.size() + 1 entries, written by each call
  int memspace = 0;
};

struct b2_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  std::string err;
  int64_t launches = 0;
  int split_max_cluster = 0;     // widest split_dp_kernel cluster the device co-schedules (0: not queried yet)
  int split_capped_max_cluster = 0;  // the same for split_capped_dp_kernel
  int split_directed_max_cluster = 0;  // the same for split_directed_dp_kernel (both directions)
  int split_breaks_max_cluster[8] = {};  // the same for split_breaks_dp_kernel<16, 10, 8, 6, 5, 4, 3, 2>
  uint64_t log2_quirk_mask = 0;  // bit k set: CPython's ceil(math.log(2**k, 2)) == k + 1
  int vad_partition_sms = 0;     // > 0: the lane-per-window VAD runs at most this many CTAs (one per SM)
  B2Capture capture;             // set by b2_capture_nominations (tests)
  B2RefCapture ref_capture;      // set by b2_capture_reference (tests)
  B2SpeechOut speech_out;        // set by b2_speech_output
  // B2_DEVICE_RESIDENT chaining of b2_sync_batch calls (api.cu): `resident_fence` is recorded on the caller's
  // stream before the LAST sub-batch's correlation chain of a pipelined call, `resident_done` after it; the
  // next resident call (if no other entry point ran in between: `resident_fence_valid`) starts its VAD behind
  // the fence instead of behind the whole stream and writes the other reference-signal buffer
  bool resident_fence_valid = false;
  cudaEvent_t resident_fence = nullptr, resident_done = nullptr;
  int refsig_parity = 0;
  // named grow-only workspaces
  enum { WS_STAGE_IN0, WS_STAGE_IN1, WS_STAGE_OUT, WS_META, WS_SPEC, WS_SCORES, WS_CAND,
         WS_SIG_REF, WS_SIG_REF2, WS_SIG_SUB, WS_MISC, WS_COUNTERS, WS_RUNS, WS_GSS, WS_GSS_OUT, WS_STAGE_SIG,
         WS_SPEECH, WS_SPLIT, WS_COUNT };
  DeviceBuf ws[WS_COUNT];
  HostBuf pinned[4];
  cudaEvent_t pinned_ev[4] = {};   // recorded after the last async copy out of pinned[i]
  // ring of metadata upload buffers (see b2i_meta_begin)
  static const int kMetaSlots = 8;
  struct MetaSlot {
    void* d = nullptr;
    void* p = nullptr;
    size_t cap = 0;
    cudaEvent_t ev = nullptr;
  };
  // one ring per stream the handle launches on (the in-order reuse argument is per stream)
  MetaSlot meta[2][kMetaSlots];
  uint64_t meta_seq[2] = {0, 0};
  int ring = 0;                    // ring in use: 0 = caller-facing stream, 1 = internal stream2
  // b2_sync_batch overlaps the VAD of sub-batch i+1 (stream2) with the alignment of sub-batch i
  // (stream); events from a small pool order the two
  // b2_vad_stream_*: ring of pinned/device chunk buffers (H2D + kernel + D2H of chunk i in flight
  // while the caller produces chunk i+1)
  struct VadStream {
    static const int kSlots = 3;
    struct Slot {
      void* hp = nullptr;     // pinned PCM
      void* dp = nullptr;     // device PCM
      float* hout = nullptr;  // pinned windows
      float* dout = nullptr;  // device windows
      size_t cap = 0, out_cap = 0;
      cudaEvent_t ev = nullptr;
      int64_t n_out = 0;
      bool busy = false;
    } slot[kSlots];
    bool active = false;
    int frame_rate = 0, sample_rate = 0, fpw = 0, z_lo = 0, z_hi = 0;
    float label = 0.f;
    int64_t thr = 0, windows = 0;
    uint64_t seq = 0;
    std::vector<float> results;
  } vs;
  // b2_ingest_*: the batched ingest session (api.cu), null until the first b2_ingest_begin
  struct IngestSession* ingest = nullptr;
  // pageable B2_HOST inputs: two pinned bounce buffers filled by a few host threads (see stage_in)
  struct Bounce {
    void* p = nullptr;
    cudaEvent_t ev = nullptr;
  } bounce[2];
  cudaStream_t stream2 = nullptr;
  static const int kEvents = 64;
  cudaEvent_t ev_pool[kEvents] = {};
  int ev_next = 0;
};

#define B2_FAIL(h, code, ...)                          \
  do {                                                 \
    char _b[512];                                      \
    snprintf(_b, sizeof(_b), __VA_ARGS__);             \
    (h)->err = _b;                                     \
    return (code);                                     \
  } while (0)

#define B2_CUDA(h, expr)                                                              \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess)                                                            \
      B2_FAIL(h, B2_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
              __FILE__, __LINE__);                                                    \
  } while (0)

#define B2_CHECK_LAUNCH(h, name)                                                         \
  do {                                                                                   \
    (h)->launches++;                                                                     \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess)                                                               \
      B2_FAIL(h, B2_ERR_CUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e));  \
  } while (0)

#define B2_TRY(expr)            \
  do {                          \
    int _s = (expr);            \
    if (_s != B2_OK) return _s; \
  } while (0)

int b2i_ws(b2_ctx* h, int which, size_t bytes, void** out);
int b2i_pinned(b2_ctx* h, int which, size_t bytes, void** out);
// Upload a small host array into the META workspace region (async on h->stream).
struct MetaArena {
  b2_ctx* h;
  char* dbase = nullptr;
  char* hbase = nullptr;
  size_t cap = 0, used = 0;
  int slot = 0, ring = 0;
};
int b2i_meta_begin(b2_ctx* h, MetaArena* a, size_t bytes);
void* b2i_meta_put(MetaArena* a, const void* src, size_t bytes);  // returns device pointer
void* b2i_meta_reserve(MetaArena* a, size_t bytes, void** host_view);
int b2i_meta_commit(MetaArena* a);

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- kernels' host launchers (defined in the .cu files) ------------------------------------
// e_min_full: smallest sum of squares of a full window that is speech.  tail_emin_host (nullable,
// [B]): evaluate each signal's trailing partial window against its own floor (auditok contract);
// null = partial windows are non-speech (webrtc contract).
// packed (lane-per-window kernel only, B2_ERR_UNSUPPORTED otherwise): instead of the floats, the bits
// m = (r == 1.0f) of every window, 32 to a word; signal b's words start at d_out + out_off_host[b] (read as
// uint32), ceil(windows / 32) of them, with zero bits past its last window.
// pcm_end_host (nullable, [B]): signal b spans pcm_off_host[b] .. pcm_end_host[b] (signals with gaps between them, or
// overlapping: the sampled segments of b2_sync_tracks_seg); null = pcm_off_host[b + 1].  Lane eligibility (8-sample
// aligned starts) is decided per non-empty signal either way.
bool b2i_vad_lane_eligible(const int64_t* pcm_off_host, int B, int fpw);
int b2i_vad_launch(b2_ctx* h, const int16_t* d_pcm, const int64_t* pcm_off_host, int B, int fpw,
                   float non_speech_label, int64_t e_min_full, int z_lo, int z_hi,
                   float* d_out, const int64_t* out_off_host, const int64_t* tail_emin_host = nullptr,
                   bool packed = false, const int64_t* pcm_end_host = nullptr);
struct B2TokenizerParams {
  double min_length, max_continuous_silence, non_speech_label;
  long long max_length;
};
// flags / out share the offset table off_host[n_chunks + 1] (one detector call per chunk)
int b2i_tokenize_launch(b2_ctx* h, const float* d_flags, const int64_t* off_host, int n_chunks,
                        const B2TokenizerParams& tp, double* d_out);
// The same scan writing float32 over its own flags (the energy pass's label-0 output): the reference
// signal of b2_sync_tracks_auditok, built in place in the reference-signal buffer.  end_host (nullable,
// [n_chunks]): chunk c spans off_host[c] .. end_host[c] (chunks need not abut: b2_sync_tracks_subs leaves
// the subtitle references' ranges out); null = off_host[c + 1].
int b2i_tokenize_inplace_launch(b2_ctx* h, float* d_flags_sig, const int64_t* off_host, int n_chunks,
                                const B2TokenizerParams& tp, const int64_t* end_host = nullptr);
int b2i_synth_launch(b2_ctx* h, const uint8_t* d_cls, int64_t n_windows, int fpw, uint32_t seed,
                     int16_t* d_out);
int b2i_raster_launch(b2_ctx* h, const double* cue_start, const double* cue_end,
                      const uint8_t* cue_keep, const int64_t* cue_off, int B, const double* ratios,
                      int K, int per_pair_ratios, const double* levels, int sample_rate,
                      double start_seconds, float* d_out, const int64_t* out_off_host);
// Subtitle references of b2_sync_tracks_subs: for each of the n_subs videos videos[i] (indices into the host
// tables cue_off / out_off [n_videos + 1], absolute), zero d_out[out_off[v] .. out_off[v+1]) and write 1.0 over
// its kept cues at ratio 1.0 - b2_rasterize at ratio 1.0 and level 1.0, at per-video bases.  pgs: the lists are
// PGS intervals (b2_sync_tracks_pgs, b2_rasterize_pgs), written by b2_pgs_bounds; cue_keep is not read.
int b2i_raster_ref_launch(b2_ctx* h, const double* cue_start, const double* cue_end, const uint8_t* cue_keep,
                          const int64_t* cue_off, const int64_t* out_off, int n_videos, const int* videos, int n_subs,
                          int sample_rate, double start_seconds, float* d_out, bool pgs = false);
// Signal references of b2_sync_tracks_sig (K1s, sig_ref.cu): for each of the n_sig videos videos[i] (ascending
// indices into the host tables x_off / out_off [n_videos + 1], absolute), write the frames of the stored values
// d_x[x_off[v] ..] (sig_ref.cuh), out_off[v+1] - out_off[v] of them, to d_out + out_off[v]: floats, or with packed
// ceil(R/32) words of the bits m = (r == 1.0f) with zero bits past R.  d_first_bad[v] is reset first and ends as the
// first out-of-domain frame (kSigNoBadFrame: none).  The grid keeps to h->vad_partition_sms SMs when it is set.
int b2i_sig_ref_launch(b2_ctx* h, const double* d_x, const int64_t* x_off, const int64_t* out_off, int n_videos,
                       const int* videos, int n_sig, float label, bool packed, float* d_out,
                       unsigned long long* d_first_bad);
// Sampled-segment references of b2_sync_tracks_seg (K1m, seg_ref.cu): for each of the n_seg videos videos[i]
// (ascending indices into the host table out_off [n_videos + 1]), write every frame of d_out + out_off[v], L =
// out_off[v+1] - out_off[v] of them, from the segments' detector output d_scratch by the owned-frame runs
// run_first[i] .. run_first[i+1]-1 (run_lo / run_src, sync_plan.h), 0.0 where no segment owns the frame: floats, or
// with packed ceil(L/32) words of the bits m = (r == 1.0f) with zero bits past L.  d_speech[v] is reset first and ends
// as the video's first frame > 0 (kSigNoBadFrame: none).  The grid keeps to h->vad_partition_sms SMs when it is set.
int b2i_seg_ref_launch(b2_ctx* h, const float* d_scratch, const int64_t* out_off, const int* videos, int n_seg,
                       const int* run_first, const int64_t* run_lo, const int64_t* run_src, bool packed,
                       float* d_out, unsigned long long* d_speech);
// The speech output (K1o, speech_out.cu): frames off[i] .. off[i+1] of d_out (host table off [n+1]) are listed video i's
// reference signal, read from the reference buffer d_ref at vids[i] (speech_out.cuh), widened to float64.
struct B2SpeechVideo;
int b2i_speech_out_launch(b2_ctx* h, const float* d_ref, const int64_t* off, const B2SpeechVideo* vids, int n,
                          double* d_out);
// The outputs of one batched sync call that sentinel_kernel overwrites for the tracks of a flagged video
// (device arrays; a_* [T * cols], evals [T * n_evals] and ratio may be null)
struct B2SigBadOut {
  double* bs;
  int32_t* bo;
  int32_t* bk;
  double* a_score;
  int32_t* a_offset;
  int cols;
  double* ratio;
  double* evals;
  int n_evals;
};
// For each video videos[i] whose flag d_flag[v] is set (!= kSigNoBadFrame) when bad_if_set, or unset when not:
// best_k = sentinel, best_score, all_score, gss_ratio and gss_evals NaN, best_offset and all_offset 0, on every track
// trk_off[v] .. trk_off[v+1]-1.  Signal videos: their first out-of-domain frame, set = B2_BEST_K_BAD_SIGNAL; segment
// videos: their first frame > 0, unset = B2_BEST_K_NO_SPEECH.
int b2i_sentinel_launch(b2_ctx* h, const unsigned long long* d_flag, const int* videos, int n, const int* trk_off,
                        const B2SigBadOut& out, int sentinel, bool bad_if_set);
int b2i_bounds_launch(b2_ctx* h, const float* d_sig, const int64_t* off_host, int n,
                      int64_t* d_first, int64_t* d_last);
int b2i_blend_launch(b2_ctx* h, const float* d_a, const float* d_b, int64_t n, int mode, double wa,
                     double wb, float* d_out);
// Cue mode of the aligner (b2_sync_batch): the subtitle signals are rasterised from the cue list
// into bit masks (never into float signals); all arrays are HOST pointers, cue_off has B+1
// absolute entries.
struct B2CueSource {
  const double* cue_start;
  const double* cue_end;
  const uint8_t* cue_keep;   // may be null
  const int64_t* cue_off;
  const double* ratios;      // [K]
  int sample_rate;
  double start_seconds;
  float ref_label;           // the reference is this call's detector output (or subtitle references, 1.0 / 0.0):
  bool ref_two_level;        // every value is 1.0f or ref_label when this is set (the run path and the GSS rounds
                             // rely on it); the auditok signal is a clipped cumsum with other levels unless its label
                             // is 0, and subtitle and audio references mixed at a non-zero label have three levels
  bool ref_packed = false;   // the detector wrote the reference as packed bits m = (r == 1.0f), one 32-bit word per
                             // 32 frames from each video's ref_off on, and no floats (run-path chains only)
};
int b2i_raster_bits_launch(b2_ctx* h, const B2CueSource* src, int B, int K, const int64_t* sig_off,
                           const long long* bits_off, uint32_t* d_bits);
// The same cue list already on the device (the GSS rounds upload it once per chain): DEVICE arrays,
// cue_off[n_sig + 1] absolute into start / end / keep.
struct B2CueDev {
  const double* start;
  const double* end;
  const uint8_t* keep;       // may be null
  const long long* cue_off;
  int sample_rate;
  double start_seconds;
};
// Zeroes n_sig masks of sig_words words each (signal b at d_bits + b * sig_words) and rasterises signal b at
// the ratio d_ratio[b] and length d_len[b] (device arrays written by an earlier kernel).  No host upload.
int b2i_raster_bits_dev_launch(b2_ctx* h, const B2CueDev& cues, int n_sig, int64_t max_cues, const double* d_ratio,
                               const long long* d_len, long long sig_words, uint32_t* d_bits);
// capture_j0: global index of job 0 of this call in the arrays of b2_capture_nominations (b2_sync_batch's
// sub-batches align a range of pairs at a time).  ref_off_host has V+1 entries; reference v is shared by
// the tracks trk_off[v] .. trk_off[v+1]-1 (trk_off[V] == B), each with K ratio jobs t*K + k.  trk_off == NULL:
// V == B, reference b belongs to pair b alone.
int b2i_align_launch(b2_ctx* h, const float* d_ref, const int64_t* ref_off_host, int V, const int* trk_off,
                     const float* d_sub, const int64_t* sub_off_host, int B, int K,
                     int64_t max_offset_samples, double* d_score, int32_t* d_offset,
                     int32_t* d_status, int winner_only, const B2CueSource* cue_src,
                     long long capture_j0);
int b2i_reduce_launch(b2_ctx* h, const double* d_score, const int32_t* d_offset,
                      const int32_t* d_status, int B, int K, int64_t max_offset_samples,
                      double* d_best_score, int32_t* d_best_offset, int32_t* d_best_k);
// Golden-section search over the ratio for the tracks [0, T) of one chain (runcorr.cu, DESIGN.md section 4
// "K8g"), after the grid chain wrote its reduced (score, offset, k) to bs / bo / bk and its per-ratio results
// to g_score / g_offset [T*K].  Everything is enqueued on h->stream without a synchronisation.  ref_off_host
// [V+1] and trk_off[V+1] as for b2i_align_launch; max_end[t]: the track's largest cue end (0 without cues).
// Writes gss_ratio[t] (NaN for an empty reference), evals[t * kGssEvals + r] when evals is not null, merges the
// GSS candidate into bs / bo / bk, and, when a_score / a_offset are not null, the grid's K results plus the
// candidate into a_*[t * (K + 1) + k].
struct B2GssOut {
  double* bs;
  int32_t* bo;
  int32_t* bk;
  const double* g_score;
  const int32_t* g_offset;
  double* a_score;     // may be null
  int32_t* a_offset;   // may be null
  double* gss_ratio;
  double* evals;       // may be null
};
int b2i_gss_launch(b2_ctx* h, const float* d_ref, const int64_t* ref_off_host, int V, const int* trk_off, int K,
                   const B2CueSource& src, const double* max_end, int64_t max_offset_samples, const B2GssOut& out);
// b2_apply_sync's kernel (sync_output.cu): best_* / gss (nullable) / the outputs are DEVICE arrays, cue_start /
// cue_end / cue_off [T+1] (absolute cue indices, also those of d_start_us / d_end_us) and ratios [K] HOST arrays.
// Fails with B2_ERR_BAD_ARG before the launch, naming the cue, when a cue time is not finite or |t| >= t_max.
struct B2SyncRule;
int b2i_apply_sync_launch(b2_ctx* h, const double* d_bs, const int32_t* d_bo, const int32_t* d_bk,
                          const double* d_gss, int T, const double* cue_start, const double* cue_end,
                          const int64_t* cue_off, double t_max, const double* ratios, int K, const B2SyncRule& rule,
                          int64_t* d_start_us, int64_t* d_end_us, double* d_offset_seconds, double* d_scale,
                          int32_t* d_status);
// Per-segment offsets of b2_split_tracks (K9s, split.cu) for T tracks against the reference frames d_ref (float64 when
// ref_f64, else float32; DEVICE) of V videos at the HOST offsets ref_off [V+1].  Host arrays: track_video, the cue
// lists (cue_off [T+1] absolute, also into d_cue_offset), ratio [T] (NaN = skipped) and len [T] (each track's mask
// length at its ratio).  The caller has checked every argument.  refuse_three_levels: synchronise after the reference
// scan and fail with B2_ERR_UNSUPPORTED for a video with a third level (h_ref: its host frames for the message, float64
// when h_ref_f64, or null); otherwise that video's tracks get n_segments = -1.  Everything else is enqueued without a synchronisation.
// wide: b2_split_tracks_wide's envelope (h->split_max_cluster CTAs per track) instead of b2_split_tracks' 32768 offsets.
// max_segments > 0: b2_split_tracks_capped (at most that many segments, clusters of max_segments x C CTAs up to
// h->split_capped_max_cluster; wide must be set) and d_profile [T x max_segments] (DEVICE) gets each layer's maximum.
// direction +1 / -1: b2_split_tracks_directed (offsets only grow / only shrink along the track; clusters up to
// h->split_directed_max_cluster; wide must be set, max_segments 0).
// n_breaks > 0: b2_split_tracks_breaks (breaks [n_breaks] of +1 / -1, HOST, checked; clusters up to
// h->split_breaks_max_cluster for the kernel's layer count; wide must be set, max_segments and direction 0) and
// d_profile [T x (n_breaks + 1)] (DEVICE) gets each exact break count's maximum.
int b2i_split_launch(b2_ctx* h, const void* d_ref, bool ref_f64, const int64_t* ref_off, int V,
                     const int32_t* track_video, int T, const double* cue_start, const double* cue_end,
                     const uint8_t* cue_keep, const int64_t* cue_off, const double* ratio, const int64_t* len,
                     int sample_rate, double start_seconds, int64_t max_offset_samples, double penalty,
                     bool refuse_three_levels, const void* h_ref, bool h_ref_f64, bool wide, int* d_cue_offset,
                     int* d_n_segments, double* d_split_score, int max_segments = 0, double* d_profile = nullptr,
                     int direction = 0, const int32_t* breaks = nullptr, int n_breaks = 0);
// Sets h->split_max_cluster (split.cu) if it is not set yet.
int b2i_split_max_cluster(b2_ctx* h);
// Sets h->split_capped_max_cluster (split.cu) if it is not set yet.
int b2i_split_capped_max_cluster(b2_ctx* h);
// Sets h->split_directed_max_cluster (split.cu) if it is not set yet.
int b2i_split_directed_max_cluster(b2_ctx* h);
// Sets h->split_breaks_max_cluster for split_breaks_dp_kernel<kM> (kM = 32 / (n_breaks + 1) offsets a thread;
// split.cu) if it is not set yet.
int b2i_split_breaks_max_cluster(b2_ctx* h, int kM);
// b2_apply_split's kernel (sync_output.cu): n_segments / cue_offset / the outputs are DEVICE arrays, ratio [T] and the
// cue tables HOST arrays (absolute cue indices, as for b2i_apply_sync_launch).
int b2i_apply_split_launch(b2_ctx* h, const double* ratio, const int32_t* d_n_segments, const int32_t* d_cue_offset,
                           int T, const double* cue_start, const double* cue_end, const int64_t* cue_off, double t_max,
                           const B2SyncRule& rule, int64_t* d_start_us, int64_t* d_end_us, int32_t* d_status);
