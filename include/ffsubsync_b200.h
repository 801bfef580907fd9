/*
 * ffsubsync_b200.h - C ABI of the H100-native ffsubsync alignment hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no torch / C++ types.  Each entry
 * point names the piece of the reference (smacke/ffsubsync, paths relative to the reference
 * root) whose work it replaces.  The Python host layer (ffsubsync_b200/*.py) binds these
 * with ctypes and mirrors the reference's transformer API on top; INTEGRATION.md shows the
 * binding a reference maintainer would add.
 *
 * Conventions
 *   - every function returns B2_OK (0) or a negative b2_status; b2_last_error(h) gives text.
 *   - "memspace" says where the BULK arrays of that call live: B2_HOST (the library copies them
 *     to the device - directly from pinned memory; large pageable buffers through its own pinned
 *     double buffer filled by a few host threads - copies results back and synchronises before
 *     returning) or
 *     B2_DEVICE (pointers are device pointers on the handle's device - a pointer that belongs to
 *     another device is rejected with B2_ERR_BAD_ARG; the call only enqueues work on the handle's
 *     stream and does not synchronise).  Calls leave the caller thread's current CUDA device as
 *     they found it.
 *   - METADATA arrays (offset tables "*_off", cue lists, ratio lists) are always host pointers.
 *   - offset tables have n+1 entries, in elements (not bytes): item i is [off[i], off[i+1]).
 *   - a handle owns its stream/workspace and is not thread-safe; use one handle per thread
 *     (the reference runs up to 4 VideoSpeechTransformer.fit calls on threads,
 *     ffsubsync/speech_transformers.py:872-877).
 */
#ifndef FFSUBSYNC_B200_H
#define FFSUBSYNC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2_ctx* b2_handle;

typedef enum {
  B2_OK = 0,
  B2_ERR_BAD_ARG = -1,
  B2_ERR_CUDA = -2,
  B2_ERR_EMPTY_INPUT = -3,   /* ffsubsync/aligners.py:58-66  -> FailedToFindAlignmentException */
  B2_ERR_NO_ALIGNMENT = -4,  /* ffsubsync/aligners.py:160-165 -> FailedToFindAlignmentException */
  B2_ERR_NOMEM = -5,
  B2_ERR_UNSUPPORTED = -6
} b2_status;

enum {
  B2_HOST = 0,
  B2_DEVICE = 1,
  /* b2_sync_batch only: B2_DEVICE, plus the caller's promise that the INPUT arrays (pcm) are resident -
     not written by anything queued on the handle's stream before this call.  The call may then start
     reading them (its VAD runs on an internal stream) while the tail of the previous b2_sync_batch call
     on this handle is still computing; outputs stay ordered on the handle's stream as with B2_DEVICE,
     results are identical.  Back-to-back batches of a resident corpus: DESIGN.md section 4 K1p. */
  B2_DEVICE_RESIDENT = 2
};

/* Per-(pair, ratio) status written by the aligner. */
enum {
  B2_ALIGN_OK = 0,
  B2_ALIGN_EMPTY = 1,        /* reference or subtitle signal has length 0 */
  B2_ALIGN_ALL_MASKED = 2,   /* max_offset mask left nothing: score = -inf, offset = N-1-S */
  B2_ALIGN_CAND_OVERFLOW = 4, /* more near-maximal candidates than the re-score budget (flag) */
  B2_ALIGN_APPROX = 8 /* b2_sync_batch without per-ratio outputs: this ratio cannot be the pair's best
                         (its fp32 maximum plus the round-off bound tau lies below another ratio's
                         maximum minus tau), so it was not re-scored; fp32 score / its argmax kept */
};

/* FFTAligner(max_offset_samples=None).  Every other int64 value is a mask width and goes through the
 * reference's slice arithmetic (ffsubsync/aligners.py:31-43) literally - negative widths mask
 * everything (score -inf, offset N-1-S), widths beyond the padded length mask nothing. */
#define B2_MAX_OFFSET_NONE INT64_MIN

/* best_k of a track whose video's serialized signal reference holds a value outside its domain (> 1.0 or NaN;
 * b2_sync_tracks_sig).  best_k = -1 stays the reference's FailedToFindAlignment (an empty signal). */
#define B2_BEST_K_BAD_SIGNAL (-2)

/* best_k of a track whose video's sampled segments hold no frame > 0 (b2_sync_tracks_seg): the reference's
 * "Unable to detect speech in any sampled segment" (MultiSegmentVideoSpeechTransformer.fit). */
#define B2_BEST_K_NO_SPEECH (-3)

/* ---- lifecycle ----------------------------------------------------------------------- */
int b2_version(void);
int b2_create(int device, b2_handle* out);
int b2_destroy(b2_handle h);
/* Launch on a caller-owned CUDA stream (cudaStream_t passed as void*); NULL = own stream. */
int b2_set_stream(b2_handle h, void* cuda_stream);
int b2_synchronize(b2_handle h);
const char* b2_last_error(b2_handle h);
/* Number of kernel launches issued through this handle since creation (bench: gpu_launches). */
int64_t b2_launch_count(b2_handle h);

/* ---- VAD: replaces the per-window detector loop ----------------------------------------
 * ffsubsync/speech_transformers.py:155-183 (_make_webrtcvad_detector._detect: window size,
 * output length, labels, partial-window rule) called from the chunk loop :710-753.
 * Rule (this repo's detector, DESIGN.md): speech <=> sum x^2 >= fpw*energy_threshold and
 * z_lo <= #sign changes inside the window <= z_hi.  z_lo/z_hi < 0 select the defaults.
 * pcm: int16 mono samples of all B signals back to back (memspace); out: float per window.
 * b2_vad_energy_zcr is one detector call per signal: ceil(n / fpw) windows.  The reference's chunk loop calls the
 * detector once per (2 frame_rate // sample_rate) * 5000 samples, and every call restarts the window grid; where that
 * is not a whole number of windows (22.05 kHz: 2 205 000 samples of 221) each call ends in a non-speech partial
 * window.  b2_vad_call_samples gives the samples per call there and 0 where the calls divide into windows (one call
 * per video then gives the same frames).  The batched sync calls and the ingest session follow the chunk loop:
 * b2_vad_num_windows is their reference length for a video of n_samples, the sum over its calls of ceil(len / fpw);
 * b2_vad_energy_zcr over the calls as separate signals gives their frames. */
int b2_vad_frames_per_window(int frame_rate, int sample_rate);
int64_t b2_vad_call_samples(int frame_rate, int sample_rate);
int64_t b2_vad_num_windows(int64_t n_samples, int frame_rate, int sample_rate);
int b2_vad_energy_zcr(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int B,
                      int frame_rate, int sample_rate, float non_speech_label,
                      int64_t energy_threshold, int z_lo, int z_hi,
                      float* out, const int64_t* out_off, int memspace);

/* Streaming form of the same detector for the reference's chunk loop
 * (ffsubsync/speech_transformers.py:710-746: read <= 100 s of ffmpeg's pipe, detect, append):
 * b2_vad_stream_push copies the HOST chunk into a pinned ring slot, enqueues H2D copy + kernel +
 * D2H of the chunk's windows and returns without synchronising, so decoding chunk i+1 overlaps
 * the transfer and detection of chunk i.  Every chunk is detected on its own exactly like one
 * detector call (ceil(n/fpw) windows, a partial last window is non-speech; an odd trailing byte is
 * ignored).  b2_vad_stream_end waits, writes all windows in push order to HOST out
 * (capacity in floats, B2_ERR_BAD_ARG when too small) and closes the stream.
 * b2_vad_stream_windows = windows pushed so far (what `out` must hold). */
int b2_vad_stream_begin(b2_handle h, int frame_rate, int sample_rate, float non_speech_label,
                        int64_t energy_threshold, int z_lo, int z_hi);
int b2_vad_stream_push(b2_handle h, const void* pcm_bytes, int64_t n_bytes);
int64_t b2_vad_stream_windows(b2_handle h);
int b2_vad_stream_end(b2_handle h, float* out, int64_t capacity, int64_t* n_out);

/* ---- auditok detector: replaces _make_auditok_detector._detect ------------------------------
 * ffsubsync/speech_transformers.py:101-152.  The third-party arithmetic (auditok==0.1.5, absent from
 * the image) is restated from its published algorithm in oracle/auditok_oracle.py:
 *   energy test per 10 ms block (AudioEnergyValidator, :125): 10*log10(sum x^2 / n) >= energy_threshold_db,
 *     evaluated as  sum x^2 >= b2_auditok_energy_floor(n, energy_threshold_db)  (integer-exact; a
 *     trailing shorter block is tested on the samples it has);
 *   StreamTokenizer(min_length, max_length, max_continuous_silence) (:126-131) over the block flags;
 *   start / end+1 impulses, float64 cumsum, clip to [0, 1] (:146-150).
 * Each signal is cut into detector calls of chunk_samples samples (0 = one call per signal; the
 * reference's chunk loop uses 100 s, :710-746) and the tokenizer restarts in every call (:142).
 * out: float64 per block, ceil(chunk/fpw) per call, fpw = frame_rate // sample_rate; out_off[b] spans
 * the blocks of signal b.  pcm/out follow memspace.  B2_ERR_UNSUPPORTED when auditok's block size
 * int(frame_rate * (1/sample_rate)) differs from frame_rate // sample_rate. */
int b2_auditok_block_size(int frame_rate, int sample_rate);
int64_t b2_auditok_energy_floor(int n_samples, double energy_threshold_db);
int b2_vad_auditok(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int B,
                   int frame_rate, int sample_rate, double non_speech_label,
                   double energy_threshold_db, double min_length, int64_t max_length,
                   double max_continuous_silence, int64_t chunk_samples,
                   double* out, const int64_t* out_off, int memspace);

/* ---- subtitle side: replaces SubtitleScaler.fit + SubtitleSpeechTransformer.fit ----------
 * ffsubsync/subtitle_transformers.py:35-47 and ffsubsync/speech_transformers.py:957-980.
 * Cues (seconds, float64, unscaled) of pair b are [cue_off[b], cue_off[b+1]); keep[i]==0 for
 * cues the metadata filter drops (they still count for the array length).  Signal (b,k) uses
 * ratio ratios[b*K+k] when per_pair_ratios != 0, else ratios[k].  The written level is
 * min(1/ratio, 1) (speech_transformers.py:977) unless levels (same shape as ratios) is given:
 * SubtitleSpeechTransformer alone = ratios of 1.0 (times already scaled) + levels.
 * b2_rasterize_lengths computes len = int(max_end*sample_rate)+2 per (b,k) on the host.
 * The cue arithmetic is the reference's bit for bit for finite positive ratios, finite cue times t with
 * |t|*ratio < 2^53 us (9007199254.740992 s, about 285 years) and |start_seconds| below the same limit;
 * everything else (the reference raises in timedelta for non-finite times) is B2_ERR_BAD_ARG, here and
 * in b2_sync_batch / b2_sync_tracks.  Metadata cues (keep == 0) are checked too. */
int b2_rasterize_lengths(const double* cue_end_s, const int64_t* cue_off, int B,
                         const double* ratios, int K, int per_pair_ratios, int sample_rate,
                         int64_t* lengths /* [B*K] */);
int b2_rasterize(b2_handle h, const double* cue_start_s, const double* cue_end_s,
                 const uint8_t* cue_keep, const int64_t* cue_off, int B,
                 const double* ratios, int K, int per_pair_ratios,
                 const double* levels /* or NULL */, int sample_rate, double start_seconds,
                 float* out, const int64_t* out_off /* [B*K+1] */, int memspace);

/* ---- PGSSpeechTransformer.fit: bitmap-subtitle (PGS) display intervals -> 100 Hz speech signal ---------------
 * ffsubsync/speech_transformers.py:1186-1198, for B interval lists (list b: off[b] .. off[b+1], seconds as ffprobe's
 * pts_time and pts_time + duration_time).  Not the text rule of b2_rasterize: raw float64 times, each end rounded on
 * its own, s = int(round((t - start_seconds) * sample_rate)) (half to even), signal length
 * int(max_end * sample_rate) + 2 (truncation toward zero, no max(0, .)), and an interval fills [max(s0, 0),
 * min(s1, n)) with 1.0 when that is not empty (intervals may overlap, be unsorted or have a negative duration).
 * b2_rasterize_pgs_lengths (host) gives the lengths; b2_rasterize_pgs writes signal b at out + out_off[b] (out_off
 * [B+1], normally the cumulative lengths; the n of the clamp is out_off[b+1] - out_off[b]), out following memspace.
 * B2_ERR_BAD_ARG (the message names the list or interval) for an empty list (the reference raises ValueError), a
 * non-finite time, |t| >= B2_MAX_CUE_SECONDS, a negative length (np.zeros raises), a non-monotone off, sample_rate
 * outside (0, 2^28] or |start_seconds| >= B2_MAX_CUE_SECONDS.  b2_rasterize_pgs_lengths reads only end times. */
int b2_rasterize_pgs_lengths(const double* end_s, const int64_t* off /* [B+1] */, int B, int sample_rate,
                             int64_t* lengths /* [B] */);
int b2_rasterize_pgs(b2_handle h, const double* start_s, const double* end_s, const int64_t* off /* [B+1] */, int B,
                     int sample_rate, double start_seconds, float* out, const int64_t* out_off /* [B+1] */,
                     int memspace);

/* ---- fused-VAD blend ------------------------------------------------------------------------
 * ffsubsync/speech_transformers.py:281-294 (_make_fused_detector._detect): two detector outputs
 * clipped to their common length n and combined element-wise.
 * mode 0 "intersection" = min(a, b); 1 "union" = max(a, b); 2 "weighted" = wa*a + wb*b computed
 * in float64 like the reference (0.6 * silero + 0.4 * webrtc there) and rounded once to float32. */
int b2_blend_signals(b2_handle h, const float* a, const float* b, int64_t n, int mode, double wa,
                     double wb, float* out, int memspace);

/* ---- ComputeSpeechFrameBoundariesMixin.fit_boundaries -------------------------------------
 * ffsubsync/speech_transformers.py:310-317: first/last index with value > 0.5, or -1/-1. */
int b2_first_last_nonzero(b2_handle h, const float* sig, const int64_t* sig_off, int n,
                          int64_t* first, int64_t* last, int memspace);

/* ---- FFTAligner.fit for a batch of B references x K subtitle signals ----------------------
 * ffsubsync/aligners.py:50-80 (+ mask :31-43, argmax :45-48).  Signals are the raw values the
 * caller would hand to FFTAligner (the 2x-1 map is applied inside).  For every (b,k):
 * score[b*K+k], offset[b*K+k] = (best_score_, best_offset_), status = B2_ALIGN_* flags.
 * max_offset_samples = B2_MAX_OFFSET_NONE reproduces max_offset_samples=None.
 * score/offset/status follow memspace like the signals. */
int b2_align_batch(b2_handle h, const float* ref, const int64_t* ref_off /* [B+1] */,
                   const float* sub, const int64_t* sub_off /* [B*K+1] */, int B, int K,
                   int64_t max_offset_samples,
                   double* score, int32_t* offset, int32_t* status, int memspace);

/* ---- MaxScoreAligner.transform over the K candidates of each pair -------------------------
 * ffsubsync/aligners.py:154-167: drop |offset| > max_offset_samples, highest score, first in
 * list order wins ties.  best_k[b] = -1 when nothing survives (-> B2_ERR_NO_ALIGNMENT in the
 * single-pair wrappers). */
int b2_reduce_ratios(b2_handle h, const double* score, const int32_t* offset,
                     const int32_t* status, int B, int K, int64_t max_offset_samples,
                     double* best_score, int32_t* best_offset, int32_t* best_k, int memspace);

/* ---- the whole hot path for a batch of (video, subtitle) pairs -----------------------------
 * VAD on each pair's PCM -> rasterise its cues at K ratios -> align -> reduce
 * (ffsubsync/ffsubsync.py:637 + :196-235).  The VAD follows the reference's chunk loop: b2_vad_energy_zcr over each
 * b2_vad_call_samples call of the PCM (over the whole PCM where that is 0), b2_vad_num_windows frames.  pcm and the outputs follow memspace; memspace may also be
 * B2_DEVICE_RESIDENT (see the enum): consecutive calls over resident PCM then overlap across the call boundary. */
int b2_sync_batch(b2_handle h, const int16_t* pcm, const int64_t* pcm_off, int B,
                  int frame_rate, int sample_rate, float non_speech_label,
                  int64_t energy_threshold, int z_lo, int z_hi,
                  const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                  const int64_t* cue_off, const double* ratios, int K, double start_seconds,
                  int64_t max_offset_samples,
                  double* best_score, int32_t* best_offset, int32_t* best_k,
                  double* all_score /* [B*K] or NULL */, int32_t* all_offset /* or NULL */,
                  int memspace);

/* ---- the whole hot path for several subtitle tracks per video ------------------------------
 * `ffs movie.mkv -i en.srt de.srt ...` (ffsubsync/ffsubsync.py:637 + the loop of try_sync over
 * args.srtin, :186-235) for V videos and T tracks in one call: track t (cue list
 * cue_off[t] .. cue_off[t+1]) is synced against the PCM of video track_video[t].  track_video is a host
 * array, non-decreasing, every entry in [0, V).  Each video's PCM goes through the VAD once and its
 * reference spectra are shared by all its tracks.  Track t gets exactly what b2_sync_batch returns for the
 * pair (PCM of video track_video[t], cue list t): best_*[t], and all_*[t*K + k] when requested.
 * A video without tracks is legal; its VAD still runs (its PCM is read, nothing of it is returned).
 * memspace as for b2_sync_batch (B2_HOST, B2_DEVICE, B2_DEVICE_RESIDENT; resident calls chain with
 * b2_sync_batch calls too).  B2_ERR_BAD_ARG for a track_video entry out of range or smaller than the one
 * before, a non-monotone pcm_off or cue_off, a null output or, with B2_DEVICE, a host pointer among pcm
 * and the outputs. */
int b2_sync_tracks(b2_handle h, const int16_t* pcm, const int64_t* pcm_off /* [V+1] */, int V,
                   const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                   float non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                   const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                   const int64_t* cue_off /* [T+1] */, const double* ratios, int K, double start_seconds,
                   int64_t max_offset_samples, double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                   double* all_score /* [T*K] or NULL */, int32_t* all_offset /* [T*K] or NULL */,
                   int memspace);

/* ---- the grid plus the golden-section search over the ratio (--gss) ----------------------------
 * `ffs movie.mkv -i a.srt ... --gss`: the reference's ratio list is the grid plus a golden-section search
 * (ffsubsync/ffsubsync.py:131-142; MaxScoreAligner.fit_gss, ffsubsync/aligners.py:111-129;
 * ffsubsync/golden_section_search.py:15-74).  Track t gets exactly what the reference's try_sync returns for the
 * candidates [ratios[0..K-1], GSS]: the GSS candidate is the (score, offset) of the 17th evaluation of the search
 * over [0.9, 1.1] with tolerance 1e-4 (fixed), and it goes through the same |offset| <= max_offset_samples filter
 * and first-wins tie rule as a (K+1)-th ratio: best_k[t] == K means it won, and on an exact tie a grid ratio wins.
 * Arguments as for b2_sync_tracks, plus gss_ratio[T] (the 17th point; NaN for a track whose video has no
 * windows, which gets best_k = -1 and is not searched) and gss_evals[T*17] (every point in evaluation order, or
 * NULL).  all_score / all_offset, when given, are [T*(K+1)]: column K holds the GSS candidate.  memspace as for
 * b2_sync_tracks; resident calls chain with b2_sync_batch / b2_sync_tracks in either order.  The 17 rounds run
 * on the handle's stream without a host synchronisation (DESIGN.md section 4 "K8g").  B2_ERR_UNSUPPORTED unless
 * 0 <= max_offset_samples <= 16384 (every mask window then holds at most 2*max_offset_samples <= 32768 offsets),
 * every track has at most 16384 cues and non_speech_label is finite; the message names the limit. */
int b2_sync_tracks_gss(b2_handle h, const int16_t* pcm, const int64_t* pcm_off /* [V+1] */, int V,
                       const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                       float non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                       const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                       const int64_t* cue_off /* [T+1] */, const double* ratios, int K, double start_seconds,
                       int64_t max_offset_samples, double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                       double* all_score /* [T*(K+1)] or NULL */, int32_t* all_offset /* [T*(K+1)] or NULL */,
                       double* gss_ratio /* [T] */, double* gss_evals /* [T*17] or NULL */, int memspace);

/* ---- the whole hot path with the reference's auditok detector (--vad auditok) ----------------------------
 * `ffs movie.mkv -i a.srt ... --vad auditok [--gss]` for V videos and T tracks.  Track t gets exactly what this
 * composition of public calls returns: b2_vad_auditok on the PCM of video track_video[t] with these detector
 * arguments and chunk_samples, rounded once to float32, then b2_sync_tracks (b2_sync_tracks_gss when gss_ratio is
 * not NULL) with that signal in place of the energy / ZCR VAD output.  Detector arguments as for b2_vad_auditok
 * (B2_ERR_UNSUPPORTED for a block-size mismatch, B2_ERR_BAD_ARG for bad tokenizer parameters); each video is cut
 * into detector calls of chunk_samples samples and the tokenizer restarts in every call, so a video's reference
 * signal holds the sum over its chunks of ceil(len/fpw) blocks.  Every other argument as for b2_sync_tracks /
 * b2_sync_tracks_gss: gss_ratio NULL = the grid only, all_* [T*K]; else gss_ratio [T], gss_evals [T*17] or NULL,
 * all_* [T*(K+1)].  The search needs non_speech_label == 0 (only then is the signal two-level, 1.0 and 0.0; the
 * rounds run on the run path): any other label is B2_ERR_UNSUPPORTED with gss_ratio.  Grid calls with another
 * label align on the FFT paths.  memspace: B2_HOST, B2_DEVICE or B2_DEVICE_RESIDENT; resident calls chain with
 * b2_sync_batch, b2_sync_tracks and b2_sync_tracks_gss in any order.  The pair form (b2_sync_batch) is the
 * identity track map. */
int b2_sync_tracks_auditok(b2_handle h, const int16_t* pcm, const int64_t* pcm_off /* [V+1] */, int V,
                           const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                           double non_speech_label, double energy_threshold_db, double min_length, int64_t max_length,
                           double max_continuous_silence, int64_t chunk_samples,
                           const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                           const int64_t* cue_off /* [T+1] */, const double* ratios, int K, double start_seconds,
                           int64_t max_offset_samples, double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                           double* all_score, int32_t* all_offset /* [T*K], [T*(K+1)] with the search, or NULL */,
                           double* gss_ratio /* [T] or NULL = grid only */, double* gss_evals /* [T*17] or NULL */,
                           int memspace);

/* ---- embedded subtitle streams as references (--vad subs_then_webrtc / subs_then_auditok) -----------------
 * `ffs movie.mkv -i a.srt ...` with a subs_then_ detector for V videos and T tracks: a video with a text subtitle
 * stream is synced against that stream rasterised (VideoSpeechTransformer.fit -> try_fit_using_embedded_subs,
 * ffsubsync/speech_transformers.py:479-523,609-619), any other video against the detector's output.  Choosing the
 * stream (the reference takes the one with the largest max_end - start_seconds, the first on a tie), parsing it
 * and the metadata flags are the caller's; so is extracting streams from containers.
 * Arguments as for b2_sync_tracks_auditok, plus:
 *   detector             B2_DETECTOR_ENERGY_ZCR (energy_threshold, z_lo, z_hi as for b2_sync_tracks; the label is
 *                        rounded to float) or B2_DETECTOR_AUDITOK (energy_threshold_db ... chunk_samples as for
 *                        b2_sync_tracks_auditok); the other detector's arguments are not read.
 *   ref_is_subs [V]      non-zero: video v has a subtitle reference.  NULL = none (every video is audio).
 *   ref_cue_start_s, ref_cue_end_s, ref_cue_keep, ref_cue_off [V+1]
 *                        host arrays: video v's reference cues are ref_cue_off[v] .. ref_cue_off[v+1] (seconds,
 *                        unscaled, keep as for b2_rasterize; ref_cue_keep may be NULL = keep all).  A video without a
 *                        subtitle reference has an empty list; a subtitle reference may be empty (a 2-frame signal).
 * Track t gets exactly what this composition of public calls returns: the reference of video track_video[t] -
 * b2_rasterize of its cue list at ratio 1.0 with level 1.0 (int(max_end * sample_rate) + 2 frames, max_end over
 * all its cues, metadata ones included, 0 without cues) for a subtitle video, the detector's output as in
 * b2_sync_tracks / b2_sync_tracks_auditok otherwise - then b2_align_batch and b2_reduce_ratios over the ratios,
 * plus the golden-section search's candidate as in b2_sync_tracks_gss when gss_ratio is not NULL.
 * A subtitle video's PCM range must be empty (B2_ERR_BAD_ARG otherwise): its audio is never read, and pcm may be
 * NULL when no video has samples.  Reference cue times get the checks of b2_rasterize (B2_ERR_BAD_ARG, the message
 * names the index); so does a non-monotone ref_cue_off, or cues given for a video without a subtitle reference.
 * Levels: a subtitle reference holds 1.0 and 0.0, the detector's 1.0 and non_speech_label.  A call that mixes the
 * two at a non-zero label, or runs auditok at a non-zero label on any video, aligns on the FFT paths; with
 * gss_ratio it is B2_ERR_UNSUPPORTED (the search runs on the run path).  Without subtitle videos the call returns
 * what b2_sync_tracks / b2_sync_tracks_gss / b2_sync_tracks_auditok return.  memspace: B2_HOST, B2_DEVICE or
 * B2_DEVICE_RESIDENT; resident calls chain with the other sync calls in any order. */
enum { B2_DETECTOR_ENERGY_ZCR = 0, B2_DETECTOR_AUDITOK = 1 };
int b2_sync_tracks_subs(b2_handle h, const int16_t* pcm /* or NULL without audio */, const int64_t* pcm_off /* [V+1] */,
                        int V, const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                        int detector, double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                        double energy_threshold_db, double min_length, int64_t max_length,
                        double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs /* [V] */,
                        const double* ref_cue_start_s, const double* ref_cue_end_s, const uint8_t* ref_cue_keep,
                        const int64_t* ref_cue_off /* [V+1] */, const double* cue_start_s, const double* cue_end_s,
                        const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */, const double* ratios, int K,
                        double start_seconds, int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                        int32_t* best_k /* [T] */,
                        double* all_score, int32_t* all_offset /* [T*K], [T*(K+1)] with the search, or NULL */,
                        double* gss_ratio /* [T] or NULL = grid only */, double* gss_evals /* [T*17] or NULL */,
                        int memspace);

/* ---- PGS subtitle timings as references (--pgs-ref-stream) ------------------------------------------------
 * `ffs movie.mkv -i a.srt ... --pgs-ref-stream [S]` for V videos and T tracks: a video with a PGS (hdmv_pgs_subtitle)
 * stream is synced against that stream's display intervals rasterised (PGSSpeechTransformer, ffsubsync/ffsubsync.py:
 * 307-327), any other video as in b2_sync_tracks_subs.  Running ffprobe and choosing the stream are the caller's.
 * Arguments as for b2_sync_tracks_subs (ref_is_subs and ref_cue_* may be NULL: no text references), plus:
 *   ref_is_pgs [V]       non-zero: video v has a PGS reference.  NULL = none.
 *   pgs_start_s, pgs_end_s, pgs_off [V+1]
 *                        host arrays: video v's intervals are pgs_off[v] .. pgs_off[v+1] (seconds: pts_time and
 *                        pts_time + duration_time).  A video without a PGS reference has an empty list.
 * Track t gets exactly what this composition of public calls returns: the reference of video track_video[t] -
 * b2_rasterize_pgs of its intervals for a PGS video, what b2_sync_tracks_subs uses otherwise - then b2_align_batch
 * and b2_reduce_ratios over the ratios, plus the golden-section search's candidate as in b2_sync_tracks_gss when
 * gss_ratio is not NULL.  The PGS reference has no inferred framerate ratio: the grid is the caller's.
 * A PGS reference counts as a subtitle reference for the rules of b2_sync_tracks_subs: levels 1.0 and 0.0, an empty
 * PCM range, and the same label / path / B2_ERR_UNSUPPORTED rules.  B2_ERR_BAD_ARG also for the errors of
 * b2_rasterize_pgs, a PGS video with a non-empty PCM range, a video marked both PGS and text, intervals given for a
 * video without ref_is_pgs and a non-monotone pgs_off.  Without PGS videos the call returns what b2_sync_tracks_subs
 * returns.  memspace: B2_HOST, B2_DEVICE or B2_DEVICE_RESIDENT; resident calls chain with the other sync calls in any
 * order. */
int b2_sync_tracks_pgs(b2_handle h, const int16_t* pcm /* or NULL without audio */, const int64_t* pcm_off /* [V+1] */,
                       int V, const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                       int detector, double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                       double energy_threshold_db, double min_length, int64_t max_length,
                       double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs /* [V] */,
                       const double* ref_cue_start_s, const double* ref_cue_end_s, const uint8_t* ref_cue_keep,
                       const int64_t* ref_cue_off /* [V+1] or NULL */, const uint8_t* ref_is_pgs /* [V] */,
                       const double* pgs_start_s, const double* pgs_end_s, const int64_t* pgs_off /* [V+1] */,
                       const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                       const int64_t* cue_off /* [T+1] */, const double* ratios, int K, double start_seconds,
                       int64_t max_offset_samples, double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                       double* all_score, int32_t* all_offset /* [T*K], [T*(K+1)] with the search, or NULL */,
                       double* gss_ratio /* [T] or NULL = grid only */, double* gss_evals /* [T*17] or NULL */,
                       int memspace);

/* ---- serialized speech signals as references (`ffs ref.npz -i in.srt`) -------------------------------------
 * The signals that --serialize-speech / --make-test-case store (DeserializeSpeechTransformer, ffsubsync/
 * speech_transformers.py:987-1009) as references of V videos and T tracks.  Arguments as for b2_sync_tracks_pgs,
 * plus:
 *   ref_is_sig [V]       host; non-zero: video v's reference is its stored signal.  NULL = none.
 *   x                    the stored values as float64 (np.load's dtype), in memspace: video v's are
 *                        x[sig_off[v] .. sig_off[v+1]).  B2_DEVICE_RESIDENT: the resident promise (nothing queued
 *                        on the handle's stream before the call writes pcm) covers x too.
 *   sig_off [V+1]        host; a video without a signal reference has an empty range.
 * Frame i of a signal video is (float)(x < 1.0 ? non_speech_label : x) - the rule in float64, rounded once (so
 * values in (1 - 2^-25, 1) stay non-speech) - with the call's own label; start_seconds does not apply.  Every
 * stored value must be < 1.0 or exactly 1.0 (what the reference's detectors and rasterisers write), so a signal
 * reference has the levels 1.0 and the label like the energy detector's output, and counts like a detector video
 * for the label / path / B2_ERR_UNSUPPORTED rules of b2_sync_tracks_subs: signals alone are two-level with either
 * detector; mixed with text / PGS references or auditok audio at a non-zero label they make three levels.
 * A value > 1.0 or NaN is outside the domain: every track of that video gets best_k = B2_BEST_K_BAD_SIGNAL,
 * best_score NaN, best_offset 0, all_score NaN / all_offset 0 in every column, gss_ratio and gss_evals NaN, without
 * a host synchronisation; the other tracks are unaffected.  An empty signal gives best_k = -1.
 * Track t gets exactly what this composition of public calls returns: the rule applied to its video's signal (what
 * b2_sync_tracks_pgs uses for other videos), then b2_align_batch and b2_reduce_ratios over the ratios, plus the
 * golden-section search's candidate as in b2_sync_tracks_gss when gss_ratio is not NULL.  No inferred framerate
 * ratio: the grid is the caller's.  B2_ERR_BAD_ARG also for a non-monotone sig_off, values given for a video without
 * ref_is_sig, a signal video with a non-empty PCM range, a video marked signal and text or signal and PGS, a null x
 * under non-empty ranges and a host x under B2_DEVICE.  memspace: B2_HOST, B2_DEVICE or B2_DEVICE_RESIDENT;
 * resident calls chain with the other sync calls in any order. */
int b2_sync_tracks_sig(b2_handle h, const int16_t* pcm /* or NULL without audio */, const int64_t* pcm_off /* [V+1] */,
                       int V, const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                       int detector, double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                       double energy_threshold_db, double min_length, int64_t max_length,
                       double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs /* [V] */,
                       const double* ref_cue_start_s, const double* ref_cue_end_s, const uint8_t* ref_cue_keep,
                       const int64_t* ref_cue_off /* [V+1] or NULL */, const uint8_t* ref_is_pgs /* [V] */,
                       const double* pgs_start_s, const double* pgs_end_s, const int64_t* pgs_off /* [V+1] or NULL */,
                       const uint8_t* ref_is_sig /* [V] */, const double* x, const int64_t* sig_off /* [V+1] */,
                       const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                       const int64_t* cue_off /* [T+1] */, const double* ratios, int K, double start_seconds,
                       int64_t max_offset_samples, double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                       double* all_score, int32_t* all_offset /* [T*K], [T*(K+1)] with the search, or NULL */,
                       double* gss_ratio /* [T] or NULL = grid only */, double* gss_evals /* [T*17] or NULL */,
                       int memspace);

/* ---- sampled segments as references (`ffs movie.mkv -i in.srt --multi-segment-sync`) -----------------------
 * MultiSegmentVideoSpeechTransformer.fit (ffsubsync/speech_transformers.py:811-900) as the reference of some of V
 * videos: the detector runs only on a few sampled windows of the video, and the reference is 0.0 elsewhere.
 * Arguments as for b2_sync_tracks_sig (ref_is_subs, ref_is_pgs, ref_is_sig and their tables may be NULL), plus
 * these host arrays:
 *   n_seg_videos = P     videos with segments.  0 = none.
 *   seg_video [P]        their indices, increasing.
 *   seg_total [P]        the probed duration in seconds (ffprobe's format duration; samples / frame_rate for raw PCM).
 *   seg_off [P+1]        video i's segments are seg_off[i] .. seg_off[i+1]-1 of the arrays below.
 *   seg_start            per segment: its start in whole seconds (MultiSegmentVideoSpeechTransformer._segment_starts),
 *                        strictly increasing within a video.
 *   seg_lo, seg_hi       per segment: its samples pcm[pcm_off[v] + seg_lo .. pcm_off[v] + seg_hi), inside the video's
 *                        PCM range.  Ranges may overlap and leave gaps: the video's range may hold its whole decode
 *                        (segments are slices of it) or only the decoded windows back to back.  Samples outside the
 *                        segments are never read, and B2_HOST copies only the segments (and the audio videos) to the
 *                        device.
 * Segment j writes what the call's detector returns for its samples taken as one signal - energy / ZCR: the chunk
 * loop of b2_vad_call_samples from the segment's first sample (one call where that is 0), ceil(len / fpw) frames per
 * call, a trailing partial window non-speech; auditok: the chunk loop of chunk_samples from the
 * segment's first sample, the tokenizer restarting in every chunk - to the frames [seg_start * sample_rate,
 * min(seg_start * sample_rate + len, L)) of a reference of L = int(seg_total * sample_rate) + 2 frames (float64
 * product, truncated), in increasing start order, so that a later segment overwrites an earlier one where they
 * overlap.  Frames no segment covers are 0.0.  start_seconds does not apply to a segment reference (the reference's
 * transformer has no such argument); it still applies to the subtitle tracks.
 * A segment reference has the levels 0.0, 1.0 and the label: it is two-level only at label 0, where it counts like a
 * subtitle reference for the label / path / B2_ERR_UNSUPPORTED rules of b2_sync_tracks_subs (the search needs label 0
 * in a call with segment videos).
 * A video none of whose reference frames is > 0 has no speech (the reference raises "Unable to detect speech in any
 * sampled segment"): every track of that video gets best_k = B2_BEST_K_NO_SPEECH, best_score NaN, best_offset 0,
 * all_score NaN / all_offset 0 in every column, gss_ratio and gss_evals NaN, without a host synchronisation; the
 * other tracks are unaffected.
 * Track t gets exactly what this composition of public calls returns: for a segment video the reference above, built
 * from b2_vad_energy_zcr (or b2_vad_auditok rounded to float32) over its segments, for the others what
 * b2_sync_tracks_sig uses, then b2_align_batch and b2_reduce_ratios over the ratios, plus the golden-section search's
 * candidate as in b2_sync_tracks_gss when gss_ratio is not NULL.
 * B2_ERR_BAD_ARG also for a non-monotone seg_off, seg_video not increasing or out of [0, V), a seg_total that is not
 * finite or gives a negative length, a negative start or one not after the previous one, a range outside the video's
 * PCM range, null segment arrays under segments, and a segment video that also has a text, PGS or signal reference
 * (a video has one reference).  Without segment videos the call returns what b2_sync_tracks_sig returns.
 * memspace: B2_HOST, B2_DEVICE or B2_DEVICE_RESIDENT; resident calls chain with the other sync calls in any order. */
int b2_sync_tracks_seg(b2_handle h, const int16_t* pcm /* or NULL without audio */, const int64_t* pcm_off /* [V+1] */,
                       int V, const int32_t* track_video /* [T] */, int T, int frame_rate, int sample_rate,
                       int detector, double non_speech_label, int64_t energy_threshold, int z_lo, int z_hi,
                       double energy_threshold_db, double min_length, int64_t max_length,
                       double max_continuous_silence, int64_t chunk_samples, const uint8_t* ref_is_subs /* [V] */,
                       const double* ref_cue_start_s, const double* ref_cue_end_s, const uint8_t* ref_cue_keep,
                       const int64_t* ref_cue_off /* [V+1] or NULL */, const uint8_t* ref_is_pgs /* [V] */,
                       const double* pgs_start_s, const double* pgs_end_s, const int64_t* pgs_off /* [V+1] or NULL */,
                       const uint8_t* ref_is_sig /* [V] */, const double* x, const int64_t* sig_off /* [V+1] or NULL */,
                       int n_seg_videos, const int32_t* seg_video /* [P] */, const double* seg_total /* [P] */,
                       const int64_t* seg_off /* [P+1] */, const int64_t* seg_start, const int64_t* seg_lo,
                       const int64_t* seg_hi, const double* cue_start_s, const double* cue_end_s,
                       const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */, const double* ratios, int K,
                       double start_seconds, int64_t max_offset_samples, double* best_score, int32_t* best_offset,
                       int32_t* best_k /* [T] */,
                       double* all_score, int32_t* all_offset /* [T*K], [T*(K+1)] with the search, or NULL */,
                       double* gss_ratio /* [T] or NULL = grid only */, double* gss_evals /* [T*17] or NULL */,
                       int memspace);

/* ---- try_sync's epilogue: synced cue times and the low-quality gate ----------------------------------------
 * What ffsubsync/ffsubsync.py:236-299 does with the aligner's answer, for the T tracks of a finished batched sync
 * call (any of the calls above, or b2_reduce_ratios): best_score, best_offset, best_k [T] and, when the call ran
 * the golden-section search, gss_ratio [T] (NULL otherwise) are that call's outputs, in memspace.  Per track t:
 *   scale          ratios[best_k] for 0 <= best_k < K; gss_ratio[t] for best_k == K with gss_ratio (a value outside
 *                  [0.9, 1.1] - the search's interval - fails the track); otherwise the track FAILED (the reference's
 *                  FailedToFindAlignmentException): nothing is written, scale and offset_seconds are NaN.
 *   offset_seconds best_offset / (double)sample_rate + apply_offset_seconds (two correctly rounded operations).
 *   status         B2_SYNC_* bits below, in the reference's order: failure, negative score (SUCCESSFUL cleared, the
 *                  output still written), the gate when gate_enabled (assess_alignment_quality: best_score < min_score,
 *                  |offset_seconds| > quality_max_offset_seconds, |scale - 1| > max_framerate_deviation, plain IEEE
 *                  comparisons - a gated track gets its original cues WRITTEN, is not SUCCESSFUL, and the reference
 *                  leaves its result["offset_seconds"] / ["framerate_scale_factor"] unset), then suppression when
 *                  has_suppress and suppress_output_if_offset_less_than is not 0.0 (`thresh or -inf`): an
 *                  offset_seconds below it (or a NaN threshold) is SUPPRESSED instead of WRITTEN.
 * Per cue i of track t (cue_off[t] <= i < cue_off[t+1]; metadata cues too - the reference writes them), into
 * synced_start_us[i] / synced_end_us[i] (int64 microseconds): for an APPLIED track
 * timedelta(seconds=t_i * scale) + timedelta(seconds=offset_seconds) - each rounded half-to-even to the microsecond
 * on its own (SubtitleScaler, SubtitleShifter) - and timedelta(seconds=t_i) (the parsed original) otherwise.
 * cue_start_s, cue_end_s, cue_off [T+1] and ratios [K] are host metadata; the outputs follow memspace (B2_HOST copies
 * back and synchronises; B2_DEVICE enqueues one kernel on the handle's stream behind the call that wrote the inputs
 * and returns).  Unlike every other entry point it does not break a chain of B2_DEVICE_RESIDENT sync calls.
 * B2_ERR_BAD_ARG (the message names the item) for a non-monotone cue_off, a non-finite cue time, ratio or
 * apply_offset_seconds, sample_rate <= 0, a cue time with |t| >= (B2_MAX_CUE_SECONDS - 2^31 / sample_rate -
 * |apply_offset_seconds|) / smax (smax: the largest of 1, |ratios[k]| and 1.1 with gss_ratio - a bound on every output
 * time that does not need the device results), a null input or output, and a host pointer under B2_DEVICE. */
enum {
  B2_SYNC_WRITTEN = 1,        /* the reference writes this track's output file */
  B2_SYNC_APPLIED = 2,        /* synced_* hold the scaled and shifted times (else the originals) */
  B2_SYNC_SUCCESSFUL = 4,     /* the track leaves try_sync's sync_was_successful true */
  B2_SYNC_FAILED = 8,         /* no alignment (best_k < 0 or out of range) */
  B2_SYNC_SUPPRESSED = 16,    /* --suppress-output-if-offset-less-than held the output back */
  B2_SYNC_LOW_SCORE = 32,     /* gate: best_score < min_score */
  B2_SYNC_LOW_OFFSET = 64,    /* gate: |offset_seconds| > quality_max_offset_seconds */
  B2_SYNC_LOW_FRAMERATE = 128 /* gate: |scale - 1| > max_framerate_deviation */
};
int b2_apply_sync(b2_handle h, const double* best_score, const int32_t* best_offset, const int32_t* best_k,
                  const double* gss_ratio /* [T] or NULL */, int T, const double* cue_start_s, const double* cue_end_s,
                  const int64_t* cue_off /* [T+1] */, const double* ratios, int K, int sample_rate,
                  double apply_offset_seconds, int gate_enabled, double min_score, double quality_max_offset_seconds,
                  double max_framerate_deviation, int has_suppress, double suppress_output_if_offset_less_than,
                  int64_t* synced_start_us, int64_t* synced_end_us, double* offset_seconds /* [T] */,
                  double* scale /* [T] */, int32_t* status /* [T] */, int memspace);

/* ---- per-segment offsets with a split penalty, after any batched sync call ---------------------------------
 * One offset per track (ffsubsync/aligners.py:24-86) fails when the video has a break the subtitles do not have, or
 * the reverse.  This splits each track's cue runs into segments with their own offsets (DESIGN.md section 4 "K9s").
 * Track t's mask is its kept cues rasterised at ratio[t] as the sync calls do (S frames, level (float)min(1/x, 1));
 * unit j is the gap before its j-th run of 1s and that run (the leading gap in unit 0, the frames after the last run
 * in the last unit; a mask without runs is one unit).  u_j(o) is unit j's four-count run-path score at offset o
 * against the reference of video track_video[t] (levels 1.0 and one other finite value beta per video).  Over the
 * window of offsets the aligner keeps for (R, S, max_offset_samples), the programme
 *     V_0(o) = u_0(o),   V_j(o) = u_j(o) + max(V_{j-1}(o), max_o V_{j-1} - split_penalty)
 * is solved in float64 with every operation rounded on its own; staying wins a tie, and among equal maxima the
 * largest offset wins (the aligner's rule).  No cap on the number of splits, no order between adjacent segments'
 * offsets, one ratio per track: split_penalty is the only knob, and +inf never switches.
 *   ref            the videos' reference frames, float64 (ref_is_f64, what b2_speech_output writes) or float32, at
 *                  ref_off [V+1] (host); in memspace.
 *   ratio [T]      host: each track's ratio (ratios[best_k], or gss_ratio when best_k == K); NaN skips the track.
 *   cue_*          host, as for b2_sync_tracks; cue_offset is indexed like the cues (absolute indices).
 * Per track: n_segments (0 for a skipped track or one whose window is empty), split_score = the sum of u_j over the
 * chosen path without penalties (NaN when skipped), and for every cue (kept or not) cue_offset = the offset of the
 * unit holding its rasterised start frame clamped into [0, S) (0 when skipped).  memspace B2_HOST copies in and
 * out and synchronises; B2_DEVICE enqueues on the handle's stream without a host synchronisation (behind the sync
 * call that wrote the reference), and a video whose reference has a third level gives its tracks n_segments = -1,
 * NaN and offsets 0 there, where B2_HOST refuses it with B2_ERR_UNSUPPORTED naming the video and frame.
 * B2_ERR_UNSUPPORTED also for a window wider than 32768 offsets (b2_split_tracks_wide below goes further) and a track with more than 16384 kept cues (each
 * run holds one); B2_ERR_BAD_ARG for a NaN or negative split_penalty, a ratio that is not NaN or finite positive,
 * a track_video entry outside [0, V), a non-monotone ref_off / cue_off, the cue checks of b2_rasterize and host
 * pointers under B2_DEVICE. */
int b2_split_tracks(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off /* [V+1] */, int V,
                    const int32_t* track_video /* [T] */, int T, const double* cue_start_s, const double* cue_end_s,
                    const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */, const double* ratio /* [T] */,
                    int sample_rate, double start_seconds, int64_t max_offset_samples, double split_penalty,
                    int32_t* cue_offset, int32_t* n_segments /* [T] */, double* split_score /* [T] */, int memspace);
/* b2_split_tracks with a wider envelope: the same arguments, outputs, memspaces and refusals, but windows of up to
 * 16384 x C offsets, C the widest thread-block cluster of 512-thread CTAs the device co-schedules (at most 16:
 * 262144 offsets, +-1310 s at 100 Hz; the refusal names the limit).  The window is absolute and shared by all of a
 * track's segments, so it must cover the sync offset plus the breaks before the last segment.  Results equal
 * b2_split_tracks' bit for bit wherever both run. */
int b2_split_tracks_wide(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off /* [V+1] */, int V,
                         const int32_t* track_video /* [T] */, int T, const double* cue_start_s,
                         const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */,
                         const double* ratio /* [T] */, int sample_rate, double start_seconds,
                         int64_t max_offset_samples, double split_penalty, int32_t* cue_offset,
                         int32_t* n_segments /* [T] */, double* split_score /* [T] */, int memspace);
/* b2_split_tracks_wide with at most max_segments segments per track (DESIGN.md section 4 "K9s", the capped
 * programme).  Layer k = 0 .. N-1 (N = max_segments) counts the switches allowed so far:
 *     V_{0,k}(o) = u_0(o),   V_{j,0}(o) = u_j(o) + V_{j-1,0}(o),
 *     V_{j,k}(o) = u_j(o) + max(V_{j-1,k}(o), M_{j-1,k-1} - split_penalty)  (k >= 1),   M_{j,k} = max_o V_{j,k}(o)
 * with b2_split_tracks' rounding, tie and argmax rules.  cue_offset, n_segments (<= N) and split_score come from the
 * top layer's path; a track with at most N units gets b2_split_tracks_wide's results bit for bit, and N = 1 its
 * results at split_penalty = +inf.  split_profile [T x N] (f64, in memspace): split_profile[t*N + k] = the best
 * penalised objective with at most k+1 segments, M_{last,k} (at split_penalty 0 the best plain score per segment
 * count); NaN for a skipped track, an empty window or (B2_DEVICE) a three-level reference.  Refusals: those of
 * b2_split_tracks_wide; B2_ERR_BAD_ARG for max_segments < 1; B2_ERR_UNSUPPORTED for max_segments > 16 and for a
 * track whose N x ceil(window / 16384) CTAs exceed the widest cluster the device co-schedules for this kernel (16 on
 * an H100: +-60 s at 100 Hz up to N = 16, +-150 s up to N = 8), the message naming the widest window at that N. */
int b2_split_tracks_capped(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off /* [V+1] */, int V,
                           const int32_t* track_video /* [T] */, int T, const double* cue_start_s,
                           const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */,
                           const double* ratio /* [T] */, int sample_rate, double start_seconds,
                           int64_t max_offset_samples, double split_penalty, int max_segments, int32_t* cue_offset,
                           int32_t* n_segments /* [T] */, double* split_score /* [T] */,
                           double* split_profile /* [T x max_segments] */, int memspace);
/* b2_split_tracks_wide with segment offsets that only move one way along the track (DESIGN.md section 4 "K9s", the
 * directed programme).  direction = +1: offsets only grow (the video has breaks the subtitles lack: ad breaks, an
 * intermission); -1: offsets only shrink (the subtitles have content the video lacks: a cut release, a pruned recap).
 * A switch at offset o may only come from an offset o' < o (+1) or o' > o (-1):
 *     P_{j-1}(o) = max { V_{j-1}(o') : o' on that side of o }  (-inf when empty),
 *     V_j(o) = u_j(o) + max(V_{j-1}(o), P_{j-1}(o) - split_penalty)
 * with b2_split_tracks' rounding, tie (staying wins) and argmax rules; a switch's source is the argmax of V_{j-1} over
 * that side, the largest offset among equal maxima.  The path is monotone in the direction, and at split_penalty =
 * +inf every output equals b2_split_tracks_wide's.  Outputs, memspaces, three-level handling and the 16 384-cue limit
 * are b2_split_tracks_wide's.  Refusals: those of b2_split_tracks_wide; B2_ERR_BAD_ARG for a direction other than
 * +-1; B2_ERR_UNSUPPORTED for a window wider than 16 384 offsets x the widest cluster of this call's kernel the
 * device co-schedules (16 CTAs, 262 144 offsets, on an H100), the message naming the limit. */
int b2_split_tracks_directed(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off /* [V+1] */, int V,
                             const int32_t* track_video /* [T] */, int T, const double* cue_start_s,
                             const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */,
                             const double* ratio /* [T] */, int sample_rate, double start_seconds,
                             int64_t max_offset_samples, double split_penalty, int direction, int32_t* cue_offset,
                             int32_t* n_segments /* [T] */, double* split_score /* [T] */, int memspace);
/* b2_split_tracks_wide along stated breaks (DESIGN.md section 4 "K9s", the programme along breaks): breaks [n_breaks]
 * (HOST) lists d_1 .. d_n, each +1 (that break moves the offset up: an ad break, an intermission) or -1 (down: a cut,
 * a pruned recap), 1 <= n <= 15.  A path may have m <= n breaks, and its i-th break (in track order) moves the offset
 * strictly in direction d_i.  Layer m holds the paths with exactly m breaks:
 *     V_{0,0} = u_0,  V_{0,m} = -inf (m >= 1),  V_{j,0}(o) = u_j(o) + V_{j-1,0}(o),
 *     V_{j,m}(o) = u_j(o) + max(V_{j-1,m}(o), P^{d_m}_{j-1,m-1}(o) - split_penalty)  (m >= 1)
 * with P^{+1} the maximum over o' < o, P^{-1} over o' > o (-inf when empty), and b2_split_tracks' rounding and tie
 * (staying wins) rules.  The path ends at the largest V_{last,m}(o) over (m, o), ties to the largest offset and then
 * the smallest m; a break's source is the argmax of V_{j-1,m-1} over the d_m side, the largest offset among equal
 * maxima.  cue_offset, n_segments (= m + 1) and split_score come from that path.  split_profile [T x (n + 1)] (f64,
 * in memspace): split_profile[t*(n+1) + m] = max_o V_{last,m}(o), the best penalised objective with exactly m breaks
 * following d_1 .. d_m (-inf when no such path fits the window or the units, NaN for a track whose n_segments is
 * <= 0).  At split_penalty = +inf every output equals b2_split_tracks_wide's, with split_profile[t*(n+1)] finite and
 * the other columns -inf.  Outputs, memspaces, three-level handling and the 16 384-cue limit are b2_split_tracks_wide's.
 * Refusals: those of b2_split_tracks_wide; B2_ERR_BAD_ARG for n_breaks < 1 or an entry other than +-1;
 * B2_ERR_UNSUPPORTED for n_breaks > 15 and for a window wider than this call's envelope at that n: 512 x 32 / L
 * offsets a CTA (L = the smallest of 2, 4, 8, 16 holding n + 1 layers) x the widest cluster of the kernel for L the
 * device co-schedules, the message naming the limit. */
int b2_split_tracks_breaks(b2_handle h, const void* ref, int ref_is_f64, const int64_t* ref_off /* [V+1] */, int V,
                           const int32_t* track_video /* [T] */, int T, const double* cue_start_s,
                           const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */,
                           const double* ratio /* [T] */, int sample_rate, double start_seconds,
                           int64_t max_offset_samples, double split_penalty, const int32_t* breaks /* [n_breaks] */,
                           int n_breaks, int32_t* cue_offset, int32_t* n_segments /* [T] */,
                           double* split_score /* [T] */, double* split_profile /* [T x (n_breaks + 1)] */,
                           int memspace);
/* try_sync's output step (ffsubsync/ffsubsync.py:272-286, SubtitleScaler + SubtitleShifter) with each cue's own
 * offset: for a track with n_segments > 0, cue i gets timedelta(seconds=t_i * ratio[t]) + timedelta(seconds=
 * cue_offset[i] / sample_rate + apply_offset_seconds), each rounded half-to-even to the microsecond as b2_apply_sync
 * rounds them, and status WRITTEN | APPLIED; other tracks are FAILED and keep their original times.  The quality gate
 * and suppression do not apply.  ratio and the cue tables are host metadata; n_segments, cue_offset and the outputs
 * follow memspace (B2_DEVICE: one kernel on the handle's stream, a chain of resident sync calls stays intact).
 * B2_ERR_BAD_ARG as for b2_apply_sync. */
int b2_apply_split(b2_handle h, const double* ratio /* [T] */, const int32_t* n_segments /* [T] */,
                   const int32_t* cue_offset, int T, const double* cue_start_s, const double* cue_end_s,
                   const int64_t* cue_off /* [T+1] */, int sample_rate, double apply_offset_seconds,
                   int64_t* synced_start_us, int64_t* synced_end_us, int32_t* status /* [T] */, int memspace);

/* ---- diagnostics for tests: the aligner's nomination stage ----------------------------------
 * Exposes the fp32 correlation the aligner nominates candidates from - the conv[] array of
 * ffsubsync/aligners.py:67-80 over the offsets that survive the mask, and the argmax of :45-48 before
 * the exact float64 re-score.  While set, every aligner stage on this handle (b2_align_batch,
 * b2_sync_batch) also writes, for each (pair, ratio) j = b*K + k of the call, into caller-owned DEVICE
 * arrays (on the handle's stream):
 *   win[2j], win[2j+1]    first surviving offset, number of surviving offsets (0: empty / all masked)
 *   stat[2j], stat[2j+1]  fp32 maximum over the window, round-off bound tau
 *   cand[j]               offsets with fp32 score >= max - tau (uncapped count); -1 = B2_ALIGN_APPROX
 *   scores[j*stride + i]  fp32 score of offset win[2j] + i, 0 <= i < win[2j+1]
 * The arrays must hold B*K entries (x2 for win and stat).  A window longer than stride fails the call
 * with B2_ERR_BAD_ARG.  scores == NULL clears the capture.  Not for production use: each capture costs
 * one extra launch per alignment (per group of the large-window path).
 * A capture keeps cue-mode calls on the FFT paths, unless the environment sets B2_ALIGN_PATH=runs and the
 * run path fits the call; then the fields hold the run path's nomination stage:
 *   scores                its float64 score of each offset (exact counts, see DESIGN.md 4 "K4r"), rounded to fp32
 *   stat[2j], stat[2j+1]  float64 maximum and margin epsilon in place of tau, both rounded to fp32
 *   cand[j]               offsets with score >= max - epsilon (uncapped count); -1 = B2_ALIGN_APPROX */
int b2_capture_nominations(b2_handle h, float* scores, int64_t stride, int64_t* win, float* stat,
                           int32_t* cand);

/* ---- diagnostics for tests: the batched sync calls' reference signals ------------------------
 * Exposes the per-video reference signal a batched sync call (b2_sync_batch, b2_sync_tracks, _gss, _auditok,
 * _subs, _pgs, _sig) builds in its detector step - the detector's output, the tokenised auditok signal, a rasterised
 * subtitle / PGS reference or a serialized signal's frames, ffsubsync/speech_transformers.py's
 * VideoSpeechTransformer.fit / DeserializeSpeechTransformer.fit output.  While set, every
 * such call with at least one track writes, overwriting the previous call's:
 *   ref[0 .. ref_off[V])  its reference buffer (DEVICE array; one device-to-device copy on the handle's stream after
 *                         the call's last kernel).  Video v's signal is ref[ref_off[v] .. ref_off[v+1]) as float32,
 *                         or, when packed[v] is set, ceil(R/32) uint32 words of bits m = (r == 1.0f) from ref_off[v]
 *                         on (R = ref_off[v+1] - ref_off[v]; zero bits past R; the rest of the range is not the
 *                         signal's).
 *   ref_off[0 .. V]       HOST array: the call's per-video offsets.
 *   packed[0 .. V-1]      HOST array: 1 where the video's sub-batch got packed words, else 0.
 * A call needing more than `capacity` floats or `max_videos` videos fails with B2_ERR_BAD_ARG before anything is
 * enqueued.  The capture changes nothing the call plans, launches or returns.  ref == NULL clears the capture. */
int b2_capture_reference(b2_handle h, float* ref, int64_t capacity, int64_t* ref_off, uint8_t* packed,
                         int64_t max_videos);

/* ---- speech output of the batched sync calls (--serialize-speech) ----------------------------
 * While set on a handle, every batched sync call (b2_sync_batch, b2_sync_tracks, _gss, _auditok, _subs, _pgs, _sig,
 * _seg) writes the reference signal of each listed video as float64: listed video i = videos[i] lands at
 * speech[speech_off[i] .. speech_off[i+1]), its length the call's own reference length (b2_vad_num_windows frames for
 * energy / ZCR, the chunk loop's blocks for auditok, int(max_end*sr) + 2 for a text stream or PGS, int(seg_total*sr)
 * + 2 for segments, the stored length for a signal).  Each frame is the float32 frame the call aligned against,
 * widened: VideoSpeechTransformer's output rounded to float32 for detector videos, the rasterised stream for text,
 * PGSSpeechTransformer for PGS, the sparse MultiSegmentVideoSpeechTransformer signal for segments and
 * DeserializeSpeechTransformer(label) for signal videos.  Videos the call flags (best_k -2 or -3) are written too, as
 * the call built them (a stored value > 1.0 or NaN as the label).  A call with T == 0 has no tracks to carry those
 * flags: a segment video's signal without a frame > 0 is written as it is, and the caller applies the reference's
 * no-speech rule to it (batch.save_serialized_speech does).
 * speech_off is a HOST array of n_videos + 1 entries that each call fills when it is planned.  The call fails with
 * B2_ERR_BAD_ARG before anything is enqueued when the listed videos need more than `capacity` frames, when a listed
 * video is >= V, or when the call's memspace is not the output's (B2_DEVICE_RESIDENT counts as B2_DEVICE).
 * memspace B2_DEVICE: speech is device memory of the handle's device, written by one kernel behind the call's last
 * chain with no host synchronisation.  B2_HOST: speech is host memory, copied back with the call's results.
 * A call with T == 0 and the output set runs the detector step of the listed videos and writes them, and nothing
 * else (the reference's serialize-only run); without the output T == 0 returns at once, as before.
 * videos must be increasing and >= 0; a host speech pointer under B2_DEVICE is refused.  Setting or clearing the
 * output enqueues nothing and leaves a chain of resident calls intact; with it cleared every call plans, launches
 * and returns what it does without it.  speech == NULL clears it. */
int b2_speech_output(b2_handle h, double* speech, int64_t capacity, const int32_t* videos /* [n], increasing */,
                     int n_videos, int64_t* speech_off /* host [n+1], written by each call */, int memspace);
/* MultiSegmentVideoSpeechTransformer.fit's reference length int(total_seconds * sample_rate) + 2, or -1 when total is
 * not finite, too large, or gives a negative length (the length b2_sync_tracks_seg gives a segment video) */
int64_t b2_segment_length(double total_seconds, int sample_rate);

/* ---- batched ingest session: the chunk loop for a batch of decoders --------------------------------------------
 * The reference reads ffmpeg's pipe 100 s at a time and runs the detector on each chunk as it arrives
 * (ffsubsync/speech_transformers.py:680-753).  A session does that for V videos at once: their PCM arrives as host
 * chunks of any size in any interleaving across videos, the detector runs on the device as they come, and only each
 * video's reference signal stays on the device - never its PCM.  A final call runs the batched sync chain over them.
 * Let P_v be all bytes pushed for video v, in push order, with a trailing odd byte dropped.  Whatever the cut of P_v
 * into pushes (1-byte and odd pushes, pushes that split a window or a detector call) and the interleaving:
 *   energy / ZCR   video v's reference is b2_vad_energy_zcr over each b2_vad_call_samples call of P_v (over P_v
 *                  where that is 0), b2_vad_num_windows frames, a call's partial last window non-speech;
 *   auditok        it is b2_vad_auditok over P_v with chunk_samples, rounded once to float32: the tokenizer restarts
 *                  at every chunk_samples boundary of P_v wherever the pushes fell (read(n) on a pipe returns n bytes
 *                  until EOF, so the stream fixes the boundaries, not the caller);
 *   the sync call  returns exactly what b2_sync_tracks (b2_sync_tracks_gss with gss_ratio) for energy / ZCR, or
 *                  b2_sync_tracks_auditok for auditok, returns for the same tracks and arguments over the PCM
 *                  P_0 ... P_{V-1} back to back, b2_speech_output included.
 * b2_ingest_begin     opens the session: the detector arguments and their checks are b2_sync_tracks_subs's (detector,
 *                     label, energy_threshold, z_lo, z_hi for energy / ZCR; energy_threshold_db ... chunk_samples for
 *                     auditok).  expect_samples [V] (or NULL) is a sizing hint, e.g. ffprobe's duration: a video that
 *                     outgrows it grows its buffer, it never fails.  B2_ERR_BAD_ARG for a second begin.
 * b2_ingest_push      appends n host chunks: chunk i (bytes[i], n_bytes[i] bytes) to video video[i]; within a video
 *                     in push order.  The library copies the chunks before it returns (the caller may reuse its buffers
 *                     at once), enqueues the copy to the device and the detector on the handle's stream and returns
 *                     without a host synchronisation (it waits only for the push three calls earlier to have left its
 *                     staging slot).  B2_ERR_BAD_ARG (the message names the chunk) for a video out of range, a negative
 *                     n_bytes or a null chunk with n_bytes > 0; such a call pushes nothing.
 * b2_ingest_windows   windows [V]: the reference frames the pushes so far fix (an unfinished window is held back).
 * b2_ingest_sync_tracks  flushes every video's held-back samples, then runs the chain of b2_sync_tracks (with the
 *                     search when gss_ratio is not NULL) over the references: arguments and outputs as there, memspace
 *                     (B2_HOST or B2_DEVICE) for the outputs only.  T == 0 with b2_speech_output set writes only the
 *                     signals (the reference's serialize-only run).  The session closes, whatever the outcome.
 * b2_ingest_abort     closes the session without a sync (no session: nothing to do).
 * A push, windows or sync call without an open session is B2_ERR_BAD_ARG.  A failed call leaves the handle usable.
 * The handle stays single-threaded: decoder threads hand their chunks to the one thread that pushes. */
int b2_ingest_begin(b2_handle h, int V, int frame_rate, int sample_rate, int detector, double non_speech_label,
                    int64_t energy_threshold, int z_lo, int z_hi, double energy_threshold_db, double min_length,
                    int64_t max_length, double max_continuous_silence, int64_t chunk_samples,
                    const int64_t* expect_samples /* [V] or NULL */);
int b2_ingest_push(b2_handle h, int n, const int32_t* video /* [n] */, const void* const* bytes /* [n] */,
                   const int64_t* n_bytes /* [n] */);
int b2_ingest_windows(b2_handle h, int64_t* windows /* [V] */);
int b2_ingest_sync_tracks(b2_handle h, const int32_t* track_video /* [T] */, int T, const double* cue_start_s,
                          const double* cue_end_s, const uint8_t* cue_keep, const int64_t* cue_off /* [T+1] */,
                          const double* ratios, int K, double start_seconds, int64_t max_offset_samples,
                          double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                          double* all_score, int32_t* all_offset /* [T*K], [T*(K+1)] with the search, or NULL */,
                          double* gss_ratio /* [T] or NULL = grid only */, double* gss_evals /* [T*17] or NULL */,
                          int memspace);
/* b2_ingest_sync_refs  b2_ingest_sync_tracks with references that need no audio: the reference tables of
 *                     b2_sync_tracks_sig, in its order (text streams ref_is_subs .. ref_cue_off, PGS intervals
 *                     ref_is_pgs .. pgs_off, stored signals ref_is_sig, x, sig_off; each group may be NULL), then
 *                     b2_ingest_sync_tracks' arguments.  A reference video has no pushes (empty P_v).  The call
 *                     returns exactly what b2_sync_tracks_seg returns for the same tracks, arguments and tables over
 *                     the PCM P_0 ... P_{V-1} back to back with the session's segment table (as b2_ingest_sync_tracks
 *                     builds it): b2_speech_output, B2_BEST_K_BAD_SIGNAL, B2_BEST_K_NO_SPEECH, the label / level / path
 *                     rules and their B2_ERR_UNSUPPORTED refusals included.  B2_ERR_BAD_ARG for a text, PGS or signal
 *                     video that received pushed bytes (the message names it), for a segment video given a reference,
 *                     and for every table refusal of b2_sync_tracks_sig / _seg.  memspace covers the outputs and x:
 *                     B2_HOST stages a host x, B2_DEVICE refuses one.  The tables are host arrays.  The session closes
 *                     whatever the outcome; b2_ingest_sync_tracks is this call with every table NULL. */
int b2_ingest_sync_refs(b2_handle h, const uint8_t* ref_is_subs /* [V] or NULL */, const double* ref_cue_start_s,
                        const double* ref_cue_end_s, const uint8_t* ref_cue_keep, const int64_t* ref_cue_off /* [V+1] */,
                        const uint8_t* ref_is_pgs /* [V] or NULL */, const double* pgs_start_s, const double* pgs_end_s,
                        const int64_t* pgs_off /* [V+1] */, const uint8_t* ref_is_sig /* [V] or NULL */,
                        const double* x, const int64_t* sig_off /* [V+1] */, const int32_t* track_video /* [T] */,
                        int T, const double* cue_start_s, const double* cue_end_s, const uint8_t* cue_keep,
                        const int64_t* cue_off /* [T+1] */, const double* ratios, int K, double start_seconds,
                        int64_t max_offset_samples, double* best_score, int32_t* best_offset, int32_t* best_k /* [T] */,
                        double* all_score, int32_t* all_offset, double* gss_ratio, double* gss_evals, int memspace);
int b2_ingest_abort(b2_handle h);

/* ---- sampled segments in a session (--multi-segment-sync) ------------------------------------------------------
 * MultiSegmentVideoSpeechTransformer.fit decodes only a few windows of each video (ffmpeg -ss start -t duration per
 * segment, ffsubsync/speech_transformers.py:849-900) and skips a segment whose decode fails.  A session does that for
 * segment videos next to audio videos: each segment's PCM is pushed on its own, the detector runs on it as it arrives
 * (energy / ZCR restarts its windows and auditok its chunk loop at the segment's first sample), and the sync assembles
 * the sparse reference on the device.  Let S_{v,j} be all bytes pushed to live (not dropped) segment j of video v,
 * trailing odd byte dropped.  The sync call returns exactly what b2_sync_tracks_seg returns for the same tracks and
 * arguments over the PCM of each audio video's pushes and each segment video's live S_{v,j} back to back in segment
 * order, with the segment table seg_lo / seg_hi over those pieces and the dropped segments removed - b2_speech_output,
 * B2_BEST_K_NO_SPEECH (a video whose segments were all dropped or never pushed included) and the label-0 rule of the
 * search included.
 * b2_ingest_segments      declares the segment videos: seg_video [P] (increasing), seg_total [P] (probed duration,
 *                         seconds), seg_off [P+1], seg_start (whole seconds, increasing per video); the checks are
 *                         b2_sync_tracks_seg's.  At most once per session, before any push to a listed video.
 *                         b2_ingest_begin's expect_samples[v] of a segment video is the hint for each of its segments.
 * b2_ingest_push_segments appends chunk i to segment segment[i] (counted within its video) of video video[i]; copies
 *                         and enqueues as b2_ingest_push.  Segments and videos may interleave in any order.
 *                         B2_ERR_BAD_ARG (the message names the chunk; nothing is pushed) for a video without segments,
 *                         a segment out of range or a dropped segment; b2_ingest_push refuses a segment video.
 * b2_ingest_drop_segment  discards a segment (what was pushed to it and any later push, refused): it takes no part in
 *                         the reference and overwrites no earlier segment (the reference's "failed to extract segment").
 * b2_ingest_windows gives a segment video the frames its live segments have fixed so far. */
int b2_ingest_segments(b2_handle h, int P, const int32_t* seg_video /* [P] */, const double* seg_total /* [P] */,
                       const int64_t* seg_off /* [P+1] */, const int64_t* seg_start);
int b2_ingest_push_segments(b2_handle h, int n, const int32_t* video /* [n] */, const int64_t* segment /* [n] */,
                            const void* const* bytes /* [n] */, const int64_t* n_bytes /* [n] */);
int b2_ingest_drop_segment(b2_handle h, int video, int64_t segment);

/* ---- synthetic PCM (bench / tests): counter-hash generator replayable in numpy -------------
 * oracle/vad_oracle.py:synth_pcm.  window_class: uint8 per 10 ms window (0 silence, 1 voiced,
 * 2 loud hiss), device or host per memspace; writes n_windows*fpw int16 samples. */
int b2_synth_pcm(b2_handle h, const uint8_t* window_class, int64_t n_windows, int fpw,
                 uint32_t seed, int16_t* pcm_out, int memspace);

#ifdef __cplusplus
}
#endif
#endif /* FFSUBSYNC_B200_H */
