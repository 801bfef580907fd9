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
 * pcm: int16 mono samples of all B signals back to back (memspace); out: float per window. */
int b2_vad_frames_per_window(int frame_rate, int sample_rate);
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
 * (ffsubsync/ffsubsync.py:637 + :196-235).  pcm and the outputs follow memspace; memspace may also be
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

/* ---- synthetic PCM (bench / tests): counter-hash generator replayable in numpy -------------
 * oracle/vad_oracle.py:synth_pcm.  window_class: uint8 per 10 ms window (0 silence, 1 voiced,
 * 2 loud hiss), device or host per memspace; writes n_windows*fpw int16 samples. */
int b2_synth_pcm(b2_handle h, const uint8_t* window_class, int64_t n_windows, int fpw,
                 uint32_t seed, int16_t* pcm_out, int memspace);

#ifdef __cplusplus
}
#endif
#endif /* FFSUBSYNC_B200_H */
