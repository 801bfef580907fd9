// Host-side plan of one batched sync call (b2_sync_batch, b2_sync_tracks, b2_sync_tracks_gss,
// b2_sync_tracks_auditok, b2_sync_tracks_subs, b2_sync_tracks_pgs, b2_sync_tracks_sig, b2_sync_tracks_seg): every argument check and every
// host table the pipeline in api.cu reads.  No CUDA call happens here, so tests/host_emul/plan_emul.cu runs the same code on the CPU.
#pragma once

#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "align_path.h"    // b2_plan_align_jobs, b2_align_path
#include "common.cuh"      // B2_FAIL, B2TokenizerParams
#include "corr_jobs.cuh"   // kRunMaxCues, kRunMaxWindow
#include "job_plan.cuh"    // B2_GSS_HI, b2_signal_length, B2_MAX_CUE_SECONDS

// ---- cue lists --------------------------------------------------------------------------------
// Bits of |x| as an integer: ordered like |x| for every double, with inf above every finite value and
// NaN above inf, so one integer maximum over a cue array finds its largest or non-finite time.
static inline uint64_t magnitude_bits(double x) {
  uint64_t u;
  memcpy(&u, &x, 8);
  return u & 0x7fffffffffffffffull;
}

static inline double from_bits(uint64_t u) {
  double x;
  memcpy(&x, &u, 8);
  return x;
}

// The cue arithmetic (raster_math.cuh) reproduces the reference for finite times with
// |t| * ratio < B2_MAX_CUE_SECONDS; fl(|t| * r) is monotone in |t| and r, so the largest magnitude and
// the largest ratio of a pair decide.  NaN and inf fail the comparison.
static inline bool cue_magnitude_ok(uint64_t max_bits, double r_max) {
  return from_bits(max_bits) * r_max < B2_MAX_CUE_SECONDS;
}

static inline bool ratio_ok(double r) { return r > 0.0 && r < INFINITY; }

// Why the cues of pairs [0, B) cannot be rasterised exactly, or nullptr: start_seconds, a ratio that is
// not finite and positive, or a cue time (start or end; either array may be null = not checked) beyond
// the limit above.  For non-finite times the reference raises in timedelta.  Metadata cues count: the
// reference scales them too.  *at: the offending ratio or cue index, *val its value.
static const char* bad_cue_input(const double* cue_start_s, const double* cue_end_s, const int64_t* cue_off,
                                 int B, const double* ratios, int K, int per_pair_ratios, double start_seconds,
                                 int64_t* at, double* val) {
  *at = -1;
  *val = start_seconds;
  if (!(fabs(start_seconds) < B2_MAX_CUE_SECONDS)) return "start_seconds is not finite or too large";
  for (int b = 0; b < B; ++b) {
    double r_max = 0.0;
    for (int k = 0; k < K; ++k) {
      const size_t i = per_pair_ratios ? (size_t)b * K + k : (size_t)k;
      *at = (int64_t)i;
      *val = ratios[i];
      if (!ratio_ok(ratios[i])) return "ratio is not a finite positive number";
      r_max = std::max(r_max, ratios[i]);
    }
    const int64_t c0 = cue_off[b], c1 = cue_off[b + 1];
    for (const double* t : {cue_start_s, cue_end_s}) {
      if (!t) continue;
      // one branch-free pass (four independent chains); the offending cue is looked for only on failure
      uint64_t m4[4] = {0, 0, 0, 0};
      int64_t c = c0;
      for (; c + 4 <= c1; c += 4)
        for (int i = 0; i < 4; ++i) m4[i] = std::max(m4[i], magnitude_bits(t[c + i]));
      for (; c < c1; ++c) m4[0] = std::max(m4[0], magnitude_bits(t[c]));
      if (cue_magnitude_ok(std::max(std::max(m4[0], m4[1]), std::max(m4[2], m4[3])), r_max)) continue;
      for (int64_t c = c0; c < c1; ++c)
        if (!cue_magnitude_ok(magnitude_bits(t[c]), r_max)) {
          *at = c;
          *val = t[c];
          return t == cue_start_s ? "cue start time times ratio is not finite or too large"
                                  : "cue end time times ratio is not finite or too large";
        }
    }
  }
  return nullptr;
}

// b2_rasterize_lengths, also checking the start times when cue_start_s is not null (the sync calls: one
// pass over the cues for both)
static int rasterize_lengths(const double* cue_start_s, const double* cue_end_s, const int64_t* cue_off, int B,
                             const double* ratios, int K, int per_pair_ratios, int sample_rate, int64_t* lengths) {
  if (B < 0 || K < 0 || !cue_off || (!ratios && K) || !lengths || sample_rate <= 0)
    return B2_ERR_BAD_ARG;
  for (int b = 0; b < B; ++b) {
    // max over cues of scaled(end) == scaled(max end) for ratio > 0: the product, the microsecond
    // rounding and the division are all monotone non-decreasing (speech_transformers.py:958-960).
    // The same pass finds the largest magnitude for the input check (see bad_cue_input).
    // (four independent chains: this runs over every cue of every b2_sync_batch call).  A NaN end
    // fails the check, so max_end may ignore it.
    const int64_t c0 = cue_off[b], c1 = cue_off[b + 1];
    const bool any = c1 > c0;
    double e4[4];
    uint64_t m4[4] = {0, 0, 0, 0};
    for (int i = 0; i < 4; ++i) e4[i] = any ? cue_end_s[c0] : 0.0;
    int64_t c = c0;
    for (; c + 4 <= c1; c += 4)
      for (int i = 0; i < 4; ++i) {
        e4[i] = std::max(e4[i], cue_end_s[c + i]);
        m4[i] = std::max(m4[i], magnitude_bits(cue_end_s[c + i]));
        if (cue_start_s) m4[i] = std::max(m4[i], magnitude_bits(cue_start_s[c + i]));
      }
    for (; c < c1; ++c) {
      e4[0] = std::max(e4[0], cue_end_s[c]);
      m4[0] = std::max(m4[0], magnitude_bits(cue_end_s[c]));
      if (cue_start_s) m4[0] = std::max(m4[0], magnitude_bits(cue_start_s[c]));
    }
    const double max_end = std::max(std::max(e4[0], e4[1]), std::max(e4[2], e4[3]));
    const uint64_t m = std::max(std::max(m4[0], m4[1]), std::max(m4[2], m4[3]));
    for (int k = 0; k < K; ++k) {
      double r = per_pair_ratios ? ratios[(size_t)b * K + k] : ratios[k];
      if (!ratio_ok(r) || !cue_magnitude_ok(m, r)) return B2_ERR_BAD_ARG;
      lengths[(size_t)b * K + k] = b2_signal_length(any ? max_end : 0.0, r, sample_rate);
    }
  }
  return B2_OK;
}

// The signal lengths of the cue lists [0, B) at the K shared ratios, with start_seconds and every cue time
// checked.  The lengths pass checks too; the offending input is looked for only on failure, and the message is
// "<who>: <what><why> (index i: value)".  When no single input is to blame the message is "<who>: <fallback>",
// or with a null fallback "<who>: <what>bad cue list (index -1: start_seconds)".
static int cue_lengths(std::string* err, const char* who, const char* what, const char* fallback,
                       const double* cue_start_s, const double* cue_end_s, const int64_t* cue_off, int B,
                       const double* ratios, int K, double start_seconds, int sample_rate, int64_t* lengths) {
  if (fabs(start_seconds) < B2_MAX_CUE_SECONDS &&
      rasterize_lengths(cue_start_s, cue_end_s, cue_off, B, ratios, K, 0, sample_rate, lengths) == B2_OK)
    return B2_OK;
  int64_t at;
  double val;
  const char* why = bad_cue_input(cue_start_s, cue_end_s, cue_off, B, ratios, K, 0, start_seconds, &at, &val);
  char b[512];
  if (why || !fallback)
    snprintf(b, sizeof(b), "%s: %s%s (index %lld: %g)", who, what, why ? why : "bad cue list", (long long)at, val);
  else
    snprintf(b, sizeof(b), "%s: %s", who, fallback);
  *err = b;
  return B2_ERR_BAD_ARG;
}

// ---- PGS interval lists ------------------------------------------------------------------------
// Why interval list [i0, i1) cannot be rasterised by PGSSpeechTransformer.fit's rule (raster_math.cuh b2_pgs_bounds),
// or nullptr; else *len = its signal length int(max_end * sample_rate) + 2.  The reference raises for an empty list
// (ValueError), a non-finite time (round / int) and a negative length (np.zeros); times of magnitude
// B2_MAX_CUE_SECONDS and more are rejected too, so that every frame index fits an int64.  start_s may be null (not
// checked: b2_rasterize_pgs_lengths).  *at: the offending interval (-1: the list), *val its value.
static const char* pgs_list_check(const double* start_s, const double* end_s, int64_t i0, int64_t i1, int sample_rate,
                                  int64_t* len, int64_t* at, double* val) {
  *at = -1;
  *val = (double)(i1 - i0);
  if (i1 <= i0) return "empty interval list";
  double max_end = end_s[i0];
  for (int64_t i = i0; i < i1; ++i) {
    for (const double* t : {start_s, end_s}) {
      if (!t || fabs(t[i]) < B2_MAX_CUE_SECONDS) continue;
      *at = i;
      *val = t[i];
      return t == start_s ? "interval start time is not finite or too large" : "interval end time is not finite or too large";
    }
    max_end = std::max(max_end, end_s[i]);
  }
  *len = b2_pgs_length(max_end, sample_rate);
  if (*len < 0) {
    *val = max_end;
    return "negative signal length int(max_end * sample_rate) + 2";
  }
  return nullptr;
}

// The signal lengths of the interval lists [0, B) (off [B+1], absolute), with sample_rate, the offset table, null
// arrays, start_seconds and the start times (when check_start) and every time checked; lists with only && !only[b] are skipped (length -1).  Messages
// "<who>: <what><why> (index i: value)"; the index is the interval's, or "list b" for a list-level error.
static int pgs_lengths(std::string* err, const char* who, const char* what, const double* start_s, const double* end_s,
                       const int64_t* off, int B, int sample_rate, bool check_start, double start_seconds,
                       const uint8_t* only, int64_t* lengths) {
  char b[512];
  if (sample_rate <= 0 || sample_rate > B2_PGS_MAX_SAMPLE_RATE) {
    snprintf(b, sizeof(b), "%s: sample_rate %d is out of (0, %d]", who, sample_rate, B2_PGS_MAX_SAMPLE_RATE);
    *err = b;
    return B2_ERR_BAD_ARG;
  }
  if (check_start && !(fabs(start_seconds) < B2_MAX_CUE_SECONDS)) {
    snprintf(b, sizeof(b), "%s: start_seconds is not finite or too large (%g)", who, start_seconds);
    *err = b;
    return B2_ERR_BAD_ARG;
  }
  // the whole table first: only a monotone one bounds every list by [off[0], off[B]), so that a null array is
  // read by no list exactly when that range is empty
  for (int v = 0; v < B; ++v)
    if (off[v + 1] < off[v]) {
      snprintf(b, sizeof(b), "%s: %soff not monotone at %d", who, what, v);
      *err = b;
      return B2_ERR_BAD_ARG;
    }
  if (B > 0 && off[B] > off[0] && (!end_s || (check_start && !start_s))) {
    snprintf(b, sizeof(b), "%s: null %sinterval arrays", who, what);
    *err = b;
    return B2_ERR_BAD_ARG;
  }
  for (int v = 0; v < B; ++v) {
    lengths[v] = -1;
    if (only && !only[v]) continue;
    int64_t at;
    double val;
    if (const char* why = pgs_list_check(start_s, end_s, off[v], off[v + 1], sample_rate, &lengths[v], &at, &val)) {
      if (at < 0) snprintf(b, sizeof(b), "%s: %s%s (list %d: %g)", who, what, why, v, val);
      else snprintf(b, sizeof(b), "%s: %s%s (index %lld: %g)", who, what, why, (long long)at, val);
      *err = b;
      return B2_ERR_BAD_ARG;
    }
  }
  return B2_OK;
}

// ---- detectors --------------------------------------------------------------------------------
static inline int vad_frames_per_window(int frame_rate, int sample_rate) {
  if (frame_rate <= 0 || sample_rate <= 0) return 0;
  // speech_transformers.py:163-164: int(window_duration * frame_rate + 0.5)
  return (int)((1.0 / (double)sample_rate) * (double)frame_rate + 0.5);
}

// The reference's chunk loop reads (2 fr // sr) * 5000 samples per detector call (VideoSpeechTransformer._chunks:
// (2 fr // sr) * 10000 bytes), and energy / ZCR restarts its window grid in every call, so a call that is not a whole
// number of windows ends in a non-speech partial window and the next call's windows start on a new grid (22.05 kHz:
// 2 205 000 samples of 221-sample windows).  The samples per call where that happens; 0 where the calls divide into
// windows (8, 11.025, 12, 16, 24, 32, 44.1, 48, 96 kHz), since one call over the whole video then gives the same
// frames.
static inline int64_t energy_call_samples(int frame_rate, int sample_rate) {
  const int fpw = vad_frames_per_window(frame_rate, sample_rate);
  if (fpw <= 0) return 0;
  const int64_t call = (2 * (int64_t)frame_rate / sample_rate) * 5000;
  return call % fpw ? call : 0;
}

// Frames of a detector over n samples cut into calls of `call` samples (0: one call), windows of fpw
static inline int64_t chunked_num_windows(int64_t n, int fpw, int64_t call) {
  if (call <= 0) return (n + fpw - 1) / fpw;
  return n / call * ((call + fpw - 1) / fpw) + (n % call + fpw - 1) / fpw;
}

static inline int auditok_block_size(int frame_rate, int sample_rate) {
  if (frame_rate <= 0 || sample_rate <= 0) return 0;
  // ADSFactory.ads(block_dur=1.0/sample_rate): int(sampling_rate * block_dur), speech_transformers.py:140;
  // the output length formula uses frame_rate // sample_rate (:122,143-145): the two must agree
  volatile double dur = 1.0 / (double)sample_rate;
  volatile double prod = (double)frame_rate * dur;
  const int block = (int)prod;
  return block == frame_rate / sample_rate ? block : 0;
}

static inline int64_t auditok_energy_floor(int n_samples, double energy_threshold_db) {
  // smallest integer sum of squares E with 10*log10(E/n) >= threshold, evaluated with the same
  // float64 expression auditok's AudioEnergyValidator uses (log energy -200 for E = 0)
  if (n_samples <= 0) return INT64_MAX;
  if (-200.0 >= energy_threshold_db) return 0;
  auto valid = [&](int64_t e) {
    volatile double energy = (double)e / (double)n_samples;
    volatile double le = 10.0 * log10(energy);
    return le >= energy_threshold_db;
  };
  const double guess = (double)n_samples * pow(10.0, energy_threshold_db / 10.0);
  const double e_max = (double)n_samples * 32768.0 * 32768.0;   // int16 blocks cannot exceed this
  if (!(guess <= 2.0 * e_max)) return INT64_MAX;
  int64_t lo = 0, hi = (int64_t)guess + 1;                       // !valid(0) holds: log energy -200
  while (!valid(hi)) {
    if ((double)hi > 4.0 * e_max) return INT64_MAX;
    hi *= 2;
  }
  while (hi - lo > 1) {
    const int64_t mid = lo + (hi - lo) / 2;
    if (valid(mid)) hi = mid;
    else lo = mid;
  }
  return hi;
}

// StreamTokenizer.__init__'s argument checks, and a chunk length that is not negative
static inline bool tokenizer_params_ok(double min_length, int64_t max_length, double max_continuous_silence,
                                       int64_t chunk_samples) {
  return max_length > 0 && min_length > 0 && min_length <= (double)max_length &&
         max_continuous_silence < (double)max_length && chunk_samples >= 0;
}

// The reference's chunk loop.  Video v is cut into detector calls of chunk_samples samples (0: one call),
// chunks first[v] .. first[v+1]-1; chunk c spans samples pcm[c] .. pcm[c+1] (relative to `base`) and blocks
// out[c] .. out[c+1] of the detector's output, ceil(len/fpw) of them, so a video's signal is the sum over its
// chunks of ceil(len/fpw) long.  tail[c]: the energy floor of the chunk's short last block (0: none).  Chunk
// starts are multiples of chunk_samples from the video's start ((2 fr // sr) * 5000 samples in the Python layer:
// a multiple of 8, so aligned videos stay eligible for the lane-per-window energy kernel).
// With subs_len (b2_sync_tracks_subs / _pgs), a video with subs_len[v] >= 0 has a subtitle reference (text or PGS) and no PCM: it is
// one empty chunk spanning its reference's subs_len[v] frames, so the energy pass has no tiles there, and the
// tokenizer's table tok_* (chunks tok_first[v] .. tok_first[v+1]-1, frames tok_off[k] .. tok_end[k]) leaves it
// out, so only the rasteriser writes it.  Without subs_len the tok_* tables stay empty (the tokenizer reads out).
// A video whose pcm_off decreases gets no chunk; callers reject it.
struct ChunkTable {
  std::vector<int64_t> pcm, out, tail, tok_off, tok_end;
  std::vector<int> first, tok_first;
};

static void build_chunk_table(const int64_t* pcm_off, int V, int64_t base, int fpw, int64_t chunk_samples,
                              double energy_threshold_db, const int64_t* subs_len, ChunkTable* ct) {
  ct->first.assign(V + 1, 0);
  ct->pcm.assign(1, V ? pcm_off[0] - base : 0);
  ct->out.assign(1, 0);
  if (subs_len) ct->tok_first.assign(V + 1, 0);
  int tail_rem = -1;
  int64_t tail_floor = 0;
  for (int v = 0; v < V; ++v) {
    const int64_t n = pcm_off[v + 1] - pcm_off[v];
    if (subs_len && subs_len[v] >= 0) {
      ct->pcm.push_back(pcm_off[v + 1] - base);
      ct->out.push_back(ct->out.back() + subs_len[v]);
      ct->tail.push_back(0);
    } else {
      const int64_t step = chunk_samples > 0 ? chunk_samples : (n > 0 ? n : 1);
      for (int64_t s = 0; s < n; s += step) {
        const int64_t len = std::min(step, n - s);
        ct->pcm.push_back(pcm_off[v] - base + s + len);
        ct->out.push_back(ct->out.back() + (len + fpw - 1) / fpw);
        const int rem = (int)(len % fpw);
        if (rem && rem != tail_rem) {
          tail_rem = rem;
          tail_floor = auditok_energy_floor(rem, energy_threshold_db);
        }
        ct->tail.push_back(rem ? tail_floor : 0);
        if (subs_len) {
          ct->tok_off.push_back(ct->out[ct->out.size() - 2]);
          ct->tok_end.push_back(ct->out.back());
        }
      }
    }
    ct->first[v + 1] = (int)ct->tail.size();
    if (subs_len) ct->tok_first[v + 1] = (int)ct->tok_off.size();
  }
}

// ---- the request and its plan ----------------------------------------------------------------
// Everything one batched sync call received.  Only the arguments of `detector` are read.
struct SyncRequest {
  const char* who;                 // the entry point, as messages name it
  const int16_t* pcm;
  const int64_t* pcm_off;          // [V+1]
  int V;
  const int32_t* track_video;      // [T], non-decreasing; null: V == T, track t against video t (b2_sync_batch)
  int T;
  int frame_rate, sample_rate;
  int detector;                    // B2_DETECTOR_ENERGY_ZCR or B2_DETECTOR_AUDITOK
  struct {
    float non_speech_label;
    int64_t energy_threshold;
    int z_lo, z_hi;                // < 0: defaults
  } energy;
  struct {                         // b2_vad_auditok's arguments
    double non_speech_label, energy_threshold_db, min_length, max_continuous_silence;
    int64_t max_length, chunk_samples;
  } auditok;
  // Subtitle references (b2_sync_tracks_subs; cue_off null: none): videos with is_subs[v] != 0 take their cue
  // list cue_off[v] .. cue_off[v+1] (host arrays, absolute indices), rasterised at ratio 1.0 and level 1.0, as
  // reference signal instead of the detector's output.
  struct {
    const uint8_t* is_subs;        // may be null: no video
    const double* cue_start_s;
    const double* cue_end_s;
    const uint8_t* cue_keep;       // may be null
    const int64_t* cue_off;        // [V+1]
  } refs;
  const double* cue_start_s;
  const double* cue_end_s;
  const uint8_t* cue_keep;         // may be null
  const int64_t* cue_off;          // [T+1]
  const double* ratios;            // [K]
  int K;
  double start_seconds;
  int64_t max_offset_samples;
  double* best_score;
  int32_t* best_offset;
  int32_t* best_k;
  double* all_score;               // may be null; [T*K], or [T*(K+1)] with the search
  int32_t* all_offset;
  bool search;                     // the golden-section search runs as candidate K
  double* gss_ratio;               // [T]: the search's ratio
  double* gss_evals;               // may be null
  int memspace;
  // PGS references (b2_sync_tracks_pgs; off null: none): videos with is_pgs[v] != 0 take their intervals
  // off[v] .. off[v+1] (host arrays, absolute indices), rasterised by PGSSpeechTransformer's rule, as reference
  // signal.  The value-initialised state is "no PGS video", so the other entry points leave it out.
  struct {
    const uint8_t* is_pgs;         // may be null: no video
    const double* start_s;
    const double* end_s;
    const int64_t* off;            // [V+1]
  } pgs;
  // Serialized speech signals (b2_sync_tracks_sig; off null: none): videos with is_sig[v] != 0 take the stored
  // float64 values x[off[v] .. off[v+1]) (x follows memspace, off is a host array of absolute indices), each
  // frame (float)(x < 1.0 ? label : x) (DeserializeSpeechTransformer), as reference signal.  The
  // value-initialised state is "no signal video", so the other entry points leave it out.
  struct {
    const uint8_t* is_sig;         // may be null: no video
    const double* x;
    const int64_t* off;            // [V+1]
  } sig;
  // Sampled segments (b2_sync_tracks_seg, --multi-segment-sync; off null: none): video video[i] (increasing) has the
  // probed duration total[i] seconds and the segments off[i] .. off[i+1]-1, segment j starting at start[j] whole
  // seconds (strictly increasing within a video) with the samples pcm_off[v] + lo[j] .. pcm_off[v] + hi[j].  Its
  // reference is MultiSegmentVideoSpeechTransformer.fit's sparse signal.  All host arrays; the value-initialised state
  // is "no segment video", so the other entry points leave it out.
  struct {
    int n;                         // P: videos with segments
    const int32_t* video;          // [P]
    const double* total;           // [P]
    const int64_t* off;            // [P+1]
    const int64_t* start;          // per segment
    const int64_t* lo;
    const int64_t* hi;
  } seg;
  // Ingested references (b2_ingest_sync_tracks; len null: none): every video's reference is already on the device,
  // the detector's output over its PCM as the ingest session's pushes wrote it - video v's len[v] frames at
  // ref + at[v] (at, len: host arrays [V]).  The call has no PCM (pcm_off all equal); its detector step copies the
  // references into the reference buffer, and the videos count as detector videos for every level and path rule.
  // The value-initialised state is "no ingested references", so the other entry points leave it out.
  // With sampled segments (seg.off set; their sample ranges lo / hi all empty) a segment video's reference is
  // assembled from its segments' detector output, segment j's seg_len[j] frames at ref + seg_at[j] (indexed as
  // seg.start), and its own len is not read.
  struct {
    const float* ref;
    const int64_t* at;
    const int64_t* len;
    const int64_t* seg_at;
    const int64_t* seg_len;
  } ready;
};

// What plan_sync reads from the handle and the environment: the SM count, the most sub-batches the handle's
// event pool orders, B2_SUBBATCHES / B2_VAD_SMS (null: unset) and the energy kernel's lane-per-window
// eligibility test (b2i_vad_lane_eligible).
// For the reference format (plan_ref_format) also what the aligner's path choice reads (align_path.h): the
// handle's log2 quirk mask and capture state, B2_ALIGN_PATH, whether the subtitle signals are bit masks
// (B2_FUSED_RASTER), and B2_REF_PACKED ("0": every reference as floats).
struct SyncPipeEnv {
  int sm_count, max_sub;
  const char* subbatches;
  const char* vad_sms;
  bool (*lane_eligible)(const int64_t* pcm_off, int n, int fpw);
  uint64_t quirk_mask = 0;
  bool capture = false;
  const char* align_path = nullptr;
  bool fused = true;
  const char* ref_packed = nullptr;
  bool speech_out = false;         // b2_speech_output is set: a call without tracks still plans its references
};

struct SyncPlan {
  std::string err;
  bool gss = false, auditok = false;
  bool any_subs = false;           // a video has a subtitle reference, text or PGS (levels 1 and 0, no PCM)
  int fpw = 0, z_lo = 0, z_hi = 0;
  // Samples per detector call (0: one call per video): auditok's chunk_samples, or energy_call_samples.  The main
  // detector launch runs over the chunk table ch when chunked: always for auditok, for energy / ZCR where call > 0.
  int64_t call = 0;
  bool chunked = false;
  // the reference's levels (B2CueSource::ref_label / ref_two_level)
  float label = 0.0f, ref_label = 0.0f;
  bool two_level = false;
  int64_t audio_samples = 0;       // samples the detector reads
  std::vector<int> trk_off;        // [V+1]: first track of video v
  std::vector<int64_t> ref_off;    // [V+1]: reference signal of video v
  std::vector<int64_t> sub_off;    // [T*K+1]: float subtitle signal of job j (unfused raster)
  std::vector<int> sub_video;      // the videos with a text subtitle reference, ascending
  std::vector<int> pgs_video;      // the videos with a PGS reference, ascending
  std::vector<int> sig_video;      // the videos with a serialized signal reference, ascending
  // a video's reference is not the detector's (text, PGS or signal): it has no PCM, its length comes from its
  // reference, and the tokenizer's table leaves it out.  Without signal videos this is any_subs.
  bool any_ref = false;
  ChunkTable ch;                   // chunked
  int64_t auditok_e_min = 0;
  B2TokenizerParams tok{0.0, 0.0, 0.0, 0};
  std::vector<double> max_end;     // GSS: each track's largest cue end (its signal length at any ratio)
  // Sub-batches of the pipeline: videos cut[i] .. cut[i+1]-1; the later ones' detector runs on vad_sms SMs
  int n_sub = 1, vad_sms = 0;
  std::vector<int> cut;
  // per sub-batch: its detector writes the reference as packed bits instead of floats (plan_ref_format)
  std::vector<uint8_t> ref_packed;
  // Sampled segments (plan_segments).  seg_video: the segment videos, ascending; seg_of[v]: v's index into the
  // request's seg arrays, -1 for other videos.
  std::vector<int> seg_video, seg_of;
  // det_end: with segment videos, the end of every entry of the main detector launch (videos, or auditok's chunks),
  // which then starts at r.pcm_off / ch.pcm as before; a segment video's entry is empty (its PCM is read only through
  // the segment items below).  Empty without segment videos.
  std::vector<int64_t> det_end;
  // The detector launch over the sampled segments: item k reads the samples item_start[k] .. item_end[k] (absolute
  // in the call's pcm) and writes the scratch frames item_out[k] .. item_out[k+1]; item_tail[k] is auditok's energy
  // floor of its short last block (0: none).  One item per detector call of `call` samples from the segment's first
  // sample (the window grid and auditok's tokenizer restart in every item), one per segment without calls.  item_first[v] .. item_first
  // [v+1]-1: the items of video v (none for other videos).  item_start has one spare entry (the vad launch's table
  // has n + 1 entries).  seg_frames: the scratch's size.
  std::vector<int64_t> item_start, item_end, item_out, item_tail;
  std::vector<int> item_first;
  int64_t seg_frames = 0;
  // Owned frames of segment video seg_video[i]: runs run_first[i] .. run_first[i+1]-1 cover its reference [0, L) in
  // order; run r starts at frame run_lo[r] and ends where the next starts (or at L), and takes scratch frames from
  // run_src[r] on (-1: 0.0, no segment covers it).  Segments write in increasing start order, the later one wins.
  std::vector<int> run_first;
  std::vector<int64_t> run_lo, run_src;
  // B2_HOST with segment videos: the sample ranges [stage_lo[i], stage_hi[i]) (ascending, disjoint) that the
  // detector reads - the audio videos' and the segments' - copied to the device at their own positions.
  std::vector<int64_t> stage_lo, stage_hi;
};

// Sub-batches are cut at video boundaries (a video's tracks run in the chain behind its own VAD) and balanced by
// track count, since the chain's work scales with tracks: cut i is the first video whose tracks start at or
// after track T*i/n_sub.  With one track per video these are T*i/n_sub exactly.  Cuts that would leave a
// sub-batch without tracks are dropped; a video without tracks has its VAD run in the sub-batch of the next video
// that has tracks (trailing ones: of the last).  Where the cuts fall changes no result.
// Defaults: 3 sub-batches, the later VADs on 54 % of the SMs (71 of an H100's 132; tools/pipeline_probe.py sweeps
// both), on the lane-per-window kernel only; small batches stay unpipelined (the alignment of a third of a small
// batch is launch- and tail-bound).  B2_SUBBATCHES / B2_VAD_SMS override the defaults; 1 / 0 = off.
// Lane eligibility of ranges [start[i], end[i]) that need not abut (the tables of a call with segment videos): each
// non-empty range on its own, and the window size through an empty table.
static bool ranges_lane_ok(const SyncPipeEnv& env, const int64_t* start, const int64_t* end, int n, int fpw) {
  bool ok = env.lane_eligible(start, 0, fpw);
  for (int i = 0; i < n && ok; ++i) {
    const int64_t t[2] = {start[i], end[i]};
    if (end[i] > start[i]) ok = env.lane_eligible(t, 1, fpw);
  }
  return ok;
}

// The audio videos [v0, v1) of the main detector launch (segment videos are empty there)
static bool audio_lane_ok(const SyncRequest& r, const SyncPipeEnv& env, const SyncPlan* p, int v0, int v1) {
  if (p->det_end.empty()) return env.lane_eligible(r.pcm_off + v0, v1 - v0, p->fpw);
  return ranges_lane_ok(env, r.pcm_off + v0, p->det_end.data() + v0, v1 - v0, p->fpw);
}

static void plan_cuts(const SyncRequest& r, const SyncPipeEnv& env, SyncPlan* p) {
  const int V = r.V, T = r.T;
  if (r.ready.len) {   // ingested references: no detector step for the chains to overlap
    p->n_sub = 1;
    p->vad_sms = 0;
    p->cut = {0, V};
    return;
  }
  // lane eligibility is decided on the tables the energy kernel reads: the videos, or the detector calls, and the
  // sampled segments' items
  bool lane_ok;
  if (p->det_end.empty())
    lane_ok = p->chunked ? env.lane_eligible(p->ch.pcm.data(), (int)p->ch.tail.size(), p->fpw)
                         : env.lane_eligible(r.pcm_off, V, p->fpw);
  else
    lane_ok = (p->chunked ? ranges_lane_ok(env, p->ch.pcm.data(), p->det_end.data(), (int)p->ch.tail.size(), p->fpw)
                          : audio_lane_ok(r, env, p, 0, V)) &&
              ranges_lane_ok(env, p->item_start.data(), p->item_end.data(), (int)p->item_end.size(), p->fpw);
  p->n_sub = 1;
  p->vad_sms = 0;
  if (T >= 96 && lane_ok) {
    p->n_sub = 3;
    p->vad_sms = (env.sm_count * 54 + 50) / 100;
  }
  if (env.subbatches) p->n_sub = std::max(1, std::min(T, atoi(env.subbatches)));
  if (env.vad_sms) p->vad_sms = std::max(0, std::min(env.sm_count, atoi(env.vad_sms)));
  p->n_sub = std::min(p->n_sub, env.max_sub);
  const std::vector<int>& trk_off = p->trk_off;
  p->cut.assign(1, 0);   // every sub-batch holds at least one track
  for (int i = 1; i < p->n_sub; ++i) {
    const int target = (int)((int64_t)T * i / p->n_sub);
    const int v = (int)(std::lower_bound(trk_off.begin(), trk_off.end(), target) - trk_off.begin());
    if (trk_off[v] > trk_off[p->cut.back()] && trk_off[v] < T) p->cut.push_back(v);
  }
  p->cut.push_back(V);
  p->n_sub = (int)p->cut.size() - 1;
}

// The reference format of each sub-batch.  The run path reads a reference only as its bits m = (r == 1.0f) (and
// r = m ? 1.0f : ref_label in the exact re-score), so a sub-batch whose detector is the lane-per-window energy
// kernel, with no subtitle reference, whose chain takes the run path has its VAD write those bits, 32 to a word,
// instead of the floats: 1/32 of the bytes written, and the chain reads bits instead of floats.  The chain's path
// is decided here by the aligner's own functions on the chain's own inputs (align_path.h, as enqueue_chain passes
// them), so the launcher reaches the same choice.  auditok, energy / ZCR cut into detector calls (packed words hold
// whole videos, not calls), subtitle references, the lane-group kernel and the FFT paths keep the float reference
// (text and PGS references alike).  B2_REF_PACKED=0 keeps it everywhere (A/B knob).
// Serialized signal references (b2_sync_tracks_sig) have the bits too: sig_ref_kernel writes them, so a sub-batch
// whose videos are all signal videos or lane-eligible energy audio is packed like an audio one, with either
// detector (auditok sub-batches qualify only when every video is a signal video).
// Sampled-segment references (b2_sync_tracks_seg) likewise: seg_ref_kernel writes their bits, so they count like
// signal videos (their chains take the run path only at label 0, where the reference has the levels 1.0 and 0.0).
static void plan_ref_format(const SyncRequest& r, const SyncPipeEnv& env, SyncPlan* p) {
  p->ref_packed.assign(p->n_sub, 0);
  // ingested audio references are floats; the run path packs them itself (ref_bits_kernel).  Segment and signal
  // videos' ones are written at sync by seg_ref_kernel and sig_ref_kernel, which write bits as they do for
  // b2_sync_tracks_seg / _sig; text and PGS ones are rasterised as floats there as in the whole call.
  const size_t n_written = p->seg_video.size() + p->sig_video.size();
  if ((r.ready.len && n_written < (size_t)r.V) || (p->auditok && p->sig_video.empty() && p->seg_video.empty()) ||
      !env.fused || (env.ref_packed && atoi(env.ref_packed) == 0))
    return;
  // how many videos of `list` lie in [v0, v1)
  auto count = [](const std::vector<int>& list, int v0, int v1) {
    return (int)(std::lower_bound(list.begin(), list.end(), v1) - std::lower_bound(list.begin(), list.end(), v0));
  };
  for (int i = 0; i < p->n_sub; ++i) {
    const int v0 = p->cut[i], v1 = p->cut[i + 1];
    if (count(p->sub_video, v0, v1) || count(p->pgs_video, v0, v1)) continue;
    const bool all_sig = count(p->sig_video, v0, v1) + count(p->seg_video, v0, v1) == v1 - v0;
    if (!all_sig && (p->chunked || !audio_lane_ok(r, env, p, v0, v1))) continue;
    const int t0 = p->trk_off[v0], nt = p->trk_off[v1] - t0;
    std::vector<int> chain_trk(v1 - v0 + 1);
    for (int v = v0; v <= v1; ++v) chain_trk[v - v0] = p->trk_off[v] - t0;
    B2AlignJobs aj;   // a chain the aligner rejects keeps the floats (and fails there with its message)
    if (b2_plan_align_jobs(p->ref_off.data() + v0, v1 - v0, chain_trk.data(), p->sub_off.data() + (size_t)t0 * r.K,
                           nt, r.K, r.max_offset_samples, env.quirk_mask, r.ratios, &aj) != B2_OK)
      continue;
    const B2AlignPathChoice c = b2_align_path(aj, chain_trk.data(), v1 - v0, r.K, r.cue_off + t0, p->two_level,
                                              p->ref_label, env.align_path, env.capture);
    p->ref_packed[i] = c.path == B2_PATH_RUNS;
  }
}

// Checks of the subtitle references (text and PGS) and of the signal references, before anything reads their
// tables.  *any_audio: a video's reference is the detector's; *any_sig: a video has a signal reference.
static int plan_refs_check(const SyncRequest& r, SyncPlan* p, bool* any_audio, bool* any_sig) {
  const char* who = r.who;
  const auto& s = r.refs;
  const auto& g = r.pgs;
  const auto& q = r.sig;
  for (int v = 0; v < r.V; ++v) {
    const bool is_subs = s.cue_off && s.is_subs && s.is_subs[v];
    const bool is_pgs = g.off && g.is_pgs && g.is_pgs[v];
    const bool is_sig = q.off && q.is_sig && q.is_sig[v];
    const bool is_seg = !p->seg_of.empty() && p->seg_of[v] >= 0;
    if (is_seg && (is_subs || is_pgs || is_sig))
      B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has sampled segments and a %s reference; a video has one reference",
              who, v, is_sig ? "serialized signal" : is_pgs ? "PGS" : "text subtitle");
    if (q.off) {
      if (q.off[v + 1] < q.off[v]) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: sig_off not monotone at %d", who, v);
      if (!is_sig && q.off[v + 1] != q.off[v])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has signal values but no signal reference (ref_is_sig[%d] = 0)",
                who, v, v);
      if (is_sig && is_subs)
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d is marked both as a signal and as a text subtitle reference", who, v);
      if (is_sig && is_pgs)
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d is marked both as a signal and as a PGS reference", who, v);
      if (is_sig && r.pcm_off[v + 1] != r.pcm_off[v])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has a signal reference and a non-empty PCM range (%lld samples); "
                "its audio is never read", who, v, (long long)(r.pcm_off[v + 1] - r.pcm_off[v]));
    }
    if (s.cue_off) {
      if (s.cue_off[v + 1] < s.cue_off[v]) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: ref_cue_off not monotone at %d", who, v);
      if (!is_subs && s.cue_off[v + 1] != s.cue_off[v])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has reference cues but no subtitle reference (ref_is_subs[%d] = 0)",
                who, v, v);
      if (is_subs && r.pcm_off[v + 1] != r.pcm_off[v])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has a subtitle reference and a non-empty PCM range (%lld samples); "
                "its audio is never read", who, v, (long long)(r.pcm_off[v + 1] - r.pcm_off[v]));
    }
    if (g.off) {
      if (g.off[v + 1] < g.off[v]) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: pgs_off not monotone at %d", who, v);
      if (!is_pgs && g.off[v + 1] != g.off[v])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has PGS intervals but no PGS reference (ref_is_pgs[%d] = 0)", who,
                v, v);
      if (is_pgs && is_subs)
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d is marked both as a PGS and as a text subtitle reference", who, v);
      if (is_pgs && r.pcm_off[v + 1] != r.pcm_off[v])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has a PGS reference and a non-empty PCM range (%lld samples); "
                "its audio is never read", who, v, (long long)(r.pcm_off[v + 1] - r.pcm_off[v]));
    }
    p->any_subs = p->any_subs || is_subs || is_pgs;
    *any_audio = *any_audio || (!is_subs && !is_pgs && !is_sig && !is_seg);
    *any_sig = *any_sig || is_sig;
  }
  if (s.cue_off && r.V > 0 && s.cue_off[r.V] > s.cue_off[0] && (!s.cue_start_s || !s.cue_end_s))
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null reference cue arrays", who);
  if (g.off && r.V > 0 && g.off[r.V] > g.off[0] && (!g.start_s || !g.end_s))
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null PGS interval arrays", who);
  if (q.off && r.V > 0 && q.off[r.V] > q.off[0] && !q.x)
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null signal values x with %lld values", who, (long long)(q.off[r.V] - q.off[0]));
  if (p->audio_samples > 0 && !r.pcm)
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null pcm with %lld samples of audio", who, (long long)p->audio_samples);
  return B2_OK;
}

// The envelope of the device-driven GSS rounds (DESIGN.md section 4 "K8g"): every round runs on the run path.
static int plan_gss_check(const SyncRequest& r, SyncPlan* p, bool auditok_two_level) {
  const char* who = r.who;
  // (compared with half the window bound: 2 * max_offset_samples overflows for widths from 2^62 on)
  if (r.max_offset_samples == B2_MAX_OFFSET_NONE || r.max_offset_samples < 0 ||
      r.max_offset_samples > (int64_t)(kRunMaxWindow / 2))
    B2_FAIL(p, B2_ERR_UNSUPPORTED, "sync_tracks_gss: max_offset_samples must lie in [0, %d] (a window of at most "
            "2 max_offset_samples <= %d offsets, one CTA of the run path)", kRunMaxWindow / 2, kRunMaxWindow);
  if (!std::isfinite(p->ref_label))
    B2_FAIL(p, B2_ERR_UNSUPPORTED, "sync_tracks_gss: non_speech_label must be finite (the run path's two-level reference)");
  if (!p->seg_video.empty() && p->label != 0.0f)
    B2_FAIL(p, B2_ERR_UNSUPPORTED, "%s: sampled segments (0.0 outside them) at non_speech_label = %g give three "
            "levels; the search runs on the run path, which needs label 0", who, (double)p->label);
  if (!p->two_level && !auditok_two_level)
    B2_FAIL(p, B2_ERR_UNSUPPORTED, "%s: non_speech_label = %g gives the auditok signal more than two levels; the "
            "search runs on the run path, which needs label 0", who, r.auditok.non_speech_label);
  if (!p->two_level)
    B2_FAIL(p, B2_ERR_UNSUPPORTED, "%s: subtitle references (levels 1 and 0) and audio references (levels 1 and "
            "non_speech_label = %g) in one call give three levels; the search runs on the run path, which needs "
            "label 0 or references of one kind", who, (double)p->label);
  for (int t = 0; t < r.T; ++t)
    if (r.cue_off[t + 1] - r.cue_off[t] > kRunMaxCues)
      B2_FAIL(p, B2_ERR_UNSUPPORTED, "sync_tracks_gss: track %d has %lld cues, more than %d", t,
              (long long)(r.cue_off[t + 1] - r.cue_off[t]), kRunMaxCues);
  return B2_OK;
}

// MultiSegmentVideoSpeechTransformer.fit's reference length int(total * sample_rate) + 2 (float64 product,
// truncated), or -1 when total is not finite, too large, or gives a negative length
static inline int64_t seg_ref_length(double total, int sample_rate) {
  if (!(fabs(total) < B2_MAX_CUE_SECONDS) || sample_rate <= 0) return -1;
  const int64_t len = (int64_t)(total * (double)sample_rate) + 2;
  return len >= 0 ? len : -1;
}

// Checks of the segment table, before anything reads it; fills seg_video / seg_of and counts the segments' samples
// (and no other sample of a segment video) in audio_samples.
static int plan_seg_check(const SyncRequest& r, SyncPlan* p) {
  const char* who = r.who;
  const auto& s = r.seg;
  const int P = s.n;
  if (P < 0 || (P > 0 && (!s.video || !s.total))) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: bad segment videos (%d)", who, P);
  for (int i = 0; i < P; ++i)
    if (s.off[i + 1] < s.off[i]) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: seg_off not monotone at %d", who, i);
  if (P > 0 && s.off[P] > s.off[0] && (!s.start || !s.lo || !s.hi))
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null segment arrays with %lld segments", who, (long long)(s.off[P] - s.off[0]));
  p->seg_of.assign(r.V, -1);
  for (int i = 0; i < P; ++i) {
    const int v = s.video[i];
    if (v < 0 || v >= r.V || (i > 0 && v <= s.video[i - 1]))
      B2_FAIL(p, B2_ERR_BAD_ARG, "%s: seg_video[%d] = %d is out of [0, %d) or not increasing", who, i, v, r.V);
    p->seg_of[v] = i;
    p->seg_video.push_back(v);
    if (seg_ref_length(s.total[i], r.sample_rate > 0 ? r.sample_rate : 1) < 0)
      B2_FAIL(p, B2_ERR_BAD_ARG, "%s: seg_total[%d] = %g (video %d) is not finite, too large, or gives a negative "
              "signal length int(total * sample_rate) + 2", who, i, s.total[i], v);
    const int64_t n = r.pcm_off[v + 1] - r.pcm_off[v];
    if (n < 0) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: pcm_off not monotone", who);
    p->audio_samples -= n;
    for (int64_t j = s.off[i]; j < s.off[i + 1]; ++j) {
      if (s.start[j] < 0 || (double)s.start[j] >= B2_MAX_CUE_SECONDS)
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: segment %lld of video %d starts at %lld s, outside [0, %.0f)", who,
                (long long)j, v, (long long)s.start[j], B2_MAX_CUE_SECONDS);
      if (j > s.off[i] && s.start[j] <= s.start[j - 1])
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: segment %lld of video %d starts at %lld s, not after the previous one (%lld s)",
                who, (long long)j, v, (long long)s.start[j], (long long)s.start[j - 1]);
      if (s.lo[j] < 0 || s.hi[j] < s.lo[j] || s.hi[j] > n)
        B2_FAIL(p, B2_ERR_BAD_ARG, "%s: segment %lld of video %d has the sample range [%lld, %lld), not inside the "
                "video's PCM range [0, %lld)", who, (long long)j, v, (long long)s.lo[j], (long long)s.hi[j],
                (long long)n);
      p->audio_samples += s.hi[j] - s.lo[j];
    }
  }
  return B2_OK;
}

// The owned-frame runs of every segment video (SyncPlan run_*): segment j's detector output is len[j] frames from
// src[j] on (indexed as r.seg.start); a sweep in start order, each segment overwriting [begin, min(begin + len, L))
// of the runs so far.
static void plan_seg_runs(const SyncRequest& r, SyncPlan* p, const int64_t* src, const int64_t* len) {
  const auto& s = r.seg;
  p->run_first.assign(1, 0);
  p->run_lo.clear();
  p->run_src.clear();
  for (int v : p->seg_video) {
    const int i = p->seg_of[v];
    const int64_t L = p->ref_off[v + 1] - p->ref_off[v];
    struct Piece { int64_t lo, hi, src; };
    std::vector<Piece> owned, next;
    for (int64_t j = s.off[i]; j < s.off[i + 1]; ++j) {
      const int64_t b = s.start[j] * (int64_t)r.sample_rate, e = std::min(b + len[j], L);
      if (e <= b) continue;
      next.clear();
      for (const Piece& q : owned) {
        if (q.lo < b) next.push_back({q.lo, std::min(q.hi, b), q.src});
        if (q.hi > e) next.push_back({std::max(q.lo, e), q.hi, q.src + (std::max(q.lo, e) - q.lo)});
      }
      next.push_back({b, e, src[j]});
      std::sort(next.begin(), next.end(), [](const Piece& x, const Piece& y) { return x.lo < y.lo; });
      owned.swap(next);
    }
    int64_t at = 0;
    for (const Piece& q : owned) {
      if (q.lo > at) {
        p->run_lo.push_back(at);
        p->run_src.push_back(-1);
      }
      p->run_lo.push_back(q.lo);
      p->run_src.push_back(q.src);
      at = q.hi;
    }
    if (at < L) {
      p->run_lo.push_back(at);
      p->run_src.push_back(-1);
    }
    p->run_first.push_back((int)p->run_lo.size());
  }
}

// The segment videos' tables (SyncPlan: det_end, item_*, run_*, stage_*), after ref_off and the chunk table.
static void plan_segments(const SyncRequest& r, SyncPlan* p) {
  const auto& s = r.seg;
  const int V = r.V, fpw = p->fpw;
  // the main launch: every entry as before, a segment video's empty
  if (p->chunked) {
    const int nc = (int)p->ch.tail.size();
    p->det_end.assign(p->ch.pcm.begin() + 1, p->ch.pcm.begin() + 1 + nc);
    for (int v : p->seg_video) p->det_end[p->ch.first[v]] = p->ch.pcm[p->ch.first[v]];
  } else {
    p->det_end.assign(r.pcm_off + 1, r.pcm_off + V + 1);
    for (int v : p->seg_video) p->det_end[v] = r.pcm_off[v];
  }
  // the segments' items: one per detector call of `call` samples from the segment's first sample (one per segment
  // without calls)
  p->item_first.assign(V + 1, 0);
  p->item_out.assign(1, 0);
  p->item_start.clear();
  p->item_end.clear();
  p->item_tail.clear();
  std::vector<int64_t> seg_scr(s.n > 0 ? (size_t)(s.off[s.n] - s.off[0]) : 0), seg_len(seg_scr.size());
  int tail_rem = -1;
  int64_t tail_floor = 0;
  for (int v = 0; v < V; ++v) {
    const int i = p->seg_of[v];
    for (int64_t j = i < 0 ? 0 : s.off[i]; i >= 0 && j < s.off[i + 1]; ++j) {
      const int64_t a = r.pcm_off[v] + s.lo[j], n = s.hi[j] - s.lo[j];
      seg_scr[j - s.off[0]] = p->item_out.back();
      const int64_t step = p->call > 0 ? p->call : (n > 0 ? n : 1);
      for (int64_t c = 0; c < n; c += step) {
        const int64_t len = std::min(step, n - c);
        p->item_start.push_back(a + c);
        p->item_end.push_back(a + c + len);
        p->item_out.push_back(p->item_out.back() + (len + fpw - 1) / fpw);
        const int rem = (int)(len % fpw);
        if (p->auditok && rem && rem != tail_rem) {
          tail_rem = rem;
          tail_floor = auditok_energy_floor(rem, r.auditok.energy_threshold_db);
        }
        p->item_tail.push_back(p->auditok && rem ? tail_floor : 0);
      }
      seg_len[j - s.off[0]] = p->item_out.back() - seg_scr[j - s.off[0]];
    }
    p->item_first[v + 1] = (int)p->item_end.size();
  }
  p->item_start.push_back(p->item_start.empty() ? 0 : p->item_start.back());
  p->seg_frames = p->item_out.back();
  plan_seg_runs(r, p, seg_scr.data() - (s.n > 0 ? s.off[0] : 0), seg_len.data() - (s.n > 0 ? s.off[0] : 0));
  // B2_HOST: the ranges the detector reads, merged
  std::vector<std::pair<int64_t, int64_t>> rg;
  for (int v = 0; v < V; ++v)
    if (p->seg_of[v] < 0 && r.pcm_off[v + 1] > r.pcm_off[v])
      rg.push_back({r.pcm_off[v], r.pcm_off[v + 1]});
  for (size_t k = 0; k < p->item_end.size(); ++k) rg.push_back({p->item_start[k], p->item_end[k]});
  std::sort(rg.begin(), rg.end());
  p->stage_lo.clear();
  p->stage_hi.clear();
  for (const auto& [a, b] : rg) {
    if (!p->stage_hi.empty() && a <= p->stage_hi.back()) p->stage_hi.back() = std::max(p->stage_hi.back(), b);
    else {
      p->stage_lo.push_back(a);
      p->stage_hi.push_back(b);
    }
  }
}

// The lengths of the videos whose reference is not the detector's, in (*subs_len)[v] (-1: a detector video), and the
// lists sub_video, pgs_video and sig_video; the cue and interval times are checked on the way.
static int plan_ref_lengths(const SyncRequest& r, SyncPlan* p, std::vector<int64_t>* subs_len) {
  const char* who = r.who;
  const int V = r.V;
  // subtitle references: int(max_end * sample_rate) + 2 frames (speech_transformers.py:958-962), the length
  // b2_rasterize gives at ratio 1.0; the lengths pass checks the cue times too (the same checks and messages as
  // the tracks' cues).  (*subs_len)[v] = -1: the video's reference is the detector's.
  // PGS references: int(max_end * sample_rate) + 2 frames, the length b2_rasterize_pgs_lengths gives.
  // Signal references: one frame per stored value, sig_off[v+1] - sig_off[v].
  subs_len->assign(V, -1);
  const uint8_t* is_subs = r.refs.cue_off ? r.refs.is_subs : nullptr;
  const uint8_t* is_pgs = r.pgs.off ? r.pgs.is_pgs : nullptr;
  if (is_subs && std::any_of(is_subs, is_subs + V, [](uint8_t x) { return x != 0; })) {
    const double one = 1.0;
    B2_TRY(cue_lengths(&p->err, who, "reference ", "bad reference cue list", r.refs.cue_start_s, r.refs.cue_end_s,
                       r.refs.cue_off, V, &one, 1, r.start_seconds, r.sample_rate, subs_len->data()));
    for (int v = 0; v < V; ++v) {
      if (is_subs[v]) p->sub_video.push_back(v);
      else (*subs_len)[v] = -1;
    }
  }
  if (is_pgs) {
    std::vector<int64_t> pgs_len(V);
    B2_TRY(pgs_lengths(&p->err, who, "PGS ", r.pgs.start_s, r.pgs.end_s, r.pgs.off, V, r.sample_rate, true,
                       r.start_seconds, is_pgs, pgs_len.data()));
    for (int v = 0; v < V; ++v)
      if (is_pgs[v]) {
        p->pgs_video.push_back(v);
        (*subs_len)[v] = pgs_len[v];
      }
  }
  if (r.sig.off && r.sig.is_sig)
    for (int v = 0; v < V; ++v)
      if (r.sig.is_sig[v]) {
        p->sig_video.push_back(v);
        (*subs_len)[v] = r.sig.off[v + 1] - r.sig.off[v];
      }
  // Segment references: int(total * sample_rate) + 2 frames (speech_transformers.py:871)
  for (int v : p->seg_video) (*subs_len)[v] = seg_ref_length(r.seg.total[p->seg_of[v]], r.sample_rate);
  return B2_OK;
}

// The detector's window size and arguments, and each video's reference length.
static int plan_references(const SyncRequest& r, SyncPlan* p) {
  const char* who = r.who;
  const int V = r.V;
  if (p->auditok) {   // b2_vad_auditok's checks
    p->fpw = auditok_block_size(r.frame_rate, r.sample_rate);
    if (p->fpw <= 0)
      B2_FAIL(p, B2_ERR_UNSUPPORTED, "%s: int(frame_rate/sample_rate) block size and frame_rate//sample_rate window "
              "size differ (or are 0) for %d / %d", who, r.frame_rate, r.sample_rate);
    const auto& a = r.auditok;
    if (!tokenizer_params_ok(a.min_length, a.max_length, a.max_continuous_silence, a.chunk_samples))
      B2_FAIL(p, B2_ERR_BAD_ARG, "%s: bad tokenizer parameters", who);
    p->auditok_e_min = auditok_energy_floor(p->fpw, a.energy_threshold_db);
    p->tok = B2TokenizerParams{a.min_length, a.max_continuous_silence, a.non_speech_label, (long long)a.max_length};
    p->call = a.chunk_samples;
  } else {
    p->fpw = vad_frames_per_window(r.frame_rate, r.sample_rate);
    p->call = energy_call_samples(r.frame_rate, r.sample_rate);
  }
  p->chunked = p->auditok || p->call > 0;
  const int fpw = p->fpw;
  if (fpw <= 0) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: bad frame_rate/sample_rate", who);
  p->z_lo = r.energy.z_lo < 0 ? 0 : r.energy.z_lo;
  p->z_hi = r.energy.z_hi < 0 ? (3 * fpw) / 8 : r.energy.z_hi;
  p->ref_off.assign(V + 1, 0);
  std::vector<int64_t> subs_len;   // [V] with any_ref: each reference video's length, -1 for a detector video
  if (p->any_ref) B2_TRY(plan_ref_lengths(r, p, &subs_len));
  if (r.ready.len) {
    // ingested references: an audio video's length is the pushes' (no chunk table, nothing to detect), a text, PGS,
    // signal or segment video's its reference's, as in the whole call (its ready.len is not read)
    for (int v = 0; v < V; ++v)
      p->ref_off[v + 1] = p->ref_off[v] + (p->any_ref && subs_len[v] >= 0 ? subs_len[v] : r.ready.len[v]);
    // segment videos: their runs point into the session's buffer, not into a scratch of this call
    if (!p->seg_video.empty()) plan_seg_runs(r, p, r.ready.seg_at, r.ready.seg_len);
    return B2_OK;
  }
  for (int v = 0; v < V; ++v) {
    const int64_t n = r.pcm_off[v + 1] - r.pcm_off[v];
    if (n < 0) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: pcm_off not monotone", who);
    if (p->any_ref && subs_len[v] >= 0) p->ref_off[v + 1] = p->ref_off[v] + subs_len[v];
    else if (!p->chunked) p->ref_off[v + 1] = p->ref_off[v] + (n + fpw - 1) / fpw;
  }
  if (p->chunked) {
    // energy / ZCR reads no tail floor (its partial window is non-speech): INFINITY makes them INT64_MAX, never met
    build_chunk_table(r.pcm_off, V, 0, fpw, p->call, p->auditok ? r.auditok.energy_threshold_db : INFINITY,
                      p->any_ref ? subs_len.data() : nullptr, &p->ch);
    for (int v = 0; v < V; ++v) p->ref_off[v + 1] = p->ch.out[p->ch.first[v + 1]];
  }
  if (!p->seg_video.empty()) plan_segments(r, p);
  return B2_OK;
}

// Every argument check and every host table of one batched sync call.  Errors go to p->err with the status.
// T == 0 returns B2_OK after the checks that do not need tracks, with no tables; with env.speech_out it also plans
// the references (ref_off and the detector's tables) as one sub-batch of floats, for the detector step alone.
static int plan_sync(const SyncRequest& r, const SyncPipeEnv& env, SyncPlan* p) {
  const char* who = r.who;
  const int V = r.V, T = r.T, K = r.K;
  p->gss = r.search;
  p->auditok = r.detector == B2_DETECTOR_AUDITOK;
  if (V < 0 || T < 0 || K <= 0 || !r.pcm_off || !r.cue_off || !r.ratios)
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: bad arguments", who);
  bool any_audio = !r.refs.cue_off && !r.pgs.off && !r.sig.off && !r.seg.off, any_sig = false;
  for (int v = 0; v < V; ++v)
    if (r.pcm_off[v + 1] > r.pcm_off[v]) p->audio_samples += r.pcm_off[v + 1] - r.pcm_off[v];
  if (r.seg.off) B2_TRY(plan_seg_check(r, p));
  if (r.refs.cue_off || r.pgs.off || r.sig.off || r.seg.off) B2_TRY(plan_refs_check(r, p, &any_audio, &any_sig));
  const bool any_seg = !p->seg_video.empty();
  p->any_ref = p->any_subs || any_sig || any_seg;
  // The run path and the GSS rounds need a reference of the two levels 1.0 and ref_label.  The detector's signal
  // has the levels 1.0 and the label, a subtitle reference 1.0 and 0.0, so ref_label is the label unless every
  // reference is a subtitle stream; a call that mixes the two at a non-zero label has three levels.  auditok's
  // clipped cumsum has two levels only at label 0 (starts and ends alternate and an overwrite only turns an end
  // into a start, so the integer sum stays in {0, 1}); other labels give further levels (0.3, 0.6, ... for 0.3).
  // A signal reference has the levels 1.0 and the label whichever the detector (its stored values are < 1.0 or
  // exactly 1.0), so it counts like energy audio: a call of signals alone is two-level.
  // A sampled-segment reference has 0.0 outside its segments and the detector's levels inside: {0, 1, label} for
  // energy / ZCR, {0, 1} for auditok at label 0.  It is two-level only at label 0, where it has the levels of a
  // subtitle reference and mixes with text / PGS references and with audio as those do.
  p->label = p->auditok ? (float)r.auditok.non_speech_label : r.energy.non_speech_label;
  p->ref_label = any_audio || any_sig ? p->label : 0.0f;
  const bool auditok_two_level = !p->auditok || r.auditok.non_speech_label == 0.0 || !any_audio;
  const bool mix_two_level = !(p->any_subs || any_seg) || p->label == 0.0f;
  p->two_level = (!any_audio && !any_sig && !any_seg) || (auditok_two_level && mix_two_level);
  if (r.track_video) {
    for (int t = 0; t < T; ++t)
      if (r.track_video[t] < 0 || r.track_video[t] >= V || (t > 0 && r.track_video[t] < r.track_video[t - 1]))
        B2_FAIL(p, B2_ERR_BAD_ARG, "sync_tracks: track_video[%d] = %d is out of [0, %d) or decreases", t,
                (int)r.track_video[t], V);
    for (int t = 0; t < T; ++t)
      if (r.cue_off[t + 1] < r.cue_off[t]) B2_FAIL(p, B2_ERR_BAD_ARG, "sync_tracks: cue_off not monotone at %d", t);
  }
  if (p->gss) B2_TRY(plan_gss_check(r, p, auditok_two_level));
  if (T == 0 && !env.speech_out) return B2_OK;
  if (T == 0) {
    B2_TRY(plan_references(r, p));
    p->trk_off.assign(V + 1, 0);
    p->sub_off.assign(1, 0);
    p->cut = {0, V};
    p->ref_packed.assign(1, 0);
    return B2_OK;
  }
  if (!r.best_score || !r.best_offset || !r.best_k) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null output", who);
  if (p->gss && !r.gss_ratio) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null gss_ratio", who);
  B2_TRY(plan_references(r, p));
  p->trk_off.resize(V + 1);
  for (int v = 0, t = 0; v <= V; ++v) {
    if (r.track_video)
      while (t < T && r.track_video[t] < v) ++t;
    else
      t = v;
    p->trk_off[v] = t;
  }
  const size_t J = (size_t)T * K;
  std::vector<int64_t> lengths(J);
  B2_TRY(cue_lengths(&p->err, who, "", "bad cue list / ratios", r.cue_start_s, r.cue_end_s, r.cue_off, T, r.ratios,
                     K, r.start_seconds, r.sample_rate, lengths.data()));
  p->sub_off.assign(J + 1, 0);
  for (size_t j = 0; j < J; ++j) p->sub_off[j + 1] = p->sub_off[j] + lengths[j];
  if (p->gss) {   // the cue times checked at the interval's upper end as well
    const double r_hi = B2_GSS_HI;
    char what[32];
    snprintf(what, sizeof(what), "at ratio %g: ", r_hi);
    std::vector<int64_t> len_hi(T);
    B2_TRY(cue_lengths(&p->err, who, what, nullptr, r.cue_start_s, r.cue_end_s, r.cue_off, T,
                       &r_hi, 1, r.start_seconds, r.sample_rate, len_hi.data()));
    p->max_end.assign(T, 0.0);
    for (int t = 0; t < T; ++t)
      for (int64_t c = r.cue_off[t]; c < r.cue_off[t + 1]; ++c)
        p->max_end[t] = c == r.cue_off[t] ? r.cue_end_s[c] : std::max(p->max_end[t], r.cue_end_s[c]);
  }
  plan_cuts(r, env, p);
  plan_ref_format(r, env, p);
  return B2_OK;
}
