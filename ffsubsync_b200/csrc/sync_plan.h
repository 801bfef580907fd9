// Host-side plan of one batched sync call (b2_sync_batch, b2_sync_tracks, b2_sync_tracks_gss,
// b2_sync_tracks_auditok, b2_sync_tracks_subs): every argument check and every host table the pipeline in
// api.cu reads.  No CUDA call happens here, so tests/host_emul/plan_emul.cu runs the same code on the CPU.
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

// ---- detectors --------------------------------------------------------------------------------
static inline int vad_frames_per_window(int frame_rate, int sample_rate) {
  if (frame_rate <= 0 || sample_rate <= 0) return 0;
  // speech_transformers.py:163-164: int(window_duration * frame_rate + 0.5)
  return (int)((1.0 / (double)sample_rate) * (double)frame_rate + 0.5);
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
// With subs_len (b2_sync_tracks_subs), a video with subs_len[v] >= 0 has a subtitle reference and no PCM: it is
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
};

struct SyncPlan {
  std::string err;
  bool gss = false, auditok = false, any_subs = false;
  int fpw = 0, z_lo = 0, z_hi = 0;
  // the reference's levels (B2CueSource::ref_label / ref_two_level)
  float label = 0.0f, ref_label = 0.0f;
  bool two_level = false;
  int64_t audio_samples = 0;       // samples the detector reads
  std::vector<int> trk_off;        // [V+1]: first track of video v
  std::vector<int64_t> ref_off;    // [V+1]: reference signal of video v
  std::vector<int64_t> sub_off;    // [T*K+1]: float subtitle signal of job j (unfused raster)
  std::vector<int> sub_video;      // the videos with a subtitle reference, ascending
  ChunkTable ch;                   // auditok
  int64_t auditok_e_min = 0;
  B2TokenizerParams tok{0.0, 0.0, 0.0, 0};
  std::vector<double> max_end;     // GSS: each track's largest cue end (its signal length at any ratio)
  // Sub-batches of the pipeline: videos cut[i] .. cut[i+1]-1; the later ones' detector runs on vad_sms SMs
  int n_sub = 1, vad_sms = 0;
  std::vector<int> cut;
  // per sub-batch: its detector writes the reference as packed bits instead of floats (plan_ref_format)
  std::vector<uint8_t> ref_packed;
};

// Sub-batches are cut at video boundaries (a video's tracks run in the chain behind its own VAD) and balanced by
// track count, since the chain's work scales with tracks: cut i is the first video whose tracks start at or
// after track T*i/n_sub.  With one track per video these are T*i/n_sub exactly.  Cuts that would leave a
// sub-batch without tracks are dropped; a video without tracks has its VAD run in the sub-batch of the next video
// that has tracks (trailing ones: of the last).  Where the cuts fall changes no result.
// Defaults: 3 sub-batches, the later VADs on 54 % of the SMs (71 of an H100's 132; tools/pipeline_probe.py sweeps
// both), on the lane-per-window kernel only; small batches stay unpipelined (the alignment of a third of a small
// batch is launch- and tail-bound).  B2_SUBBATCHES / B2_VAD_SMS override the defaults; 1 / 0 = off.
static void plan_cuts(const SyncRequest& r, const SyncPipeEnv& env, SyncPlan* p) {
  const int V = r.V, T = r.T;
  // lane eligibility is decided on the tables the energy kernel reads: the videos, or auditok's chunks
  const bool lane_ok = p->auditok ? env.lane_eligible(p->ch.pcm.data(), (int)p->ch.tail.size(), p->fpw)
                                  : env.lane_eligible(r.pcm_off, V, p->fpw);
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
// them), so the launcher reaches the same choice.  auditok, subtitle references, the lane-group kernel and the
// FFT paths keep the float reference.  B2_REF_PACKED=0 keeps it everywhere (A/B knob).
static void plan_ref_format(const SyncRequest& r, const SyncPipeEnv& env, SyncPlan* p) {
  p->ref_packed.assign(p->n_sub, 0);
  if (p->auditok || !env.fused || (env.ref_packed && atoi(env.ref_packed) == 0)) return;
  for (int i = 0; i < p->n_sub; ++i) {
    const int v0 = p->cut[i], v1 = p->cut[i + 1];
    const auto& sv = p->sub_video;
    if (std::lower_bound(sv.begin(), sv.end(), v0) != std::lower_bound(sv.begin(), sv.end(), v1)) continue;
    if (!env.lane_eligible(r.pcm_off + v0, v1 - v0, p->fpw)) continue;
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

// Checks of the subtitle references, before anything reads their tables.
static int plan_refs_check(const SyncRequest& r, SyncPlan* p, bool* any_audio) {
  const char* who = r.who;
  const auto& s = r.refs;
  for (int v = 0; v < r.V; ++v) {
    const bool is_subs = s.is_subs && s.is_subs[v];
    if (s.cue_off[v + 1] < s.cue_off[v]) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: ref_cue_off not monotone at %d", who, v);
    if (!is_subs && s.cue_off[v + 1] != s.cue_off[v])
      B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has reference cues but no subtitle reference (ref_is_subs[%d] = 0)",
              who, v, v);
    if (is_subs && r.pcm_off[v + 1] != r.pcm_off[v])
      B2_FAIL(p, B2_ERR_BAD_ARG, "%s: video %d has a subtitle reference and a non-empty PCM range (%lld samples); "
              "its audio is never read", who, v, (long long)(r.pcm_off[v + 1] - r.pcm_off[v]));
    p->any_subs = p->any_subs || is_subs;
    *any_audio = *any_audio || !is_subs;
  }
  if (r.V > 0 && s.cue_off[r.V] > s.cue_off[0] && (!s.cue_start_s || !s.cue_end_s))
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: null reference cue arrays", who);
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
  } else {
    p->fpw = vad_frames_per_window(r.frame_rate, r.sample_rate);
  }
  const int fpw = p->fpw;
  if (fpw <= 0) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: bad frame_rate/sample_rate", who);
  p->z_lo = r.energy.z_lo < 0 ? 0 : r.energy.z_lo;
  p->z_hi = r.energy.z_hi < 0 ? (3 * fpw) / 8 : r.energy.z_hi;
  // subtitle references: int(max_end * sample_rate) + 2 frames (speech_transformers.py:958-962), the length
  // b2_rasterize gives at ratio 1.0; the lengths pass checks the cue times too (the same checks and messages as
  // the tracks' cues).  subs_len[v] = -1: the video's reference is the detector's.
  std::vector<int64_t> subs_len;
  if (p->any_subs) {
    const double one = 1.0;
    subs_len.resize(V);
    B2_TRY(cue_lengths(&p->err, who, "reference ", "bad reference cue list", r.refs.cue_start_s, r.refs.cue_end_s,
                       r.refs.cue_off, V, &one, 1, r.start_seconds, r.sample_rate, subs_len.data()));
    for (int v = 0; v < V; ++v) {
      if (r.refs.is_subs[v]) p->sub_video.push_back(v);
      else subs_len[v] = -1;
    }
  }
  p->ref_off.assign(V + 1, 0);
  for (int v = 0; v < V; ++v) {
    const int64_t n = r.pcm_off[v + 1] - r.pcm_off[v];
    if (n < 0) B2_FAIL(p, B2_ERR_BAD_ARG, "%s: pcm_off not monotone", who);
    if (p->any_subs && subs_len[v] >= 0) p->ref_off[v + 1] = p->ref_off[v] + subs_len[v];
    else if (!p->auditok) p->ref_off[v + 1] = p->ref_off[v] + (n + fpw - 1) / fpw;
  }
  if (p->auditok) {
    build_chunk_table(r.pcm_off, V, 0, fpw, r.auditok.chunk_samples, r.auditok.energy_threshold_db,
                      p->any_subs ? subs_len.data() : nullptr, &p->ch);
    for (int v = 0; v < V; ++v) p->ref_off[v + 1] = p->ch.out[p->ch.first[v + 1]];
  }
  return B2_OK;
}

// Every argument check and every host table of one batched sync call.  Errors go to p->err with the status.
// T == 0 returns B2_OK after the checks that do not need tracks, with no tables.
static int plan_sync(const SyncRequest& r, const SyncPipeEnv& env, SyncPlan* p) {
  const char* who = r.who;
  const int V = r.V, T = r.T, K = r.K;
  p->gss = r.search;
  p->auditok = r.detector == B2_DETECTOR_AUDITOK;
  if (V < 0 || T < 0 || K <= 0 || !r.pcm_off || !r.cue_off || !r.ratios)
    B2_FAIL(p, B2_ERR_BAD_ARG, "%s: bad arguments", who);
  bool any_audio = !r.refs.cue_off;
  for (int v = 0; v < V; ++v)
    if (r.pcm_off[v + 1] > r.pcm_off[v]) p->audio_samples += r.pcm_off[v + 1] - r.pcm_off[v];
  if (r.refs.cue_off) B2_TRY(plan_refs_check(r, p, &any_audio));
  // The run path and the GSS rounds need a reference of the two levels 1.0 and ref_label.  The detector's signal
  // has the levels 1.0 and the label, a subtitle reference 1.0 and 0.0, so ref_label is the label unless every
  // reference is a subtitle stream; a call that mixes the two at a non-zero label has three levels.  auditok's
  // clipped cumsum has two levels only at label 0 (starts and ends alternate and an overwrite only turns an end
  // into a start, so the integer sum stays in {0, 1}); other labels give further levels (0.3, 0.6, ... for 0.3).
  p->label = p->auditok ? (float)r.auditok.non_speech_label : r.energy.non_speech_label;
  p->ref_label = any_audio ? p->label : 0.0f;
  const bool auditok_two_level = !p->auditok || r.auditok.non_speech_label == 0.0;
  const bool mix_two_level = !p->any_subs || p->label == 0.0f;
  p->two_level = !any_audio || (auditok_two_level && mix_two_level);
  if (r.track_video) {
    for (int t = 0; t < T; ++t)
      if (r.track_video[t] < 0 || r.track_video[t] >= V || (t > 0 && r.track_video[t] < r.track_video[t - 1]))
        B2_FAIL(p, B2_ERR_BAD_ARG, "sync_tracks: track_video[%d] = %d is out of [0, %d) or decreases", t,
                (int)r.track_video[t], V);
    for (int t = 0; t < T; ++t)
      if (r.cue_off[t + 1] < r.cue_off[t]) B2_FAIL(p, B2_ERR_BAD_ARG, "sync_tracks: cue_off not monotone at %d", t);
  }
  if (p->gss) B2_TRY(plan_gss_check(r, p, auditok_two_level));
  if (T == 0) return B2_OK;
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
