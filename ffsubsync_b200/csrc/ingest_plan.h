// Host-side span planner of the batched ingest session (b2_ingest_*, DESIGN.md section 4 "K1i").  A stream's PCM (an
// audio video's, or one sampled segment's; IngestStreams below numbers them, and the planner's `video` index is that
// stream number) arrives as pushes of any byte count; the planner cuts it into spans the detector can run on as they come:
// every span starts on a window boundary and ends on one, or at the end of a detector call (auditok's chunk of
// chunk_samples, energy / ZCR's energy_call_samples), so the windows of a span are exactly the windows the one-shot detector has over the same samples.
// The samples of an unfinished window (and an odd trailing byte) are held back until the next push of that stream or
// until finish().  No CUDA call happens here, so tests/host_emul/ingest_emul.cu runs the same code on the CPU.
#pragma once

#include <stdint.h>

#include <algorithm>
#include <string>
#include <vector>

#include "sync_plan.h"   // auditok_energy_floor

// Samples [s0, s1) of one video's stream, written to its reference frames from `frame` on: ceil((s1 - s0) / fpw)
// of them.  tail: auditok's energy floor of a short last block (0: none; energy / ZCR: always 0, a partial last
// window is non-speech).
struct IngestSpan {
  int video;
  int64_t s0, s1, frame, tail;
};

// A detector call the spans so far completed: the tokenizer runs over the video's frames [f0, f1).
struct IngestChunk {
  int video;
  int64_t f0, f1;
};

struct IngestPlanner {
  int fpw = 0;
  bool auditok = false;
  int64_t chunk = 0;             // samples per detector call; 0: one call per video
  double energy_threshold_db = 0.0;
  // per video
  std::vector<int64_t> bytes;    // bytes pushed so far
  std::vector<int64_t> base;     // first sample not yet in a span (a window boundary)
  std::vector<int64_t> frames;   // frames the spans so far write
  std::vector<uint8_t> done;     // finish() ran

  // chunk_samples: samples per detector call (SyncPlan::call: auditok's chunk_samples, or energy / ZCR's
  // energy_call_samples, 0 where its calls divide into windows)
  void begin(int V, int fpw_, bool auditok_, int64_t chunk_samples, double db) {
    fpw = fpw_;
    auditok = auditok_;
    chunk = chunk_samples;
    energy_threshold_db = db;
    bytes.assign(V, 0);
    base.assign(V, 0);
    frames.assign(V, 0);
    done.assign(V, 0);
  }

  // n more streams, empty, numbered after the existing ones
  void add_streams(int n) {
    bytes.resize(bytes.size() + n, 0);
    base.resize(base.size() + n, 0);
    frames.resize(frames.size() + n, 0);
    done.resize(done.size() + n, 0);
  }

  // frames of one detector call of n samples, and the calls' geometry
  int64_t per_chunk() const { return (chunk + fpw - 1) / fpw; }
  // the frames the one-shot detector gives a video of n samples: the sum over its calls of ceil(len / fpw)
  int64_t length(int64_t n) const {
    if (chunk <= 0) return (n + fpw - 1) / fpw;
    return n / chunk * per_chunk() + (n % chunk + fpw - 1) / fpw;
  }

  // Cuts samples [base, end) of video v: whole windows of each detector call, and a call's ragged last block once
  // the call is complete (or `final`).  Spans never cross a call boundary.
  void cut(int v, int64_t end, bool final, std::vector<IngestSpan>* spans, std::vector<IngestChunk>* chunks) {
    int64_t s = base[v];
    while (s < end) {
      const int64_t k = chunk > 0 ? s / chunk : 0;
      const int64_t c0 = k * chunk, c1 = chunk > 0 ? c0 + chunk : INT64_MAX;
      const int64_t lim = std::min(end, c1);
      int64_t e = c0 + (lim - c0) / fpw * fpw;
      const bool closes = lim == c1 || final;   // the call's last block is known
      if (closes) e = lim;
      if (e <= s) break;
      const int64_t rem = (e - c0) % fpw;
      const int64_t f = k * per_chunk() + (s - c0) / fpw;
      const int64_t nf = (e - s + fpw - 1) / fpw;
      spans->push_back(IngestSpan{v, s, e, f, auditok && rem && closes ? auditok_energy_floor((int)rem,
                                                                                             energy_threshold_db) : 0});
      frames[v] = f + nf;
      if (auditok && lim == c1) chunks->push_back(IngestChunk{v, k * per_chunk(), f + nf});
      s = e;
      if (lim != c1) break;
    }
    base[v] = s;
  }

  // Video v's stream grew by nb bytes: the spans this fixes, and the detector calls it completed
  void push(int v, int64_t nb, std::vector<IngestSpan>* spans, std::vector<IngestChunk>* chunks) {
    bytes[v] += nb;
    cut(v, bytes[v] / 2, false, spans, chunks);
  }

  // End of video v's stream: its held-back samples as the final span, and its last detector call for auditok
  void finish(int v, std::vector<IngestSpan>* spans, std::vector<IngestChunk>* chunks) {
    const int64_t n = bytes[v] / 2;
    cut(v, n, true, spans, chunks);
    done[v] = 1;
    if (!auditok) return;
    const int64_t k0 = chunk > 0 ? n / chunk * per_chunk() : 0;   // the call in progress (chunk: empty when n ends one)
    if (frames[v] > k0) chunks->push_back(IngestChunk{v, k0, frames[v]});
  }
};

// The streams of a session and where each push goes.  Stream v < V is video v's own; b2_ingest_segments gives each
// sampled segment a stream of its own: segment j (counted within its video) of the i-th segment video is stream
// V + first[i] + j, so that energy / ZCR restarts its windows and auditok its chunk loop at each segment's first
// sample, as the whole-call segment path's detector items do.  A segment video's own stream takes no pushes, an audio
// video has no segment streams, and a dropped segment's stream takes none from the drop on.  The refusals leave
// everything as it was.
struct IngestStreams {
  std::string err;
  int V = 0;
  bool declared = false;
  std::vector<uint8_t> touched;   // [V]: a push named video v
  std::vector<int> seg_of;        // [V]: v's index among the segment videos, -1: an audio video
  std::vector<int32_t> video;     // [P] the segment videos, increasing
  std::vector<double> total;      // [P] their probed durations (seconds)
  std::vector<int64_t> first;     // [P+1] their segments
  std::vector<int64_t> start;     // per segment: its whole-second start
  std::vector<uint8_t> dropped;   // per segment

  void begin(int V_) {
    V = V_;
    declared = false;
    touched.assign(V, 0);
    seg_of.assign(V, -1);
    video.clear();
    total.clear();
    first.assign(1, 0);
    start.clear();
    dropped.clear();
  }

  int streams() const { return V + (int)start.size(); }
  // the stream takes pushes (an audio video, or a segment not dropped)
  bool live(int k) const { return k < V ? seg_of[k] < 0 : !dropped[k - V]; }

  // b2_ingest_segments: the table's checks are b2_sync_tracks_seg's (plan_seg_check on `det`, the session's detector
  // arguments, with empty PCM ranges and empty sample ranges), then those of the session.
  int declare(const SyncRequest& det, int P, const int32_t* vid, const double* tot, const int64_t* off,
              const int64_t* st) {
    const char* who = "ingest_segments";
    if (declared) B2_FAIL(this, B2_ERR_BAD_ARG, "%s: the session's segments are already declared", who);
    if (P < 0 || (P > 0 && (!vid || !tot || !off))) B2_FAIL(this, B2_ERR_BAD_ARG, "%s: bad segment videos (%d)", who, P);
    const int64_t S = P > 0 ? off[P] - off[0] : 0;
    std::vector<int64_t> pcm_off(V + 1, 0), no_range(S > 0 ? S : 1, 0);
    SyncRequest r = det;
    r.who = who;
    r.V = V;
    r.pcm_off = pcm_off.data();
    const int64_t* st_rel = P > 0 && st ? st + off[0] : st;
    r.seg = {P, vid, tot, off, P > 0 && st ? st : nullptr, no_range.data() - (P > 0 ? off[0] : 0),
             no_range.data() - (P > 0 ? off[0] : 0)};
    SyncPlan p;
    if (const int e = plan_seg_check(r, &p)) {
      err = p.err;
      return e;
    }
    for (int i = 0; i < P; ++i)
      if (touched[vid[i]])
        B2_FAIL(this, B2_ERR_BAD_ARG, "%s: video %d already has pushes; declare its segments before its first push",
                who, (int)vid[i]);
    declared = true;
    for (int i = 0; i < P; ++i) {
      seg_of[vid[i]] = i;
      video.push_back(vid[i]);
      total.push_back(tot[i]);
      first.push_back(off[i + 1] - off[0]);
    }
    start.assign(st_rel, st_rel + S);
    dropped.assign(S, 0);
    return B2_OK;
  }

  // The frames video v's stream fixed so far, or for a segment video its live segments' streams together
  int64_t windows(const IngestPlanner& pl, int v) const {
    int64_t n = pl.frames[v];
    const int q = seg_of[v];
    for (int64_t j = q < 0 ? 0 : first[q]; q >= 0 && j < first[q + 1]; ++j)
      if (!dropped[j]) n += pl.frames[V + j];
    return n;
  }

  // The stream of chunk i: video v's own (b2_ingest_push), or with `segmented` its segment seg
  // (b2_ingest_push_segments); -1 with err set when the chunk is refused.
  int route(const char* who, int i, int v, bool segmented, int64_t seg) {
    if (segmented) return segment(who, i, v, seg);
    if (v < 0 || v >= V) {
      snprintf(buf_, sizeof(buf_), "%s: chunk %d: video %d is out of [0, %d)", who, i, v, V);
    } else if (seg_of[v] >= 0) {
      snprintf(buf_, sizeof(buf_), "%s: chunk %d: video %d has sampled segments; push them with "
               "b2_ingest_push_segments", who, i, v);
    } else {
      return v;
    }
    err = buf_;
    return -1;
  }

  // The stream of segment seg of video v (i >= 0: names chunk i; b2_ingest_drop_segment passes -1), -1 with err set
  int segment(const char* who, int i, int v, int64_t seg) {
    char at[32] = "";
    if (i >= 0) snprintf(at, sizeof(at), " chunk %d:", i);
    if (v < 0 || v >= V) {
      snprintf(buf_, sizeof(buf_), "%s:%s video %d is out of [0, %d)", who, at, v, V);
    } else if (seg_of[v] < 0) {
      snprintf(buf_, sizeof(buf_), "%s:%s video %d has no sampled segments", who, at, v);
    } else {
      const int q = seg_of[v];
      const int64_t n = first[q + 1] - first[q];
      if (seg < 0 || seg >= n) {
        snprintf(buf_, sizeof(buf_), "%s:%s segment %lld of video %d is out of [0, %lld)", who, at, (long long)seg, v,
                 (long long)n);
      } else if (i >= 0 && dropped[first[q] + seg]) {
        snprintf(buf_, sizeof(buf_), "%s:%s segment %lld of video %d was dropped", who, at, (long long)seg, v);
      } else {
        return V + (int)(first[q] + seg);
      }
    }
    err = buf_;
    return -1;
  }

 private:
  char buf_[256];
};

// b2_ingest_sync_refs: a video given a text, PGS or signal reference (r.refs / r.pgs / r.sig, read as plan_refs_check
// reads them) has no audio, so its stream must have taken no bytes; plan_refs_check cannot tell, since a session's
// pcm_off is all zeros.  B2_ERR_BAD_ARG with st->err naming the first such video.
static int ingest_refs_check(const SyncRequest& r, IngestStreams* st, const IngestPlanner& pl) {
  for (int v = 0; v < r.V; ++v) {
    const bool is_subs = r.refs.cue_off && r.refs.is_subs && r.refs.is_subs[v];
    const bool is_pgs = r.pgs.off && r.pgs.is_pgs && r.pgs.is_pgs[v];
    const bool is_sig = r.sig.off && r.sig.is_sig && r.sig.is_sig[v];
    if ((is_subs || is_pgs || is_sig) && pl.bytes[v] > 0)
      B2_FAIL(st, B2_ERR_BAD_ARG, "%s: video %d has a %s reference and received %lld pushed bytes; its audio is never "
              "read, so it takes no pushes", r.who, v, is_sig ? "serialized signal" : is_pgs ? "PGS" : "text subtitle",
              (long long)pl.bytes[v]);
  }
  return B2_OK;
}
