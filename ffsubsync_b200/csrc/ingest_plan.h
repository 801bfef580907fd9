// Host-side span planner of the batched ingest session (b2_ingest_*, DESIGN.md section 4 "K1i").  Video v's PCM
// arrives as pushes of any byte count; the planner cuts its stream into spans the detector can run on as they come:
// every span starts on a window boundary and ends on one, or at the end of a detector call (auditok's chunk of
// chunk_samples), so the windows of a span are exactly the windows the one-shot detector has over the same samples.
// The samples of an unfinished window (and an odd trailing byte) are held back until the next push of that video or
// until finish().  No CUDA call happens here, so tests/host_emul/ingest_emul.cu runs the same code on the CPU.
#pragma once

#include <stdint.h>

#include <algorithm>
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

  void begin(int V, int fpw_, bool auditok_, int64_t chunk_samples, double db) {
    fpw = fpw_;
    auditok = auditok_;
    chunk = auditok_ ? chunk_samples : 0;
    energy_threshold_db = db;
    bytes.assign(V, 0);
    base.assign(V, 0);
    frames.assign(V, 0);
    done.assign(V, 0);
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
