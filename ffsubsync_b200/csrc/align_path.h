// The aligner's job plan and path choice for one correlation chain (b2i_align_launch), as host functions of the
// chain's shapes.  The batched sync calls' planner (sync_plan.h) runs the same two functions before any detector
// runs, so it knows which chains take the run path and may have their reference written as packed bits; the
// launcher runs them again when it aligns, so the two cannot disagree.  No CUDA call happens here
// (tests/host_emul/plan_emul.cu runs this code on the CPU).
#pragma once

#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"      // B2_FAIL, ceil_div64
#include "corr_jobs.cuh"   // SelJob, kBigMinTiles, kRun*
#include "job_plan.cuh"    // b2_plan_job

constexpr int kAlignBlock = 32768;   // real samples per overlap-save block transform (corr.cuh kP)

enum B2AlignPath { B2_PATH_TILED = 0, B2_PATH_BIG = 1, B2_PATH_RUNS = 2 };

// One plan per reference (video): its window covers the live jobs of all its tracks
struct B2AlignPairPlan {
  long long o_min, o_max;
  int n_tiles;
  bool any;
};

struct B2AlignJobs {
  std::string err;
  std::vector<SelJob> sel;                        // [B*K]; kind 0: m_lo / m_hi hold absolute offsets
  std::vector<long long> idx_lo, idx_hi, n_pad;   // surviving conv[] index range and padded length per job
  std::vector<long long> bits_off;                // cue mode: word offset of job j's mask, [B*K+1]
  std::vector<B2AlignPairPlan> pp;                // [V]
  long long max_w = 1;                            // widest window of a reference
  bool big_ok = true;                             // every live job's padded length suits the large-window path
  int Wt = 0, L = 0;                              // offsets per tile, subtitle samples per block
};

// The jobs t*K + k of the tracks trk_off[v] .. trk_off[v+1]-1 of every reference v (aligners.py:31-66 per job:
// empty input, padded length, surviving window), the windows per reference and the overlap-save tiling.
// cue_ratios (cue mode, the K ratios): the subtitle signals are bit masks, a frame inside a cue has the level
// min(1/ratio, 1).
static int b2_plan_align_jobs(const int64_t* ref_off, int V, const int* trk_off, const int64_t* sub_off, int B, int K,
                              int64_t max_offset_samples, uint64_t quirk_mask, const double* cue_ratios,
                              B2AlignJobs* a) {
  const size_t J = (size_t)B * K;
  const bool cue_mode = cue_ratios != nullptr;
  a->bits_off.assign(cue_mode ? J + 1 : 1, 0);
  if (cue_mode)
    for (size_t j = 0; j < J; ++j)
      a->bits_off[j + 1] = a->bits_off[j] + ((sub_off[j + 1] - sub_off[j]) + kAlignBlock) / 32 + 1;
  a->sel.assign(J, SelJob{});
  a->idx_lo.assign(J, 0);
  a->idx_hi.assign(J, 0);
  a->n_pad.assign(J, 0);
  a->pp.assign(V, B2AlignPairPlan{});
  a->max_w = 1;
  a->big_ok = true;
  const long long mo_clamped =
      std::max<long long>(-(1LL << 40), std::min<long long>(1LL << 40, max_offset_samples));
  for (int v = 0; v < V; ++v) {
    const long long R = ref_off[v + 1] - ref_off[v];
    if (R < 0 || R > 0x3fffffff) B2_FAIL(a, B2_ERR_BAD_ARG, "align: bad reference length at %d", v);
    B2AlignPairPlan& p = a->pp[v];
    p.any = false;
    p.o_min = 0;
    p.o_max = -1;
    for (int b = trk_off[v]; b < trk_off[v + 1]; ++b) {
      long long t_min = 0, t_max = -1;   // window of this track's K jobs (winner-only pruning is per track)
      bool t_any = false;
      for (int k = 0; k < K; ++k) {
        const size_t j = (size_t)b * K + k;
        const long long S = sub_off[j + 1] - sub_off[j];
        if (S < 0 || S > 0x3fffffff) B2_FAIL(a, B2_ERR_BAD_ARG, "align: bad subtitle length at %zu", j);
        SelJob& s = a->sel[j];
        memset(&s, 0, sizeof(s));
        s.ref_off = ref_off[v];
        s.sub_off = sub_off[j];
        s.R = (int)R;
        s.S = (int)S;
        s.out_index = (int)j;
        s.bits_off = cue_mode ? a->bits_off[j] : -1;
        s.sub_level = cue_mode ? (float)std::min(1.0 / cue_ratios[k], 1.0) : 0.f;  // speech_transformers.py:977
        const B2JobPlan jp = b2_plan_job(R, S, max_offset_samples, quirk_mask);
        if (jp.kind != 0) {
          s.kind = jp.kind;
          s.masked_offset = jp.masked_offset;
          continue;
        }
        const long long N = jp.N, o_lo = jp.o_lo, o_hi = jp.o_hi;
        a->idx_lo[j] = jp.lo;
        a->idx_hi[j] = jp.hi;
        a->n_pad[j] = N;
        if (N < (1LL << kBigMinLog2n) || N > (1LL << kBigMaxLog2n)) a->big_ok = false;
        s.kind = 0;
        s.m_lo = (int)o_lo;  // absolute offsets; each path rebases them
        s.m_hi = (int)o_hi;
        t_min = t_any ? std::min(t_min, o_lo) : o_lo;
        t_max = t_any ? std::max(t_max, o_hi) : o_hi;
        t_any = true;
      }
      if (!t_any) continue;
      p.o_min = p.any ? std::min(p.o_min, t_min) : t_min;
      p.o_max = p.any ? std::max(p.o_max, t_max) : t_max;
      p.any = true;
      if (max_offset_samples != B2_MAX_OFFSET_NONE && std::max(llabs(t_min), llabs(t_max)) > mo_clamped)
        for (int k = 0; k < K; ++k) a->sel[(size_t)b * K + k].no_prune = 1;
    }
    if (p.any) a->max_w = std::max(a->max_w, p.o_max - p.o_min + 1);
  }
  // offsets per tile: Wt = 1 (mod 32) so that L = P - Wt + 1 is a multiple of 32 (vector loads,
  // whole words of the speech bit mask per block), at most P/2 + 1
  a->Wt = (int)(a->max_w <= kAlignBlock / 2 + 1 ? 32 * ((a->max_w + 30) / 32) + 1 : (kAlignBlock / 2 + 1));
  a->L = kAlignBlock - a->Wt + 1;
  return B2_OK;
}

struct B2AlignPathChoice {
  int path;       // B2AlignPath
  int max_runs;   // run path: most cue runs of a job's mask
};

// Large windows (FFTAligner's default max_offset_samples=None, or a mask wider than a few tiles): the overlap-save
// path would recompute every block for every 16 385-offset tile; one padded-length FFT per signal (four-step,
// bigfft.cu) is cheaper from kBigMinTiles tiles on.  align_path: B2_ALIGN_PATH=tiled|big|runs (test / A-B knob).
// Cue mode (cue_off: the chain's tracks' cue list offsets, null otherwise) with the reference from this call's
// detector, two levels (1.0f and ref_label): the run path (runcorr.cu) scores every offset of the window from the
// cue runs, exactly up to a float64 margin, when its work (cues x window) is below the FFT blocks it replaces for
// every live job.  A capture of the nominations (b2_capture_nominations) probes the FFT paths and keeps them,
// unless B2_ALIGN_PATH=runs asks for the run path (then its float64 scores are captured).  A reference with
// further levels (auditok at a non-zero label) stays on the FFT paths, which read its values as they are, even
// under B2_ALIGN_PATH=runs.
static B2AlignPathChoice b2_align_path(const B2AlignJobs& a, const int* trk_off, int V, int K, const int64_t* cue_off,
                                       bool ref_two_level, float ref_label, const char* align_path, bool capture) {
  bool use_big = a.big_ok && a.max_w > (long long)kBigMinTiles * (kAlignBlock / 2 + 1);
  const bool force_runs = align_path && !strcmp(align_path, "runs");
  const bool force_tiled = align_path && !strcmp(align_path, "tiled");
  if (force_tiled || force_runs) use_big = false;
  if (align_path && !strcmp(align_path, "big") && a.big_ok) use_big = true;
  B2AlignPathChoice c{use_big ? B2_PATH_BIG : B2_PATH_TILED, 1};
  if (!cue_off || (capture && !force_runs) || use_big || !ref_two_level || !std::isfinite(ref_label) || force_tiled)
    return c;
  bool fits = true, pays = true;
  int max_runs = 1;
  for (int v = 0; v < V && fits; ++v) {
    const B2AlignPairPlan& p = a.pp[v];
    const long long n_tiles_v = p.any ? ceil_div64(p.o_max - p.o_min + 1, a.Wt) : 0;
    for (int b = trk_off[v]; b < trk_off[v + 1]; ++b) {
      const long long cues = cue_off[b + 1] - cue_off[b];  // runs of a mask <= its cues
      for (int k = 0; k < K; ++k) {
        const SelJob& s = a.sel[(size_t)b * K + k];
        if (s.kind != 0) continue;
        const long long w = (long long)s.m_hi - s.m_lo + 1;
        if (w > kRunMaxWindow || cues > kRunMaxCues || llabs((long long)s.m_lo) > (1LL << 30) ||
            llabs((long long)s.m_hi) > (1LL << 30))
          fits = false;
        if ((double)cues * (double)w > kRunCostPerBlock * (double)(n_tiles_v * (ceil_div64(s.S, a.L) + 1)))
          pays = false;
        max_runs = std::max<int>(max_runs, (int)std::min<long long>(cues, kRunMaxCues));
      }
    }
  }
  if (fits && (pays || force_runs)) c = B2AlignPathChoice{B2_PATH_RUNS, max_runs};
  return c;
}
