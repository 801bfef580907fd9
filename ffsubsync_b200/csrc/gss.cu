// K8g: golden-section search over the framerate ratio inside b2_sync_tracks_gss, one lane per track,
// every round driven on the device (DESIGN.md section 4 "K8g").  MaxScoreAligner.fit_gss
// (ffsubsync/aligners.py:111-129) + golden_section_search.gss (ffsubsync/golden_section_search.py:15-74),
// and the candidate's place in MaxScoreAligner.transform (aligners.py:154-167).
//
// gss_step_kernel turns the previous round's exact score into the next point and the run-path job that
// evaluates it; the evaluation itself is the run path of runcorr.cu, unchanged.  b2i_gss_launch
// (runcorr.cu) queues the rounds.
#include <math.h>

#include "common.cuh"
#include "corr_jobs.cuh"
#include "job_plan.cuh"

namespace {

__global__ void __launch_bounds__(128) gss_step_kernel(int r, int T, const GssTrack* __restrict__ trk,
                                                        B2GssLane* __restrict__ lane,
                                                        const double* __restrict__ prev_score,
                                                        SelJob* __restrict__ sel, double* __restrict__ xs,
                                                        long long* __restrict__ lens, double* __restrict__ evals,
                                                        long long max_offset_samples, uint64_t quirk_mask,
                                                        int sample_rate) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const GssTrack g = trk[t];
  SelJob s;
  memset(&s, 0, sizeof(s));
  s.ref_off = g.ref_off;
  s.R = g.R;
  s.out_index = t;
  s.bits_off = g.bits_off;
  s.n_tiles = 1;
  s.n_split = 1;
  s.m_hi = -1;
  if (g.R == 0) {  // empty reference: nothing is evaluated (pick_kernel reports B2_ALIGN_EMPTY)
    s.kind = 1;
    sel[t] = s;
    xs[t] = 1.0;   // a ratio the rasteriser can read; the length 0 leaves the mask empty
    lens[t] = 0;
    if (evals) evals[(size_t)t * kGssEvals + r] = __longlong_as_double(0x7ff8000000000000LL);
    return;
  }
  B2GssLane L = lane[t];
  // the objective of the reference's search is -score (aligners.py:116)
  const double x = b2_gss_step(L, r, r > 0 ? -prev_score[t] : 0.0, B2_GSS_LO, B2_GSS_HI);
  lane[t] = L;
  const long long S = b2_signal_length(g.max_end, x, sample_rate);
  const B2JobPlan p = b2_plan_job(g.R, S, max_offset_samples, quirk_mask);
  s.S = (int)S;
  s.kind = p.kind;
  s.masked_offset = p.masked_offset;
  s.sub_level = (float)fmin(__ddiv_rn(1.0, x), 1.0);  // speech_transformers.py:977
  // the run path's own window (what b2i_align_runs makes of the planner's absolute offsets); no_prune stays 0:
  // a round has one job per track and is finalised without winner-only pruning
  if (p.kind == 0) {
    s.o_first = (int)p.o_lo;
    s.m_lo = 0;
    s.m_hi = (int)(p.o_hi - p.o_lo);
  }
  sel[t] = s;
  xs[t] = x;
  lens[t] = S;
  if (evals) evals[(size_t)t * kGssEvals + r] = x;
}

__global__ void __launch_bounds__(128) gss_combine_kernel(int T, int K, const GssTrack* __restrict__ trk,
                                                           const double* __restrict__ xs,
                                                           const double* __restrict__ r_score,
                                                           const int32_t* __restrict__ r_offset,
                                                           long long max_off, B2GssOut out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const bool live = trk[t].R > 0;
  const double gs = r_score[t];
  const int go = r_offset[t];
  int bk = out.bk[t];
  if (live && (max_off == B2_MAX_OFFSET_NONE || llabs((long long)go) <= max_off) && (bk < 0 || gs > out.bs[t])) {
    out.bs[t] = gs;  // strictly greater: on a tie the grid ratio, earlier in list order, keeps its place
    out.bo[t] = go;
    out.bk[t] = K;
  }
  out.gss_ratio[t] = live ? xs[t] : __longlong_as_double(0x7ff8000000000000LL);
  const size_t a = (size_t)t * (K + 1);
  for (int k = 0; k < K; ++k) {
    if (out.a_score) out.a_score[a + k] = out.g_score[(size_t)t * K + k];
    if (out.a_offset) out.a_offset[a + k] = out.g_offset[(size_t)t * K + k];
  }
  if (out.a_score) out.a_score[a + K] = gs;
  if (out.a_offset) out.a_offset[a + K] = go;
}

}  // namespace

int b2i_gss_step_launch(b2_ctx* h, int r, int T, const GssTrack* d_trk, B2GssLane* d_lane, const double* prev_score,
                        SelJob* d_sel, double* d_x, long long* d_len, double* evals, long long max_offset_samples,
                        int sample_rate) {
  gss_step_kernel<<<(unsigned)((T + 127) / 128), 128, 0, h->stream>>>(r, T, d_trk, d_lane, prev_score, d_sel, d_x,
                                                                      d_len, evals, max_offset_samples,
                                                                      h->log2_quirk_mask, sample_rate);
  B2_CHECK_LAUNCH(h, "gss_step_kernel");
  return B2_OK;
}

int b2i_gss_combine_launch(b2_ctx* h, int T, int K, const GssTrack* d_trk, const double* d_x, const double* r_score,
                           const int32_t* r_offset, long long max_offset_samples, const B2GssOut& out) {
  gss_combine_kernel<<<(unsigned)((T + 127) / 128), 128, 0, h->stream>>>(T, K, d_trk, d_x, r_score, r_offset,
                                                                         max_offset_samples, out);
  B2_CHECK_LAUNCH(h, "gss_combine_kernel");
  return B2_OK;
}
