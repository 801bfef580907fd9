// Types and constants shared by the two correlation paths (corr.cu: overlap-save windows;
// bigfft.cu: one large FFT per signal) and their common tail (candidate selection, exact re-score,
// pick).
#pragma once
#include <stdint.h>

constexpr int kCandMax = 32;
constexpr int kRescoreSeg = 16;
// Nomination threshold tau (DESIGN.md section 4, "Round-off bound"): every offset whose fp32 score
// is within tau of the fp32 maximum is re-scored exactly, with
//     tau = u * (kTauFwd * sqrt(Es*Er) + (kTauInv + n_split - 1) * ||c||_2),   u = 2^-24,
// a first-order WORST-CASE bound on |fp32 score - exact score| (all rounding errors aligned):
//   kTauFwd: both forward transforms (first pass 95u: the twiddle w^k of the depth-4 product chain
//            carries k <= 15 times the 5.7u error of the two-table base twiddle; passes 2-4
//            32u + 22u + 3u; untangle 16u) = 2 x 168u, spectral product 3u, accumulation over
//            <= 64 blocks in fp32 <= 63u (more blocks: see window_max_kernel), retangle 16u -> <= 418u,
//            rounded up to 512 for the second-order terms;
//   kTauInv: the inverse transform is backward stable in the 2-norm, |error[m]| <= eps_inv*||c||_2
//            with eps_inv = 16u + 3u + 22u + 32u + 95u = 168u -> 192; ||c||_2 is the norm of the
//            tile's whole inverse-transform output, computed by the kernel (it exceeds sqrt(Es*Er)
//            only for signals with a large mean, whose correlation is a broad ramp);
//   n_split - 1: fp32 addition of the partial score arrays of a split job.
// Measured on random, constant, periodic, sparse and wide-dynamic-range inputs the error stays
// below tau / 400 (at most 26 u sqrt(Es*Er), tests/test_host_cpu.py::test_roundoff_bound_*); the slack
// costs nothing on real data, where the runner-up is thousands of units below the peak.
constexpr float kU = 5.9604645e-8f;
constexpr float kTauFwd = 512.0f;
constexpr float kTauInv = 192.0f;
constexpr int kTauBlocks = 64;  // block count covered by kTauFwd

// The bound above for one score array: fwd = kTauFwd (plus one per block beyond kTauBlocks),
// sqrt_e = sqrt(Es*Er), inv = kTauInv + n_split - 1, cn = ||c||_2.
__device__ __forceinline__ float tau_bound(float fwd, float sqrt_e, float inv, float cn) {
  return kU * (fwd * sqrt_e + inv * cn);
}
// The tau a job nominates with (job_stat.y): the largest tau_bound of its score arrays, padded so that
// the bound's own fp32 evaluation cannot cut off a candidate, and kept above 0.
__device__ __forceinline__ float nomination_tau(float tau) { return tau * 1.0001f + 1e-30f; }

// Offsets per chunk of the candidate selection: counting splits a window into chunks of m, the ordered
// compaction walks only the chunks that hold candidates.
constexpr int kChunk = 4096;

struct SelJob {        // one (pair, ratio)
  long long ref_off, sub_off, score_off;
  int R, S, o_first;   // offset of scores[score_off]
  int m_lo, m_hi;      // valid window of m (inclusive); m_lo > m_hi: nothing survives
  int energy_slot, n_tiles;
  int n_split;         // partial score arrays per tile (small batches split the block range over CTAs)
  int out_index;       // b*K + k
  int kind;            // 0 normal, 1 empty input, 2 everything masked
  int masked_offset;   // offset reported when kind == 2
  int no_prune;        // 1: some surviving offset of this pair exceeds max_offset_samples in magnitude (the
                       // negative-slice corners of aligners.py:31-43), so MaxScoreAligner.transform's
                       // |offset| filter (:160) may drop a ratio's winner - winner-only pruning is off
  long long bits_off;  // >= 0: the subtitle signal is a bit mask (one bit per frame)
  float sub_level;     // value of a frame inside a cue, min(1/ratio, 1) as float32 (bit-mask mode)
};


// The large-window path takes over from kBigMinTiles overlap-save tiles on; padded lengths it handles.
constexpr int kBigMinTiles = 4;
constexpr int kBigMinLog2n = 17, kBigMaxLog2n = 23;

// Common tail (corr.cu): candidate selection, exact float64 re-score of the nominated candidates and
// the argmax.  job_stat is filled by either path (window_max_kernel, big_stat_kernel); cand_off /
// cand_cnt / work_list / work_count by the selection.
struct B2CandBuffers {
  double* cand_partial;
  float2* job_stat;
  int* cand_off;
  int* cand_cnt;
  int* work_list;
  int* work_count;
};
// Candidates of n jobs: every offset whose fp32 score is within tau of the job's fp32 maximum, largest
// offset first, at most kCandMax, appended to the re-score work list.  Jobs d_jlist[0..n) (NULL:
// 0..n-1); a job's score array covers m < n_chunks * kChunk; chunk_cnt holds n * n_chunks ints.
// winner_only: a ratio that cannot be its pair's best keeps only its fp32 argmax (B2_ALIGN_APPROX).
int b2i_select_launch(b2_ctx* h, const SelJob* d_sel, const int* d_jlist, int n, const float* scores,
                      int n_chunks, int K, int winner_only, int* chunk_cnt, const B2CandBuffers& cb);
// ref_packed: d_ref holds each reference's bits m = (r == 1.0f) as words from its ref_off on (the detector's
// packed output, run-path chains only); the re-score reads r = m ? 1.0f : ref_label.
int b2i_rescore_pick(b2_ctx* h, const SelJob* d_sel, size_t J, const float* d_ref, const float* d_sub,
                     const uint32_t* d_bits, const B2CandBuffers& cb, double* d_score, int32_t* d_offset,
                     int32_t* d_status, bool ref_packed = false, float ref_label = 0.0f);
// b2_capture_nominations (corr.cu): copies the window scores, job_stat and cand_cnt of n jobs into
// h->capture at global index j0 + j, after the selection kernels.  Jobs d_jlist[0..n) (NULL: 0..n-1);
// with scores == NULL only the jobs without a live window are written, unless scores_written (the run
// path, whose kernel writes the scores itself): then every job's win / stat / cand are written.
int b2i_capture_launch(b2_ctx* h, const SelJob* d_sel, const int* d_jlist, int n, const float* scores,
                       const B2CandBuffers& cb, long long j0, bool scores_written = false);
// Run path (runcorr.cu): cue mode with a two-level reference (1.0f / ref_label).  sel: host copy of the jobs
// as the planner left them (absolute offsets in m_lo / m_hi; this call rebases them on each job's own window),
// subtitle bit masks in d_bits, at most max_runs cue runs per job.  Fills cand_off / cand_cnt / job_stat /
// work_list / work_count like the selection; the caller then runs b2i_rescore_pick on *d_sel_out.  Under a
// capture the float64 scores (rounded to float32), job_stat and cand_cnt go to it at global index capture_j0 + j.
// ref_packed: d_ref holds packed reference bits (see b2i_rescore_pick), which a scan turns into the run path's
// reference table; otherwise ref_bits_kernel packs the float reference.
int b2i_align_runs(b2_ctx* h, const float* d_ref, const int64_t* ref_off, int V, const int* trk_off, int K,
                   std::vector<SelJob>& sel, const uint32_t* d_bits, int max_runs, float ref_label, int winner_only,
                   bool ref_packed, const B2CandBuffers& cb, const SelJob** d_sel_out, long long capture_j0);
// The run path is chosen per call when every live job has cues x window <= kRunCostPerBlock x (its FFT block
// transforms): the break-even measured in the bench step on an H100 (DESIGN.md section 4, "K4r").
// kRunMaxCues bounds the shared memory of a job's run table (3 ints per run).
constexpr double kRunCostPerBlock = 5.6e5;
constexpr int kRunMaxCues = 16384;
constexpr int kRunMaxWindow = 32 * 1024;  // 32 offsets per thread, 1024 threads
// GSS rounds (gss.cu kernels, driven by b2i_gss_launch in runcorr.cu).  One lane per track of the chain.
struct GssTrack {
  long long ref_off;   // element offset of its video's reference signal
  long long bits_off;  // word offset of its mask (capacity planned at the interval's upper end)
  double max_end;      // largest unscaled cue end, 0 without cues
  int R;               // reference length
};
struct B2GssLane;
// Round r: consumes the exact score of round r - 1 (prev_score[t]), writes the job of round r (sel[t], a
// run-path job with its own window), its ratio x[t] and length len[t], and evals[t * kGssEvals + r].
int b2i_gss_step_launch(b2_ctx* h, int r, int T, const GssTrack* d_trk, B2GssLane* d_lane, const double* prev_score,
                        SelJob* d_sel, double* d_x, long long* d_len, double* evals, long long max_offset_samples,
                        int sample_rate);
// After the last round: the GSS candidate (x, score, offset, status of the last round) against the grid's
// reduced result under MaxScoreAligner.transform's rule, candidate K last in list order.
int b2i_gss_combine_launch(b2_ctx* h, int T, int K, const GssTrack* d_trk, const double* d_x, const double* r_score,
                           const int32_t* r_offset, long long max_offset_samples, const B2GssOut& out);
// Large-window path (bigfft.cu).  sel: host copy of the jobs (kind / R / S / offsets filled in by the
// planner; this call sets o_first, m_lo, m_hi, score_off), surviving index range per job in idx_lo /
// idx_hi (half open, in the reference's conv[] index space), padded lengths n_pad per job.  Reference v
// is read by the K ratio jobs of each of its tracks trk_off[v] .. trk_off[v+1]-1.
int b2i_align_big(b2_ctx* h, const float* d_ref, const float* d_sub, const uint32_t* d_bits, int V,
                  const int* trk_off, int K, std::vector<SelJob>& sel, const std::vector<long long>& idx_lo,
                  const std::vector<long long>& idx_hi, const std::vector<long long>& n_pad, int winner_only,
                  const B2CandBuffers& cb, const SelJob** d_sel_out, long long capture_j0);
