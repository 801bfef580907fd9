// V3: the auditok detector's tokenizer as a 100 Hz scan on the GPU.
//
// Replaces what _make_auditok_detector._detect does after the per-block energy test
// (ffsubsync/speech_transformers.py:126-150): auditok 0.1.5's StreamTokenizer(min_length,
// max_length, max_continuous_silence) state machine over the per-block validity flags, the
// start / end+1 impulses (ASSIGNED, not added, in token order - a token that follows a truncated one
// overwrites its predecessor's end impulse), numpy's sequential float64 cumsum and the clip to [0, 1].
// One detector call (= one chunk of the reference's chunk loop; the tokenizer restarts in every call,
// :142) is one warp:
//   pass 1  32 flags are read per step (coalesced) and packed with a ballot; every lane runs the
//           same state machine over the packed bits (uniform control flow), lane 0 writes the
//           impulses in token order as codes (+1 start, -1 end) into the output.  The machine takes
//           the runs that only move it forward - invalid frames in SILENCE, valid frames in NOISE - a
//           whole run per step (find-first-set on the packed bits), so a chunk costs about one step
//           per token edge, not one per frame,
//   pass 2  cumsum + clip: only the non-zero entries change the running sum, so each 32-wide step
//           walks its non-zero lanes in order with exact float64 adds of the decoded impulses (1.0 and
//           non_speech_label - 1.0, never rounded to the output type) - bit-identical to np.cumsum.  The
//           clipped float64 sum is rounded once to the output type.
// The output may be the flag array itself (b2_sync_tracks_auditok: the energy pass writes its 0/1 flags
// into the reference-signal buffer and the scan overwrites them with the signal).  Pass 1 therefore reads
// the flags one 32-block ahead of the machine and zeroes each block right after reading it: an impulse
// lands at most one frame past the frame being scanned (end + 1), i.e. in a block already read and zeroed,
// so no flag is overwritten before it is read and the chunk needs no staging copy of any size.
// The machine is restated from auditok's published algorithm in oracle/auditok_oracle.py (the
// wheel is absent from the image); tests compare the two bit for bit.
#include "common.cuh"

namespace {

template <typename Out>
struct TokParams {
  const float* flags;      // K1 output with label 0: non-zero = the block passed the energy test
  Out* out;                // may alias flags
  const long long* off;    // [n_chunks] first window of each chunk
  const long long* end;    // [n_chunks] one past its last window (off + 1 for abutting chunks)
  int n_chunks;
  double min_length, max_sil, down;  // down = non_speech_label - 1.0
  long long max_length;
};

enum { kSilence = 0, kNoise = 2, kPossibleSilence = 3 };

struct Machine {
  int state = kSilence, n = 0, sil = 0, start = 0, cur = 0;
  bool contig = false;
};

template <typename Out>
__device__ __forceinline__ void end_of_detection(Machine& m, const TokParams<Out>& p, Out* out, int n_out,
                                                 bool truncated, bool writer) {
  if ((double)m.n >= p.min_length || (m.n > 0 && m.contig)) {
    if (writer) {
      out[m.start] = Out(1);
      const int e1 = m.start + m.n;            // end + 1; index n_out is the slot [:-1] drops
      if (e1 < n_out) out[e1] = Out(-1);
    }
    if (truncated) m.start = m.cur + 1;
    m.contig = truncated;
  } else {
    m.contig = false;
  }
  m.n = 0;
}

template <typename Out>
__global__ void __launch_bounds__(128) auditok_tokenize_kernel(TokParams<Out> p) {
  const int chunk = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (chunk >= p.n_chunks) return;
  const long long base = p.off[chunk];
  const int n = (int)(p.end[chunk] - base);
  const float* f = p.flags + base;
  Out* out = p.out + base;

  Machine m;
  const bool writer = lane == 0;
  // block 0 read and zeroed up front; block i0 + 32 is read and zeroed before block i0 is scanned
  unsigned next = __ballot_sync(0xffffffffu, lane < n && f[lane] != 0.f);
  if (lane < n) out[lane] = Out(0);
  for (int i0 = 0; i0 < n; i0 += 32) {
    const unsigned mask = next;
    const int j = i0 + 32 + lane;
    next = __ballot_sync(0xffffffffu, j < n && f[j] != 0.f);
    if (j < n) out[j] = Out(0);
    __syncwarp();
    const int cnt = min(32, n - i0);
    for (int b = 0; b < cnt; ++b) {
      if (m.state == kSilence) {   // invalid frames change nothing in SILENCE: go to the next valid one
        const unsigned rest = mask >> b;
        if (!rest) break;
        b += __ffs(rest) - 1;
      }
      const bool ok = (mask >> b) & 1u;
      m.cur = i0 + b;
      if (m.state == kSilence) {
        if (ok) {  // init_min = 0: a single valid frame opens a token
          m.sil = 0;
          m.start = m.cur;
          m.n = 1;
          m.state = kNoise;
          if (m.n >= p.max_length) end_of_detection(m, p, out, n, true, writer);
        }
      } else if (m.state == kNoise) {
        if (ok) {
          // a run of valid frames in NOISE only counts n up (n < max_length holds here): take the run, up to
          // the frame where n reaches max_length, in one step.  Bits past cnt are 0, so run <= cnt - b.
          const unsigned inv = ~(mask >> b);
          const int run = inv ? __ffs(inv) - 1 : 32;
          const int steps = (int)min((long long)run, p.max_length - (long long)m.n);
          m.n += steps;
          b += steps - 1;
          m.cur = i0 + b;
          if (m.n >= p.max_length) end_of_detection(m, p, out, n, true, writer);
        } else if (p.max_sil <= 0.0) {
          end_of_detection(m, p, out, n, false, writer);
          m.state = kSilence;
        } else {
          m.sil = 1;
          ++m.n;
          m.state = kPossibleSilence;
          if (m.n == p.max_length) end_of_detection(m, p, out, n, true, writer);  // sil is kept
        }
      } else {  // kPossibleSilence
        if (ok) {
          ++m.n;
          m.sil = 0;
          m.state = kNoise;
          if (m.n >= p.max_length) end_of_detection(m, p, out, n, true, writer);
        } else if ((double)m.sil >= p.max_sil) {
          if (m.sil < m.n) end_of_detection(m, p, out, n, false, writer);
          else m.n = 0;
          m.state = kSilence;
          m.sil = 0;
        } else {
          ++m.n;
          ++m.sil;
          if (m.n >= p.max_length) end_of_detection(m, p, out, n, true, writer);  // sil is kept
        }
      }
    }
    __syncwarp();
  }
  if ((m.state == kNoise || m.state == kPossibleSilence) && m.n > 0 && m.n > m.sil)
    end_of_detection(m, p, out, n, false, writer);
  __syncwarp();

  double cum = 0.0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const Out c = i < n ? out[i] : Out(0);
    const double x = c > Out(0) ? 1.0 : c < Out(0) ? p.down : 0.0;
    unsigned nz = __ballot_sync(0xffffffffu, x != 0.0);
    double mine = cum;
    while (nz) {
      const int b = __ffs(nz) - 1;
      nz &= nz - 1;
      cum = cum + __shfl_sync(0xffffffffu, x, b);
      if (lane >= b) mine = cum;
    }
    if (i < n) out[i] = (Out)fmin(fmax(mine, 0.0), 1.0);
  }
}

template <typename Out>
int tokenize_launch(b2_ctx* h, const float* d_flags, const int64_t* off_host, int n_chunks,
                    const B2TokenizerParams& tp, Out* d_out, const int64_t* end_host = nullptr) {
  if (n_chunks <= 0) return B2_OK;
  B2Range range("b2:auditok_tokenize");
  MetaArena a;
  const size_t tbl = (size_t)(n_chunks + 1) * 8;
  B2_TRY(b2i_meta_begin(h, &a, 2 * tbl + 256));
  TokParams<Out> p;
  p.off = (const long long*)b2i_meta_put(&a, off_host, end_host ? tbl - 8 : tbl);
  p.end = end_host ? (const long long*)b2i_meta_put(&a, end_host, tbl - 8) : p.off + 1;
  B2_TRY(b2i_meta_commit(&a));
  p.flags = d_flags;
  p.out = d_out;
  p.n_chunks = n_chunks;
  p.min_length = tp.min_length;
  p.max_sil = tp.max_continuous_silence;
  p.max_length = tp.max_length;
  p.down = tp.non_speech_label - 1.0;
  const unsigned blocks = (unsigned)(((long long)n_chunks * 32 + 127) / 128);
  auditok_tokenize_kernel<Out><<<blocks, 128, 0, h->stream>>>(p);
  B2_CHECK_LAUNCH(h, "auditok_tokenize_kernel");
  return B2_OK;
}

}  // namespace

int b2i_tokenize_launch(b2_ctx* h, const float* d_flags, const int64_t* off_host, int n_chunks,
                        const B2TokenizerParams& tp, double* d_out) {
  return tokenize_launch(h, d_flags, off_host, n_chunks, tp, d_out);
}

int b2i_tokenize_inplace_launch(b2_ctx* h, float* d_flags_sig, const int64_t* off_host, int n_chunks,
                                const B2TokenizerParams& tp, const int64_t* end_host) {
  return tokenize_launch(h, (const float*)d_flags_sig, off_host, n_chunks, tp, d_flags_sig, end_host);
}
