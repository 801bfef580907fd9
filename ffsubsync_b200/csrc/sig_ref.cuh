// The serialized-signal reference rule (DeserializeSpeechTransformer, ffsubsync/speech_transformers.py:987-1009)
// as sig_ref_kernel applies it, shared with its CPU emulator (tests/host_emul/sig_ref_emul.cu).
//
// Stored value x (float64, as np.load returns it) -> frame (float)(x < 1.0 ? label : x): the comparison runs in
// float64 and the result is rounded once to float32.  The domain is x < 1.0 or x == 1.0 (what every detector and
// rasteriser of the reference writes), where the frame is label or exactly 1.0f: two levels, like the energy
// detector's output.  x > 1.0 and NaN are out of the domain: the frame is flagged, and written as the label so that
// the chain behind it still sees a two-level reference (the call overwrites that video's outputs afterwards).
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define SR_HD __host__ __device__ __forceinline__
#else
#define SR_HD inline
#endif

// frames per ballot word, words per warp and chunk, warps per CTA (sig_ref_kernel)
constexpr int kSigUnits = 16;      // 32-frame units per warp per chunk: 16 independent 8-byte loads per lane
constexpr int kSigThreads = 1024;
constexpr long long kSigChunkFrames = (long long)(kSigThreads / 32) * kSigUnits * 32;   // 16384 frames, 128 KB in

// first_bad of a video no frame of which is out of the domain (the flag's initial value)
constexpr unsigned long long kSigNoBadFrame = ~0ull;

// true when x lies outside the domain (x > 1.0 or NaN)
SR_HD bool b2_sig_out_of_domain(double x) { return !(x <= 1.0); }

// the frame of stored value x: exactly 1.0f for x == 1.0, else the label (x < 1.0, and out-of-domain values)
SR_HD float b2_sig_frame(double x, float label) { return x == 1.0 ? 1.0f : label; }

// packed bit of a frame: m = (r == 1.0f), the bit the run path and the GSS rounds read
SR_HD bool b2_sig_bit(double x, float label) { return b2_sig_frame(x, label) == 1.0f; }
