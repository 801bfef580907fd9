// Device building blocks of the windowed cross-correlation (K3-K5): an in-place, shared-memory
// resident, mixed-radix (16,16,16,4) complex FFT of M = 2^14 points that carries one real block
// of P = 2^15 samples (even/odd packing), the real-FFT untangle / retangle performed directly in
// the digit-reversed ("position") order the decimation-in-frequency passes leave behind, and
// the decimation-in-time inverse.  The data flow is modelled and checked against np.fft in
// tests/fft_model.py.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

// Everything here is __host__ __device__ so that tests/host_emul/corr_emul.cu can run the exact
// kernel code thread by thread on the CPU (the build container has no GPU).
#define CORR_HD __host__ __device__ __forceinline__
#ifdef __CUDA_ARCH__
#define CORR_LDG(p) __ldg(p)
#define CORR_SYNC() __syncthreads()
#else
#define CORR_LDG(p) (*(p))
#define CORR_SYNC() ((void)0)
#endif

namespace corr {

constexpr int kM = 16384;        // complex points per block transform
constexpr int kP = 2 * kM;       // real samples per block
constexpr int kThreads = 512;
constexpr int kPairs = kM / 2;   // (position, partner) pairs of the packed half spectrum

// Shared-memory layout (dynamic): float2 buf[kM] | float2 tw1024[1024] | float2 fine32[32]
constexpr size_t kSmemBytes = (size_t)kM * 8 + 1024 * 8 + 32 * 8 + 256;

// XOR swizzle of the complex index: makes every pass (strides 1024, 64, 4, 1) and the
// untangle's mirrored partner access bank-conflict free for 8-byte accesses.
CORR_HD int swz(int i) { return i ^ ((i >> 4) & 3) ^ (((i >> 6) & 3) << 2); }

CORR_HD float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
CORR_HD float2 cmul_conj_a(float2 a, float2 b) {  // conj(a) * b
  return make_float2(a.x * b.x + a.y * b.y, a.x * b.y - a.y * b.x);
}
// Componentwise complex add and fused multiply-add.  Hopper has no packed fp32x2 instructions,
// so each is two scalar FADD / FFMA; the fused form is spelled out so that the device result does
// not depend on the compiler's contraction choices.
CORR_HD float2 padd(float2 a, float2 b) {
  return make_float2(a.x + b.x, a.y + b.y);
}
CORR_HD float2 pfma(float2 a, float2 b, float2 c) {  // a*b + c, componentwise
#if defined(__CUDA_ARCH__)
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
#else
  return make_float2(a.x * b.x + c.x, a.y * b.y + c.y);
#endif
}
CORR_HD float2 cadd(float2 a, float2 b) { return padd(a, b); }
CORR_HD float2 csub(float2 a, float2 b) { return pfma(b, make_float2(-1.f, -1.f), a); }
CORR_HD float2 cconj(float2 a) { return make_float2(a.x, -a.y); }

// position <-> frequency of the in-place DIF output, radices (16,16,16,4)
CORR_HD int freq_of_pos(int p) {
  return (p >> 10) | (((p >> 6) & 15) << 4) | (((p >> 2) & 15) << 8) | ((p & 3) << 12);
}
CORR_HD int pos_of_freq(int f) {
  return ((f & 15) << 10) | (((f >> 4) & 15) << 6) | (((f >> 8) & 15) << 2) | (f >> 12);
}
CORR_HD int partner_pos(int p) {
  return pos_of_freq((kM - freq_of_pos(p)) & (kM - 1));
}

struct Tables {
  const float2* tw1024;  // exp(-2 pi i t / 1024)
  const float2* fine32;  // exp(-2 pi i t / 32768), t < 32
};

CORR_HD void init_tables(float2* tw1024, float2* fine32, int tid) {
  for (int t = tid; t < 1024; t += kThreads) {
    float s, c;
    sincospif(-(float)t * (1.0f / 512.0f), &s, &c);
    tw1024[t] = make_float2(c, s);
  }
  if (tid < 32) {
    float s, c;
    sincospif(-(float)tid * (1.0f / 16384.0f), &s, &c);
    fine32[tid] = make_float2(c, s);
  }
}

// exp(-2 pi i a / 32768) for a in [0, 32768)
CORR_HD float2 twiddle15(const Tables& t, int a) {
  return cmul(t.tw1024[a >> 5], t.fine32[a & 31]);
}

// 4-point DFT in place: forward uses exp(-i pi/2 q k), inverse the conjugate.
template <bool INV>
CORR_HD void r4(float2& a0, float2& a1, float2& a2, float2& a3) {
  const float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = csub(a1, a3);
  a0 = cadd(t0, t2);
  a2 = csub(t0, t2);
  // -/+ i * t3 = (+-t3.y, -+t3.x): one swapped copy feeds both outputs
  const float2 sw = make_float2(t3.y, t3.x);
  const float2 pm = make_float2(1.f, -1.f), mp = make_float2(-1.f, 1.f);
  if (!INV) {
    a1 = pfma(sw, pm, t1);
    a3 = pfma(sw, mp, t1);
  } else {
    a1 = pfma(sw, mp, t1);
    a3 = pfma(sw, pm, t1);
  }
}

// multiply by exp(-+ 2 pi i n / 16) (forward: -, inverse: +)
template <bool INV, int N>
CORR_HD float2 rot16(float2 v) {
  constexpr float c1 = 0.92387953251128674f, s1 = 0.38268343236508977f, r = 0.70710678118654752f;
  constexpr int n = N & 15;
  float cr, ci;
  if (n == 0) return v;
  if (n == 1) { cr = c1; ci = -s1; }
  else if (n == 2) { cr = r; ci = -r; }
  else if (n == 3) { cr = s1; ci = -c1; }
  else if (n == 4) { return INV ? make_float2(-v.y, v.x) : make_float2(v.y, -v.x); }
  else if (n == 6) { cr = -r; ci = -r; }
  else if (n == 9) { cr = -c1; ci = s1; }
  else { cr = 1.f; ci = 0.f; }
  if (INV) ci = -ci;
  return make_float2(v.x * cr - v.y * ci, v.x * ci + v.y * cr);
}

// 16-point DIF butterfly with the pass twiddles w^(j k) folded in.
// In:  v[q]      = x[j + q*sub],           q = q_lo + 4 q_hi
// Out: v[4a + b] = X[k = a + 4b] * w1^k    (to be stored at j + k*sub)
// w1 = w_span^j (forward twiddle).  Twiddle powers come from a short product chain (depth <= 4).
CORR_HD void bfly16_dif(float2 (&v)[16], float2 w1) {
#pragma unroll
  for (int q = 0; q < 4; ++q) r4<false>(v[q], v[q + 4], v[q + 8], v[q + 12]);
  const float2 w2 = cmul(w1, w1);
  const float2 w3 = cmul(w2, w1);
  // a = 1 (v[4..7]), a = 2 (v[8..11]), a = 3 (v[12..15]); q_lo = index - 4a
  v[4] = cmul(v[4], w1);
  v[5] = rot16<false, 1>(cmul(v[5], w1));
  v[6] = rot16<false, 2>(cmul(v[6], w1));
  v[7] = rot16<false, 3>(cmul(v[7], w1));
  v[8] = cmul(v[8], w2);
  v[9] = rot16<false, 2>(cmul(v[9], w2));
  v[10] = rot16<false, 4>(cmul(v[10], w2));
  v[11] = rot16<false, 6>(cmul(v[11], w2));
  v[12] = cmul(v[12], w3);
  v[13] = rot16<false, 3>(cmul(v[13], w3));
  v[14] = rot16<false, 6>(cmul(v[14], w3));
  v[15] = rot16<false, 9>(cmul(v[15], w3));
#pragma unroll
  for (int a = 0; a < 4; ++a) r4<false>(v[4 * a], v[4 * a + 1], v[4 * a + 2], v[4 * a + 3]);
  const float2 w4 = cmul(w2, w2);
  const float2 w8 = cmul(w4, w4);
  const float2 w12 = cmul(w8, w4);
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    v[4 * a + 1] = cmul(v[4 * a + 1], w4);
    v[4 * a + 2] = cmul(v[4 * a + 2], w8);
    v[4 * a + 3] = cmul(v[4 * a + 3], w12);
  }
}

// Exact mirror: In v[4a+b] = Y[k = a+4b] (from j + k*sub); Out v[q] = 16-point inverse DFT of
// Y[k] * conj(w1)^k, to be stored at j + q*sub.  w1c = conj(w_span^j).
CORR_HD void bfly16_dit(float2 (&v)[16], float2 w1c) {
  const float2 w2 = cmul(w1c, w1c);
  const float2 w3 = cmul(w2, w1c);
  const float2 w4 = cmul(w2, w2);
  const float2 w8 = cmul(w4, w4);
  const float2 w12 = cmul(w8, w4);
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    v[4 * a + 1] = cmul(v[4 * a + 1], w4);
    v[4 * a + 2] = cmul(v[4 * a + 2], w8);
    v[4 * a + 3] = cmul(v[4 * a + 3], w12);
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) r4<true>(v[4 * a], v[4 * a + 1], v[4 * a + 2], v[4 * a + 3]);
  v[4] = cmul(v[4], w1c);
  v[5] = cmul(rot16<true, 1>(v[5]), w1c);
  v[6] = cmul(rot16<true, 2>(v[6]), w1c);
  v[7] = cmul(rot16<true, 3>(v[7]), w1c);
  v[8] = cmul(v[8], w2);
  v[9] = cmul(rot16<true, 2>(v[9]), w2);
  v[10] = cmul(rot16<true, 4>(v[10]), w2);
  v[11] = cmul(rot16<true, 6>(v[11]), w2);
  v[12] = cmul(v[12], w3);
  v[13] = cmul(rot16<true, 3>(v[13]), w3);
  v[14] = cmul(rot16<true, 6>(v[14]), w3);
  v[15] = cmul(rot16<true, 9>(v[15]), w3);
#pragma unroll
  for (int q = 0; q < 4; ++q) r4<true>(v[q], v[q + 4], v[q + 8], v[q + 12]);
}

// forward twiddle w_span^j for the radix-16 pass whose element stride is 2^SUB_LOG2
template <int SUB_LOG2>
CORR_HD float2 pass_twiddle(const Tables& t, int j) {
  if (SUB_LOG2 == 10) return twiddle15(t, j << 1);  // span 16384
  if (SUB_LOG2 == 6) return t.tw1024[j];            // span 1024
  // span 64: exp(-2 pi i j / 64), j = 0..3.  Four constants selected in registers: reading
  // tw1024[16 j] is a 4-way bank conflict (4 addresses 128 bytes apart per warp).
  const float c = j == 0 ? 1.f : j == 1 ? 0.99518472667219693f : j == 2 ? 0.98078528040323043f
                                                                          : 0.95694033573220882f;
  const float s = j == 0 ? 0.f : j == 1 ? -0.09801714032956060f : j == 2 ? -0.19509032201612825f
                                                                           : -0.29028467725446233f;
  return make_float2(c, s);
}

// Swizzled shared-memory index of element q of radix-16 butterfly u, without re-deriving the
// swizzle per access (r1c profile: ~20 % of the kernel's instructions were index arithmetic).
// For butterfly u of the pass with element stride 2^S the index is base + q*2^S with
// base = ((u >> S) << (S+4)) + (u & (2^S-1)); the XOR swizzle then reduces to
//   S = 10:  swz(base) + q*1024                          (swizzle bits 4..7 come from j only)
//   S =  6:  reg[q & 3] + q*64,  reg[m] = base ^ ((j>>4)&3) ^ (m<<2)
//   S =  2:  reg ^ c(q),         reg = (blk<<6) ^ (((blk&3)<<2) | j),  c(q) compile-time
// (identities checked exhaustively in tests/test_host_cpu.py via the kernel emulation).
template <int S>
CORR_HD void pass_addr_init(int u, int (&reg)[4]) {
  const int j = u & ((1 << S) - 1);
  const int base = ((u >> S) << (S + 4)) + j;
  if (S == 10) {
    reg[0] = swz(base);
  } else if (S == 6) {
    const int b0 = base ^ ((j >> 4) & 3);
#pragma unroll
    for (int m = 0; m < 4; ++m) reg[m] = b0 ^ (m << 2);
  } else {
    const int blk = u >> 2;
    reg[0] = (blk << 6) ^ (((blk & 3) << 2) | j);
  }
}
template <int S>
CORR_HD int pass_addr(const int (&reg)[4], int q) {
  if (S == 10) return reg[0] + (q << 10);
  if (S == 6) return reg[q & 3] + (q << 6);
  return reg[0] ^ (((q & 3) << 2) | ((q >> 2) << 4) | (q >> 2));
}

// One in-place radix-16 DIF pass over shared memory (spans 1024 and 64).
template <int SUB_LOG2>
CORR_HD void dif16_pass_smem(float2* buf, const Tables& t, int tid) {
#pragma unroll 1
  for (int rep = 0; rep < 2; ++rep) {
    const int u = tid + rep * kThreads;
    const int j = u & ((1 << SUB_LOG2) - 1);
    int reg[4];
    pass_addr_init<SUB_LOG2>(u, reg);
    float2 v[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) v[q] = buf[pass_addr<SUB_LOG2>(reg, q)];
    bfly16_dif(v, pass_twiddle<SUB_LOG2>(t, j));
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) buf[pass_addr<SUB_LOG2>(reg, a + 4 * b)] = v[4 * a + b];
  }
}

template <int SUB_LOG2>
CORR_HD void dit16_pass_smem(float2* buf, const Tables& t, int tid) {
#pragma unroll 1
  for (int rep = 0; rep < 2; ++rep) {
    const int u = tid + rep * kThreads;
    const int j = u & ((1 << SUB_LOG2) - 1);
    int reg[4];
    pass_addr_init<SUB_LOG2>(u, reg);
    float2 v[16];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) v[4 * a + b] = buf[pass_addr<SUB_LOG2>(reg, a + 4 * b)];
    bfly16_dit(v, cconj(pass_twiddle<SUB_LOG2>(t, j)));
#pragma unroll
    for (int q = 0; q < 16; ++q) buf[pass_addr<SUB_LOG2>(reg, q)] = v[q];
  }
}

// last DIF pass / first DIT pass: radix 4 on 4 contiguous points, no twiddles
template <bool INV>
CORR_HD void r4_pass_smem(float2* buf, int tid) {
#pragma unroll 2
  for (int rep = 0; rep < kM / 4 / kThreads; ++rep) {
    // swz(4u + q) = swz(4u) ^ q: q only occupies bits 0..1, which the swizzle XORs but never reads
    const int s0 = swz((tid + rep * kThreads) << 2);
    float2 a0 = buf[s0], a1 = buf[s0 ^ 1], a2 = buf[s0 ^ 2], a3 = buf[s0 ^ 3];
    r4<INV>(a0, a1, a2, a3);
    buf[s0] = a0;
    buf[s0 ^ 1] = a1;
    buf[s0 ^ 2] = a2;
    buf[s0 ^ 3] = a3;
  }
}

// A real block as the kernels see it: value(t) = 2*src[t]-1 for t in [t_lo, t_hi), else 0.
struct BlockSource {
  const float* src;  // may point outside the array; only [t_lo, t_hi) is dereferenced
  int t_lo, t_hi;
};

// The 16 complex inputs (32 samples) of one first-pass butterfly, j + q*1024, q = 0..15.
// All global loads are issued back to back with clamped (always valid) addresses and masked
// afterwards, so that the 16 (or 32) loads of a thread are in flight together; a branchy
// per-element version serialised them on the memory latency.
CORR_HD void load_block16(const BlockSource& s, int j, float2 (&v)[16]) {
  if (s.t_hi <= s.t_lo) {
#pragma unroll
    for (int q = 0; q < 16; ++q) v[q] = make_float2(0.f, 0.f);
    return;
  }
  const bool vec_ok = (reinterpret_cast<uintptr_t>(s.src) & 7) == 0;
  const int n_lo = (s.t_lo + 1) >> 1, n_hi = s.t_hi >> 1;  // pairs fully inside [t_lo, t_hi)
  if (vec_ok && n_hi > n_lo) {
    const float2* src2 = reinterpret_cast<const float2*>(s.src);
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int n = j + (q << 10);
      v[q] = CORR_LDG(src2 + min(max(n, n_lo), n_hi - 1));
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int n = j + (q << 10);
      const bool full = (n >= n_lo) && (n < n_hi);
      v[q].x = full ? 2.f * v[q].x - 1.f : 0.f;
      v[q].y = full ? 2.f * v[q].y - 1.f : 0.f;
    }
    // at most two half-valid pairs per block (odd t_lo / odd t_hi)
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int n = j + (q << 10);
      if ((s.t_lo & 1) && n == n_lo - 1) v[q].y = 2.f * CORR_LDG(s.src + s.t_lo) - 1.f;
      if ((s.t_hi & 1) && n == n_hi) v[q].x = 2.f * CORR_LDG(s.src + s.t_hi - 1) - 1.f;
    }
  } else {
    float a[16], b[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int t0 = 2 * (j + (q << 10));
      a[q] = CORR_LDG(s.src + min(max(t0, s.t_lo), s.t_hi - 1));
      b[q] = CORR_LDG(s.src + min(max(t0 + 1, s.t_lo), s.t_hi - 1));
    }
#pragma unroll
    for (int q = 0; q < 16; ++q) {
      const int t0 = 2 * (j + (q << 10));
      v[q].x = (t0 >= s.t_lo && t0 < s.t_hi) ? 2.f * a[q] - 1.f : 0.f;
      v[q].y = (t0 + 1 >= s.t_lo && t0 + 1 < s.t_hi) ? 2.f * b[q] - 1.f : 0.f;
    }
  }
}

// A subtitle block rasterised into shared memory as one byte per 10 ms frame (1 = inside a cue):
// value(t) = (mask[t] ? hi : -1) for t < t_hi, else 0;  hi = 2*min(1/ratio, 1) - 1.
struct BitSource {
  const uint32_t* words;  // kP/32 words in shared memory: bit t = sample t of the block is inside a cue
  int t_hi;               // samples t >= t_hi are zero padding (t_hi <= L)
  float hi;               // value of a frame inside a cue after x -> 2x-1 (outside: -1)
};
// samples 2j', 2j'+1 (j' = j + 1024 q) are two adjacent bits of word (j >> 4) + 64 q; the shift is
// the same for all q
CORR_HD void load_block16(const BitSource& s, int j, float2 (&v)[16]) {
  const int sh = 2 * (j & 15);
  const uint32_t* w = s.words + (j >> 4);
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    const int t0 = 2 * (j + (q << 10));
    const uint32_t m = w[q << 6] >> sh;
    v[q].x = t0 < s.t_hi ? ((m & 1u) ? s.hi : -1.f) : 0.f;
    v[q].y = t0 + 1 < s.t_hi ? ((m & 2u) ? s.hi : -1.f) : 0.f;
  }
}

// A FULL bit-mask block (t_hi == L, every block of a signal but its last): which samples are zero
// padding is then a function of q alone, except for the one q that straddles L.  QB = L / 2048 is a
// compile-time constant: q < QB needs no range test (2048 (q + 1) <= L), q > QB is all padding.
// (r1k profile: the range tests were half of the 12 instructions spent per q on decoding.)
template <int QB>
struct BitSourceFull {
  const uint32_t* words;
  int L;
  float hi;
};
template <int QB>
CORR_HD void load_block16(const BitSourceFull<QB>& s, int j, float2 (&v)[16]) {
  const int sh = 2 * (j & 15);
  const uint32_t* w = s.words + (j >> 4);
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    if (q < QB) {
      const uint32_t m = w[q << 6] >> sh;
      v[q].x = (m & 1u) ? s.hi : -1.f;
      v[q].y = (m & 2u) ? s.hi : -1.f;
    } else if (q == QB) {
      const int t0 = 2 * (j + (q << 10));
      const uint32_t m = w[q << 6] >> sh;
      v[q].x = t0 < s.L ? ((m & 1u) ? s.hi : -1.f) : 0.f;
      v[q].y = t0 + 1 < s.L ? ((m & 2u) ? s.hi : -1.f) : 0.f;
    } else {
      v[q] = make_float2(0.f, 0.f);
    }
  }
}

// A float block that lies entirely inside its signal and starts 8-byte aligned (the interior
// blocks of a reference signal): no clamping, no masking.
struct BlockSourceFull {
  const float2* src2;
};
CORR_HD void load_block16(const BlockSourceFull& s, int j, float2 (&v)[16]) {
#pragma unroll
  for (int q = 0; q < 16; ++q) v[q] = CORR_LDG(s.src2 + j + (q << 10));
#pragma unroll
  for (int q = 0; q < 16; ++q) {
    v[q].x = 2.f * v[q].x - 1.f;
    v[q].y = 2.f * v[q].y - 1.f;
  }
}

// First DIF pass (span 16384) reading the block straight from its source (global memory for
// float signals, the shared-memory copy of the block's speech bits in bit-mask mode).
// Returns the thread's partial sum of squares of the (transformed) samples it loaded.
template <class Source>
CORR_HD float dif16_pass1_global(float2* buf, const Tables& t, int tid, const Source& s) {
  float ss = 0.f;
#pragma unroll 1
  for (int rep = 0; rep < 2; ++rep) {
    const int j = tid + rep * kThreads;
    float2 v[16];
    load_block16(s, j, v);
#pragma unroll
    for (int q = 0; q < 16; ++q) ss += v[q].x * v[q].x + v[q].y * v[q].y;
    bfly16_dif(v, pass_twiddle<10>(t, j));
    const int s0 = swz(j);  // swz(j + k*1024) = swz(j) + k*1024
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) buf[s0 + ((a + 4 * b) << 10)] = v[4 * a + b];
  }
  return ss;
}

// Forward transform of one real block: on return (after the trailing __syncthreads) buf holds
// DFT_M of z[n] = x[2n] + i x[2n+1] in position order.  The caller must have synchronised all
// readers of buf before calling.
template <class Source>
CORR_HD float forward_block(float2* buf, const Tables& t, int tid, const Source& s) {
  const float ss = dif16_pass1_global(buf, t, tid, s);
  CORR_SYNC();
  dif16_pass_smem<6>(buf, t, tid);
  CORR_SYNC();
  dif16_pass_smem<2>(buf, t, tid);
  CORR_SYNC();
  r4_pass_smem<false>(buf, tid);
  CORR_SYNC();
  return ss;
}

// Passes 2..4 of the forward transform (everything after the first pass), trailing barrier included.
CORR_HD void forward_rest(float2* buf, const Tables& t, int tid) {
  CORR_SYNC();
  dif16_pass_smem<6>(buf, t, tid);
  CORR_SYNC();
  dif16_pass_smem<2>(buf, t, tid);
  CORR_SYNC();
  r4_pass_smem<false>(buf, tid);
  CORR_SYNC();
}

// First pass of a bit-mask block (uniform arguments): full blocks take the variant specialised for
// L / 2048, the last block of a signal the general one.
CORR_HD float bits_pass1(float2* buf, const Tables& t, int tid, const uint32_t* words, int t_hi, int L,
                         float hi) {
  if (t_hi == L) {
    switch (L >> 11) {
      case 8: return dif16_pass1_global(buf, t, tid, BitSourceFull<8>{words, L, hi});
      case 9: return dif16_pass1_global(buf, t, tid, BitSourceFull<9>{words, L, hi});
      case 10: return dif16_pass1_global(buf, t, tid, BitSourceFull<10>{words, L, hi});
      case 11: return dif16_pass1_global(buf, t, tid, BitSourceFull<11>{words, L, hi});
      case 12: return dif16_pass1_global(buf, t, tid, BitSourceFull<12>{words, L, hi});
      case 13: return dif16_pass1_global(buf, t, tid, BitSourceFull<13>{words, L, hi});
      case 14: return dif16_pass1_global(buf, t, tid, BitSourceFull<14>{words, L, hi});
      case 15: return dif16_pass1_global(buf, t, tid, BitSourceFull<15>{words, L, hi});
      case 16: return dif16_pass1_global(buf, t, tid, BitSourceFull<16>{words, L, hi});
      default: break;
    }
  }
  return dif16_pass1_global(buf, t, tid, BitSource{words, t_hi, hi});
}

// First pass of a float block whose sample t is src[t] for t in [t_lo, t_hi) (zero elsewhere).
CORR_HD float float_pass1(float2* buf, const Tables& t, int tid, const float* src, int t_lo, int t_hi) {
  if (t_lo == 0 && t_hi == kP && (reinterpret_cast<uintptr_t>(src) & 7) == 0)
    return dif16_pass1_global(buf, t, tid, BlockSourceFull{reinterpret_cast<const float2*>(src)});
  BlockSource s;
  s.src = src;
  s.t_lo = t_lo;
  s.t_hi = t_hi;
  return dif16_pass1_global(buf, t, tid, s);
}

// Packed half spectrum (x2) of the real block at an even position p and its partner q:
//   H[p] = E - i T,  H[q] = conj(E) - i conj(T),  E = Z[p] + conj Z[q],  T = w^f (Z[p] - conj Z[q])
CORR_HD void untangle_pair(const float2* buf, const Tables& t, int p, int q,
                                              float2& hp, float2& hq) {
  const float2 zp = buf[swz(p)];
  const float2 zq = buf[swz(q)];
  const float2 e = make_float2(zp.x + zq.x, zp.y - zq.y);
  const float2 d = make_float2(zp.x - zq.x, zp.y + zq.y);
  const float2 tt = cmul(twiddle15(t, freq_of_pos(p)), d);
  hp = make_float2(e.x + tt.y, e.y - tt.x);
  hq = make_float2(e.x - tt.y, -e.y - tt.x);
}

// Same value for one arbitrary position (used for the four special positions 0..3).
CORR_HD float2 untangle_one(const float2* buf, const Tables& t, int p) {
  const int q = partner_pos(p);
  const float2 zp = buf[swz(p)];
  const float2 zq = buf[swz(q)];
  const float2 e = make_float2(zp.x + zq.x, zp.y - zq.y);
  const float2 d = make_float2(zp.x - zq.x, zp.y + zq.y);
  const float2 tt = cmul(twiddle15(t, freq_of_pos(p)), d);
  return make_float2(e.x + tt.y, e.y - tt.x);
}

// Thread-to-pair map shared by the producer (reference spectra) and the consumer (subtitle
// blocks): pair r = tid + u*kThreads covers even position p = 2r and its partner (always odd).
// The four positions whose partner is not of that form are handled by pairs 0 and 1:
//   pair 0 = (position 0: DC and Nyquist bins packed as (re, im); position 2: f = M/2, its own
//             partner),  pair 1 = (position 1, position 3), each other's partners.
CORR_HD void slot_positions(int r, int& p, int& q) {
  if (r >= 2) {
    p = 2 * r;
    q = partner_pos(p);
  } else if (r == 0) {
    p = 0;
    q = 2;
  } else {
    p = 1;
    q = 3;
  }
}

// Per-thread constants of that map, computed once per kernel.  For u >= 1 the pair r = tid + 512u
// has p = 1024u + 2 tid and partner q = 1024(16-u) + (1023 - 2 tid) (the digit-reversed image of
// f -> M - f when the lowest frequency digit u is non-zero), frequency f = F(tid) | u; the
// swizzled addresses are then a per-thread base plus a compile-time multiple of 1024.
struct PairCtx {
  int sp0;     // swz(2 tid)
  int sq0;     // swz(1023 - 2 tid)
  int sq_u0;   // swz(partner of position 2 tid)     (u = 0, tid >= 2)
  int f_base;  // freq_of_pos(2 tid): low 4 bits are zero
  // w^f_base.  The twiddle of slot u is w^(f_base | u) = w_base * fine32[u]: one broadcast table
  // read per slot.  (Reading tw1024[(f_base | u) >> 5] per slot was an 8-way bank conflict - the
  // digit-reversed f_base of neighbouring threads differ by multiples of 256 - and 43 % of the
  // product phase's shared-memory wavefronts, r1m full-load capture.)
  float2 w_base;
};
CORR_HD PairCtx pair_ctx(const Tables& t, int tid) {  // after init_tables + barrier
  PairCtx c;
  c.sp0 = swz(2 * tid);
  c.sq0 = swz(1023 - 2 * tid);
  c.sq_u0 = swz(partner_pos(2 * tid));
  c.f_base = freq_of_pos(2 * tid);
  c.w_base = twiddle15(t, c.f_base);
  return c;
}

// H[p], H[q] of pair slot u of this thread (see untangle_pair for the algebra).
CORR_HD void untangle_slot(const float2* buf, const Tables& t, const PairCtx& c, int tid, int u,
                           float2& hp, float2& hq) {
  if (u == 0 && tid < 2) {
    if (tid == 0) {
      const float2 z0 = buf[swz(0)];
      hp = make_float2(2.f * (z0.x + z0.y), 2.f * (z0.x - z0.y));
      hq = untangle_one(buf, t, 2);
    } else {
      untangle_pair(buf, t, 1, 3, hp, hq);
    }
    return;
  }
  const float2 zp = buf[c.sp0 + (u << 10)];
  const float2 zq = buf[u == 0 ? c.sq_u0 : c.sq0 + ((16 - u) << 10)];
  const float2 e = make_float2(zp.x + zq.x, zp.y - zq.y);
  const float2 d = make_float2(zp.x - zq.x, zp.y + zq.y);
  const float2 tt = cmul(cmul(c.w_base, t.fine32[u]), d);
  hp = make_float2(e.x + tt.y, e.y - tt.x);
  hq = make_float2(e.x - tt.y, -e.y - tt.x);
}

// Inverse of the packing for the accumulated product spectrum C (position order):
//   Zc[p] = E' + i T',  Zc[q] = conj(E') + i conj(T'),  E' = C[p] + conj C[q],
//   T' = conj(w^f) (C[p] - conj C[q])
CORR_HD void retangle_pair(const Tables& t, int p, float2 cp, float2 cq,
                                              float2& zp, float2& zq) {
  const float2 e = make_float2(cp.x + cq.x, cp.y - cq.y);
  const float2 d = make_float2(cp.x - cq.x, cp.y + cq.y);
  const float2 tt = cmul(cconj(twiddle15(t, freq_of_pos(p))), d);
  zp = make_float2(e.x - tt.y, e.y + tt.x);
  zq = make_float2(e.x + tt.y, -e.y + tt.x);
}

// ---- per-thread phases of the two kernels (also driven by tests/host_emul/corr_emul.cu) ------

struct SubState {
  float2 cp[16];  // accumulated conj(A) * B at the even position of each of the thread's 16 pairs
  float2 cq[16];  // ... and at its partner
  float ss;       // sum of squares of the subtitle samples this thread loaded
};

CORR_HD void sub_state_clear(SubState& st) {
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    st.cp[u] = make_float2(0.f, 0.f);
    st.cq[u] = make_float2(0.f, 0.f);
  }
  st.ss = 0.f;
}

// Producer: packed half spectrum (x2) of the reference block in buf -> spec[kPairs] float4.
CORR_HD void spec_store(const float2* buf, const Tables& t, const PairCtx& c, int tid, float4* spec) {
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    float2 hp, hq;
    untangle_slot(buf, t, c, tid, u, hp, hq);
    spec[tid + u * kThreads] = make_float4(hp.x, hp.y, hq.x, hq.y);
  }
}

// conj(A) * B for the thread's pair slot u: A from the subtitle block spectrum in buf, B = b.
CORR_HD void product_terms(const float2* buf, const Tables& t, const PairCtx& c, int tid, int u,
                           float4 b, float2& dp, float2& dq) {
  float2 hp, hq;
  untangle_slot(buf, t, c, tid, u, hp, hq);
  if (u == 0 && tid == 0) {
    dp = make_float2(hp.x * b.x, hp.y * b.y);  // two real bins: DC and Nyquist
  } else {
    dp = cmul_conj_a(hp, make_float2(b.x, b.y));
  }
  dq = cmul_conj_a(hq, make_float2(b.z, b.w));
}

// Consumer: acc += conj(A) * B for the subtitle block spectrum in buf and the stored B.
// (Used by sub_correlate_kernel on the device and by tests/host_emul on the CPU.)
CORR_HD void sub_accumulate(SubState& st, const float2* buf, const Tables& t, const PairCtx& c,
                            int tid, const float4* spec) {
  // the stored reference spectrum is read two slots ahead of its use (L2 latency)
  float4 b0 = CORR_LDG(spec + tid);
  float4 b1 = CORR_LDG(spec + tid + kThreads);
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    const int r = tid + u * kThreads;
    const float4 b = b0;
    b0 = b1;
    if (u + 2 < 16) b1 = CORR_LDG(spec + r + 2 * kThreads);
    float2 dp, dq;
    product_terms(buf, t, c, tid, u, b, dp, dq);
    st.cp[u] = cadd(st.cp[u], dp);
    st.cq[u] = cadd(st.cq[u], dq);
  }
}

// Consumer, after the last block: accumulated spectrum -> position-order input of the inverse
// transform, written into buf (every position is written exactly once).
CORR_HD void sub_retangle_store(const SubState& st, float2* buf, const Tables& t, const PairCtx& c,
                                int tid) {
#pragma unroll
  for (int u = 0; u < 16; ++u) {
    float2 zp, zq;
    if (u == 0 && tid == 0) {
      const float c0 = st.cp[0].x, cm = st.cp[0].y;
      zp = make_float2(c0 + cm, c0 - cm);
      float2 unused;
      retangle_pair(t, 2, st.cq[0], st.cq[0], zq, unused);
      buf[swz(0)] = zp;
      buf[swz(2)] = zq;
    } else if (u == 0 && tid == 1) {
      retangle_pair(t, 1, st.cp[0], st.cq[0], zp, zq);
      buf[swz(1)] = zp;
      buf[swz(3)] = zq;
    } else {
      // same algebra as retangle_pair with the thread's precomputed addresses / frequency
      const float2 cp = st.cp[u], cq = st.cq[u];
      const float2 e = make_float2(cp.x + cq.x, cp.y - cq.y);
      const float2 d = make_float2(cp.x - cq.x, cp.y + cq.y);
      const float2 tt = cmul(cconj(cmul(c.w_base, t.fine32[u])), d);
      buf[c.sp0 + (u << 10)] = make_float2(e.x - tt.y, e.y + tt.x);
      buf[u == 0 ? c.sq_u0 : c.sq0 + ((16 - u) << 10)] = make_float2(e.x + tt.y, -e.y + tt.x);
    }
  }
}

// Inverse transform of buf (position order in, natural order out).  Needs a barrier before
// (all retangle stores visible) and leaves one after.
CORR_HD void inverse_passes_1(float2* buf, int tid) { r4_pass_smem<true>(buf, tid); }
CORR_HD void inverse_passes_2(float2* buf, const Tables& t, int tid) { dit16_pass_smem<2>(buf, t, tid); }
CORR_HD void inverse_passes_3(float2* buf, const Tables& t, int tid) { dit16_pass_smem<6>(buf, t, tid); }
CORR_HD void inverse_passes_4(float2* buf, const Tables& t, int tid) { dit16_pass_smem<10>(buf, t, tid); }

// c[m] for the window: real/imag parts of the natural-order inverse output interleave.
// The transforms are unnormalised and the spectra carry factors 2 (A), 2 (B), 2 (retangle).
constexpr float kOutScale = 1.0f / (8.0f * (float)kM);
CORR_HD float window_value(const float2* buf, int m) {
  const float2 z = buf[swz(m >> 1)];
  return ((m & 1) ? z.y : z.x) * kOutScale;
}

}  // namespace corr
