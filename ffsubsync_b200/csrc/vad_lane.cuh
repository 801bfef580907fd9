// K1, lane-per-window arithmetic: one thread reduces one whole 10 ms window (energy + zero crossings)
// out of shared memory.  Replaces the inner loop of the reference's per-window detector call
// (ffsubsync/speech_transformers.py:155-183) for window sizes of C = fpw / 8 sixteen-byte chunks.
//
// Why: with 4 lanes per window (vad.cu's original layout) the per-window bookkeeping - shuffles,
// 64-bit sums, predicates - costs as many instructions as the arithmetic (3.25 instructions per byte
// and lane: the kernel saturates the issue slots of every SM to reach the HBM roofline, nothing can
// share the GPU with it).  Here a lane streams its window with 17 instructions per 16 bytes:
//   energy    x = 256 h + l (h = signed high byte, l = unsigned low byte)
//             sum x^2 = 65536 sum h^2 + 512 sum h l + sum l^2 : three 4-way byte dot products per 4 samples
//   crossings H = the 4 high bytes of 4 consecutive samples; (H ^ [H << 8 | previous H >> 24]) & 0x80808080
//             has one 0x80 byte per sign change; a dot product with 0x01010101 adds 128 per crossing
// Bank conflicts: lane i reads window i of the tile (stride 16 C bytes).  With C = 4 (mod 8) - 16 and
// 48 kHz - the 8 lanes of a quarter-warp would fall into 2 bank groups; lane i therefore starts at chunk
// r_i = (i >> 1) & 3 and walks its window circularly: bank group (4 i + r_i + c) mod 8 is a bijection of
// the 8 lanes at every step c, wrapped or not (lanes with equal r wrap together).  Other C: see lane_rotation.
//
// __host__ __device__: tests/host_emul/vad_emul.cu runs lane_window on the CPU against the plain
// definition (the build container has no GPU).
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define VAD_HD __host__ __device__ __forceinline__
#else
#define VAD_HD inline
#endif

namespace vadlane {

struct alignas(16) Chunk {   // 16 bytes = 8 samples
  uint32_t x, y, z, w;
};

VAD_HD uint32_t perm(uint32_t a, uint32_t b, uint32_t sel) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(a, b, sel);
#else
  const uint64_t v = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
  return r;
#endif
}
// 4-way byte dot products: signed x signed, signed x unsigned, unsigned x unsigned
VAD_HD int dot_ss(uint32_t a, uint32_t b, int c) {
#if defined(__CUDA_ARCH__)
  return __dp4a((int)a, (int)b, c);
#else
  for (int i = 0; i < 4; ++i) c += (int)(int8_t)(a >> (8 * i)) * (int)(int8_t)(b >> (8 * i));
  return c;
#endif
}
VAD_HD int dot_su(uint32_t a, uint32_t b, int c) {
#if defined(__CUDA_ARCH__)
  int d;
  asm("dp4a.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
  return d;
#else
  for (int i = 0; i < 4; ++i) c += (int)(int8_t)(a >> (8 * i)) * (int)(uint8_t)(b >> (8 * i));
  return c;
#endif
}
VAD_HD uint32_t dot_uu(uint32_t a, uint32_t b, uint32_t c) {
#if defined(__CUDA_ARCH__)
  return __dp4a(a, b, c);
#else
  for (int i = 0; i < 4; ++i) c += (uint32_t)(uint8_t)(a >> (8 * i)) * (uint32_t)(uint8_t)(b >> (8 * i));
  return c;
#endif
}
VAD_HD uint32_t funnel_l8(uint32_t prev, uint32_t cur) {   // (cur << 8) | (prev >> 24)
#if defined(__CUDA_ARCH__)
  return __funnelshift_l(prev, cur, 8);
#else
  return (cur << 8) | (prev >> 24);
#endif
}

struct Acc {
  int a, b;         // sum h^2, sum h l
  uint32_t c, z;    // sum l^2, 128 per sign change
};

// 4 consecutive samples = words (w0, w1); hprev = high bytes of the 4 samples before them
VAD_HD void group(uint32_t w0, uint32_t w1, uint32_t H, uint32_t& hprev, Acc& s) {
  const uint32_t L = perm(w0, w1, 0x6420);
  s.a = dot_ss(H, H, s.a);
  s.b = dot_su(H, L, s.b);
  s.c = dot_uu(L, L, s.c);
  s.z = dot_uu((H ^ funnel_l8(hprev, H)) & 0x80808080u, 0x01010101u, s.z);
  hprev = H;
}

// Largest start chunk of a lane and the start chunk of lane i, for windows of C chunks.
//   C odd      : stride already conflict-free                      r = 0
//   C = 2, 6 (8): groups (2 i) or (6 i) mod 8 hit 4 of 8 -> pairs   r = (i >> 2) & 1
//   C = 4 (8)  : groups {0, 4}                                      r = (i >> 1) & 3
//   C = 0 (8)  : all lanes in one group                             r = i & 7
VAD_HD constexpr int rotation_max(int C) { return (C & 1) ? 0 : ((C & 7) == 0 ? 7 : ((C & 7) == 4 ? 3 : 1)); }
VAD_HD int lane_rotation(int C, int lane) {
  if (C & 1) return 0;
  if ((C & 7) == 0) return lane & 7;
  if ((C & 7) == 4) return (lane >> 1) & 3;
  return (lane >> 2) & 1;
}

// Energy (sum of squares, exact) and sign changes of the window of C chunks at wbase (16-byte aligned),
// read circularly from chunk r <= RMAX = rotation_max(C).
template <int C, int RMAX>
VAD_HD void lane_window(const unsigned char* wbase, int r, long long& e, int& z) {
  const unsigned char* pb = wbase + 16 * r;
  Acc s0{0, 0, 0u, 0u}, s1{0, 0, 0u, 0u};
  uint32_t hprev = 0, hfirst = 0;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const unsigned char* p = pb + 16 * c;
    bool enters_chunk0 = false;
    if (c + RMAX >= C) {   // compile time: only the last RMAX steps can wrap
      if (r >= C - c) p -= 16 * C;
      enters_chunk0 = (r == C - c);
    }
    const Chunk v = *reinterpret_cast<const Chunk*>(p);
    const uint32_t H0 = perm(v.x, v.y, 0x7531), H1 = perm(v.z, v.w, 0x7531);
    if (c == 0) {
      hfirst = H0;
      hprev = H0 << 24;   // no sample before the first one read: its own sign, no crossing
    } else if (enters_chunk0) {
      hprev = H0 << 24;   // sample 0 of the window has no predecessor
    }
    group(v.x, v.y, H0, hprev, s0);
    group(v.z, v.w, H1, hprev, s1);
  }
  uint32_t zz = (s0.z + s1.z) >> 7;
  if (RMAX > 0) {
    // the boundary between the last chunk read (r - 1) and the first (r) was not seen by the loop
    const uint32_t closure = ((hprev >> 31) ^ (hfirst >> 7)) & 1u;
    if (r > 0) zz += closure;
  }
  z = (int)zz;
  e = 65536LL * ((long long)s0.a + s1.a) + 512LL * ((long long)s0.b + s1.b) + ((long long)s0.c + (long long)s1.c);
}

}  // namespace vadlane
