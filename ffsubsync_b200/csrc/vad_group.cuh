// K1, lane-group arithmetic: G lanes share one window, lane g reduces the contiguous 16-byte chunks
// [g*CPL, (g+1)*CPL) (vad.cu's vad_energy_zcr_kernel sums the G partial results with shuffles).  This
// is the path of every 16-byte aligned batch the lane-per-window kernel (vad_lane.cuh) does not take:
// 48 kHz, 24 / 32 / 96 kHz, and 8 / 16 kHz under B2_VAD_LAYOUT=group.
//   energy    x^2 = x*lo8(x) + 256*x*hi8(x) (lo8 unsigned, hi8 signed): two 2-way 16x8 dot products per word
//   crossings f = [x0 : previous sample]; (w ^ f) carries prev->x0 in bit 15, x0->x1 in bit 31
//
// __host__ __device__: tests/host_emul/vad_emul.cu runs window_part_fast on the CPU against the plain
// definition for every (CPL, G) the launcher picks (the build container has no GPU).
#pragma once
#include <stdint.h>

#include "vad_lane.cuh"   // VAD_HD, vadlane::perm (byte permute), vadlane::dot_uu (unsigned 4-way dot product)

namespace vadgroup {

// 2-way dot products of the two 16-bit halves of a (signed) with bytes 0, 1 of b (unsigned) ...
VAD_HD int dot2_lo_su(uint32_t a, uint32_t b, int c) {
#if defined(__CUDA_ARCH__)
  asm("dp2a.lo.s32.u32 %0, %1, %2, %0;" : "+r"(c) : "r"(a), "r"(b));
  return c;
#else
  return c + (int)(int16_t)a * (int)(uint8_t)b + (int)(int16_t)(a >> 16) * (int)(uint8_t)(b >> 8);
#endif
}
// ... and with bytes 2, 3 of b (signed)
VAD_HD int dot2_hi_ss(uint32_t a, uint32_t b, int c) {
#if defined(__CUDA_ARCH__)
  asm("dp2a.hi.s32.s32 %0, %1, %2, %0;" : "+r"(c) : "r"(a), "r"(b));
  return c;
#else
  return c + (int)(int16_t)a * (int)(int8_t)(b >> 16) + (int)(int16_t)(a >> 16) * (int)(int8_t)(b >> 24);
#endif
}
VAD_HD uint32_t funnel_l16(uint32_t prev, uint32_t cur) {   // (cur << 16) | (prev >> 16)
#if defined(__CUDA_ARCH__)
  return __funnelshift_l(prev, cur, 16);
#else
  return (cur << 16) | (prev >> 16);
#endif
}

// One 32-bit word = samples (x0 = low half, x1 = high half).
VAD_HD void accum_word(uint32_t w, uint32_t prev, int& e_lo, int& e_hi, uint32_t& z128) {
  const uint32_t perm = vadlane::perm(w, 0u, 0x3120);  // bytes [lo8(x0), lo8(x1), hi8(x0), hi8(x1)]
  e_lo = dot2_lo_su(w, perm, e_lo);
  e_hi = dot2_hi_ss(w, perm, e_hi);
  const uint32_t f = funnel_l16(prev, w);
  // bytes 1 and 3 of the masked word are 0x80 per crossing: a 4-way byte dot product with ones
  // adds 128 per crossing (one IDP.4A instead of POPC + IADD)
  z128 = vadlane::dot_uu((w ^ f) & 0x80008000u, 0x01010101u, z128);
}

// Lane g of a window owns the contiguous 16-byte chunks [g*CPL, (g+1)*CPL) (CPL = 0: cpl_rt chunks).
// Adds the lane's sum of squares to e and its sign changes to z; the change between the last sample of
// lane g - 1 and the first of lane g is lane g's.
template <int CPL>
VAD_HD void window_part_fast(const unsigned char* wbase, int g, int cpl_rt, long long& e, int& z) {
  const int cpl = CPL > 0 ? CPL : cpl_rt;
  const unsigned char* cbase = wbase + 16 * g * cpl;
  uint32_t pw = 0;
  if (g > 0) pw = *reinterpret_cast<const uint32_t*>(cbase - 4);
  // two independent accumulator sets: the IDP chains are latency-bound otherwise (a CTA that shares
  // its SM with the correlation kernel has only 8 consumer warps to hide them)
  int e_lo = 0, e_hi = 0, f_lo = 0, f_hi = 0;
  uint32_t z128 = 0, y128 = 0;
  if (CPL > 0) {
    uint4 v[CPL > 0 ? CPL : 1];
#pragma unroll
    for (int c = 0; c < CPL; ++c) v[c] = *reinterpret_cast<const uint4*>(cbase + 16 * c);
    if (g == 0) pw = v[0].x << 16;  // first sample of the window: no crossing before it
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      accum_word(v[c].x, pw, e_lo, e_hi, z128);
      accum_word(v[c].y, v[c].x, f_lo, f_hi, y128);
      accum_word(v[c].z, v[c].y, e_lo, e_hi, z128);
      accum_word(v[c].w, v[c].z, f_lo, f_hi, y128);
      pw = v[c].w;
    }
  } else {
    for (int c = 0; c < cpl; ++c) {
      const uint4 v = *reinterpret_cast<const uint4*>(cbase + 16 * c);
      if (c == 0 && g == 0) pw = v.x << 16;
      accum_word(v.x, pw, e_lo, e_hi, z128);
      accum_word(v.y, v.x, f_lo, f_hi, y128);
      accum_word(v.z, v.y, e_lo, e_hi, z128);
      accum_word(v.w, v.z, f_lo, f_hi, y128);
      pw = v.w;
      if ((c & 15) == 15) {  // keep the 32-bit partial sums far from overflow
        e += (long long)e_lo + (long long)f_lo + ((long long)e_hi + (long long)f_hi) * 256LL;
        e_lo = e_hi = f_lo = f_hi = 0;
      }
    }
  }
  e += (long long)e_lo + (long long)f_lo + ((long long)e_hi + (long long)f_hi) * 256LL;
  z += (int)((z128 + y128) >> 7);
}

}  // namespace vadgroup
