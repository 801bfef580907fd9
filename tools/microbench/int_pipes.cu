// Integer pipe throughput on sm_90a (H100): byte / halfword dot products against IMAD, LOP3, PRMT.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o int_pipes int_pipes.cu && ./int_pipes
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdint.h>

template <int OP>
__global__ void __launch_bounds__(1024) k(uint32_t* out, uint32_t seed, int iters) {
  uint32_t a[8], b = seed * 2654435761u + threadIdx.x, c = seed ^ (blockIdx.x * 40503u);
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = seed + i * 977u + threadIdx.x;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (OP == 0) asm volatile("dp4a.u32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 1) asm volatile("dp4a.s32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 2) asm volatile("dp4a.s32.s32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 3) asm volatile("dp2a.lo.s32.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 4) asm volatile("dp2a.hi.s32.s32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 5) asm volatile("mad.lo.u32 %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 6) asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 7) asm volatile("prmt.b32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 8) asm volatile("shf.l.wrap.b32 %0, %0, %1, %2;" : "+r"(a[i]) : "r"(b), "r"(c));
      if (OP == 9) asm volatile("add.u32 %0, %0, %1;" : "+r"(a[i]) : "r"(b));
      if (OP == 10) asm volatile("{.reg .u32 t; popc.b32 t, %0; add.u32 %0, t, %1;}" : "+r"(a[i]) : "r"(b));
      if (OP == 11) asm volatile("vabsdiff4.u32.u32.u32.add %0, %1, %2, %0;" : "+r"(a[i]) : "r"(b), "r"(c));
    }
  }
  uint32_t s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s ^= a[i];
  if (s == 0x12345) out[0] = s;
}

template <int OP>
void run(const char* name, uint32_t* d, int sms) {
  const int iters = 4096, blocks = sms * 2;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  k<OP><<<blocks, 1024>>>(d, 1, 16);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k<OP><<<blocks, 1024>>>(d, 3, iters);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  int clk_khz;
  cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  const double ops = (double)blocks * 1024 * iters * 8;
  const double per_clk_sm = ops / (ms * 1e-3) / ((double)clk_khz * 1e3) / sms;
  printf("%-22s %8.3f ms  %7.1f lane-ops/clk/SM (at the nominal %d MHz)\n", name, ms, per_clk_sm, clk_khz / 1000);
}

int main() {
  int sms;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  uint32_t* d;
  cudaMalloc(&d, 64);
  run<0>("dp4a.u32.u32", d, sms);
  run<1>("dp4a.s32.u32", d, sms);
  run<2>("dp4a.s32.s32", d, sms);
  run<3>("dp2a.lo.s32.u32", d, sms);
  run<4>("dp2a.hi.s32.s32", d, sms);
  run<5>("mad.lo.u32 (IMAD)", d, sms);
  run<6>("lop3", d, sms);
  run<7>("prmt", d, sms);
  run<8>("shf.l.wrap", d, sms);
  run<9>("add.u32", d, sms);
  run<10>("popc + add", d, sms);
  run<11>("vabsdiff4.add", d, sms);
  return 0;
}
