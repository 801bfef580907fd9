// Which energy kernel b2i_vad_launch (vad.cu) takes for a table of signals, as a host function of the table alone:
// the launcher and the batched sync calls' planner (sync_plan.h, through b2i_vad_lane_eligible) decide with it, and
// the planner's CPU emulator (tests/host_emul/seg_ref_emul.cu) reports it, so a test can pin which kernel a table
// reaches.
//   lane      vad_lane_kernel<C, WPL>: C = fpw / 8 sixteen-byte chunks of 10 or 20 (8 / 16 kHz at 100 windows per
//             second), every non-empty signal starting at a multiple of 8 samples, B2_VAD_LAYOUT not "group"
//   group     vad_energy_zcr_kernel's vector path: G lanes per window, cpl chunks per lane (fpw a multiple of 16,
//             every non-empty signal starting at a multiple of 8 samples)
//   generic   vad_energy_zcr_kernel's 16-bit path: any window size and start (G lanes per window)
// Only where a signal STARTS matters: its end may fall anywhere (a partial last window, or a window cut off by
// pcm_end, is judged on the samples it has).  An empty signal has no tiles, so its start does not matter.
#pragma once

#include <stdint.h>
#include <string.h>

enum VadKernel { kVadLane = 0, kVadGroup = 1, kVadGeneric = 2 };

struct VadLayout {
  int kernel;   // VadKernel
  int G;        // lanes per window (lane-group kernel)
  int cpl;      // 16-byte chunks per lane (vector path), 0 on the 16-bit path
};

constexpr int kVadGroupThreads = 256;   // consumer threads of vad_energy_zcr_kernel

// Signal b spans pcm_off[b] .. pcm_end[b] (pcm_end null: pcm_off[b + 1]); layout_env: B2_VAD_LAYOUT (null: unset).
inline VadLayout vad_layout(const int64_t* pcm_off, const int64_t* pcm_end, int B, int fpw, const char* layout_env) {
  const int C = fpw / 8;
  bool fast = fpw % 8 == 0;
  // lanes per window G: the vector path needs the window's C 16-byte chunks to split evenly over the lanes; prefer
  // an odd chunks-per-lane count (conflict-free LDS.128) and tiles <= 64 KB
  int G = 0, best_score = -1;
  for (int g = 32; g >= 2 && fast; g >>= 1) {
    if (C % g != 0) continue;
    const int cpl = C / g;
    const long long tile = (long long)(kVadGroupThreads / g) * fpw * 2;
    const int score = ((cpl & 1) ? 4 : 0) + (tile <= 65536 ? 2 : 0) + (cpl >= 3 ? 1 : 0);
    if (score > best_score) {
      best_score = score;
      G = g;
    }
  }
  if (G == 0) {   // generic 16-bit path: any window size
    fast = false;
    G = 4;
    if (C > 32) G = 8;
    if (C > 64) G = 16;
    if (C > 128) G = 32;
  }
  for (int b = 0; b < B && fast; ++b) {
    const int64_t end = pcm_end ? pcm_end[b] : pcm_off[b + 1];
    if (end > pcm_off[b] && pcm_off[b] % 8 != 0) fast = false;   // window starts not 16-byte aligned in the span
  }
  if (!fast) return VadLayout{kVadGeneric, G, 0};
  const bool group_env = layout_env && strcmp(layout_env, "group") == 0;
  if ((C == 10 || C == 20) && !group_env) return VadLayout{kVadLane, G, C / G};
  return VadLayout{kVadGroup, G, C / G};
}
