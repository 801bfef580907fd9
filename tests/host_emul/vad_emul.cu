// CPU check of the VAD arithmetic against the plain definition: E = sum x^2, Z = sign changes inside the
// window.  Covers the lane-per-window arithmetic (ffsubsync_b200/csrc/vad_lane.cuh) and the lane-group
// arithmetic (ffsubsync_b200/csrc/vad_group.cuh, G lanes per window summed like the kernel's lane_group_sum)
// for every (chunks per lane, lanes per window) pair the launcher picks.  Test infrastructure (the build
// container has no GPU); prints one line per lane-group pair, then "ok <cases>", or the first mismatches.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../ffsubsync_b200/csrc/vad_group.cuh"
#include "../../ffsubsync_b200/csrc/vad_lane.cuh"

using namespace vadlane;

static uint32_t rng_state = 12345u;
static uint32_t rnd() {
  rng_state ^= rng_state << 13;
  rng_state ^= rng_state >> 17;
  rng_state ^= rng_state << 5;
  return rng_state;
}

constexpr int kModes = 14;

// a sample of the given sign (zero counts as non-negative) and magnitude below amp (<= 32768)
static short signed_sample(bool neg, int amp) {
  return neg ? (short)-(int)(1 + rnd() % amp) : (short)(rnd() % amp);
}

// n_win consecutive windows of fpw samples of family `mode`; `period` is the lane-chunk length in samples
static void fill(short* x, int n_win, int fpw, int mode, int period, int it) {
  for (int w = 0; w < n_win; ++w) {
    short* xs = x + (size_t)w * fpw;
    const int amp = 1 << (rnd() % 16);
    const bool flip = rnd() & 1;
    const int k = 1 + (w + it) % (fpw - 1);
    bool neg = flip;
    for (int i = 0; i < fpw; ++i) {
      const int gi = w * fpw + i;
      short v;
      switch (mode) {
        case 0: v = (short)rnd(); break;                                  // full range
        case 1: v = (short)((rnd() % 7) - 3); break;                      // around zero: many crossings, zeros
        case 2: v = (gi & 1) ? 32767 : -32768; break;                     // extremes, crossing every sample
        case 3: v = -32768; break;                                        // largest energy
        case 4: v = (short)(((gi / 3) & 1) ? -(int)(rnd() % 200) : (int)(rnd() % 200)); break;
        case 5: v = (rnd() & 15) ? 0 : (short)rnd(); break;               // sparse
        case 6: v = (short)((rnd() & 1) ? 255 : -256); break;             // byte boundaries
        case 7: v = signed_sample((w & 1) != flip, amp); break;           // crossings only across windows
        case 8: v = signed_sample((i < k) != flip, amp); break;           // one crossing, at sample k
        case 9: v = signed_sample(((i / period) & 1) != flip, amp); break;   // only at lane-chunk starts
        case 10:                                                          // only at odd indices (inside words)
        case 11:                                                          // only at even indices (across words)
          if (i > 0 && (i & 1) == (mode == 10 ? 1 : 0) && rnd() % 3 == 0) neg = !neg;
          v = signed_sample(neg, amp);
          break;
        case 12: v = (short)((rnd() & 1) ? 0 : -1); break;                // zero is non-negative
        default: {                                                        // lo8 / hi8 split
          static const short b[4] = {255, 256, -256, -257};
          v = b[rnd() & 3];
        }
      }
      xs[i] = v;
    }
  }
}

static void plain(const short* xs, int n, long long& e, int& z) {
  e = 0;
  z = 0;
  for (int i = 0; i < n; ++i) {
    e += (long long)xs[i] * xs[i];
    if (i > 0) z += ((xs[i] < 0) != (xs[i - 1] < 0));
  }
}

template <int C>
static int run(int n_cases, long long* total) {
  constexpr int RMAX = rotation_max(C);
  constexpr int n = 8 * C;
  int bad = 0;
  // tile of 32 windows like the kernel sees it (+ one chunk of slack either side)
  std::vector<unsigned char> raw(16 * C * 32 + 64);
  unsigned char* tile = raw.data() + (16 - ((uintptr_t)raw.data() & 15));
  for (int it = 0; it < n_cases; ++it) {
    short* x = reinterpret_cast<short*>(tile);
    const int mode = it % kModes;
    fill(x, 32, n, mode, 8, it);
    for (int lane = 0; lane < 32; ++lane) {
      const unsigned char* wbase = tile + (size_t)lane * 16 * C;
      long long e_ref;
      int z_ref;
      plain(reinterpret_cast<const short*>(wbase), n, e_ref, z_ref);
      for (int r = 0; r <= RMAX; ++r) {   // every start chunk, not only the lane's own
        long long e;
        int z;
        lane_window<C, RMAX>(wbase, r, e, z);
        ++*total;
        if (e != e_ref || z != z_ref) {
          if (bad < 5)
            printf("mismatch C=%d mode=%d lane=%d r=%d: e %lld vs %lld, z %d vs %d\n", C, mode, lane, r, e, e_ref, z, z_ref);
          ++bad;
        }
      }
      if (lane_rotation(C, lane) > RMAX) {
        printf("rotation out of range C=%d lane=%d\n", C, lane);
        ++bad;
      }
    }
    // bank groups: the 8 lanes of every quarter-warp must hit 8 distinct 16-byte bank groups at every step
    for (int q = 0; q < 4; ++q)
      for (int c = 0; c < C; ++c) {
        unsigned seen = 0;
        for (int l = 0; l < 8; ++l) {
          const int lane = 8 * q + l, r = lane_rotation(C, lane);
          const int k = (c + r) % C;
          const int grp = (lane * C + k) & 7;
          seen |= 1u << grp;
        }
        if (seen != 0xffu) {
          if (bad < 5) printf("bank conflict C=%d quarter=%d step=%d mask=%02x\n", C, q, c, seen);
          ++bad;
        }
      }
  }
  return bad;
}

// Lane-group arithmetic for windows of G lanes x cpl chunks; CPLT > 0 is the kernel's compile-time
// instantiation (16 and 48 kHz), CPLT = 0 its runtime chunk count.
template <int CPLT>
static int run_group(int cpl, int G, int n_cases, long long* total) {
  const int fpw = 8 * cpl * G;
  constexpr int kWin = 8;
  int bad = 0;
  long long n_win = 0;
  std::vector<unsigned char> raw((size_t)16 * cpl * G * kWin + 64);
  unsigned char* tile = raw.data() + (16 - ((uintptr_t)raw.data() & 15));
  for (int it = 0; it < n_cases; ++it) {
    short* x = reinterpret_cast<short*>(tile);
    const int mode = it % kModes;
    fill(x, kWin, fpw, mode, 8 * cpl, it);
    for (int w = 0; w < kWin; ++w) {
      const unsigned char* wbase = tile + (size_t)w * fpw * 2;
      long long e_ref;
      int z_ref;
      plain(reinterpret_cast<const short*>(wbase), fpw, e_ref, z_ref);
      long long e = 0;
      int z = 0;
      for (int g = 0; g < G; ++g) {   // lane_group_sum: the lanes' partial sums add up
        long long eg = 0;
        int zg = 0;
        vadgroup::window_part_fast<CPLT>(wbase, g, cpl, eg, zg);
        e += eg;
        z += zg;
      }
      ++n_win;
      if (e != e_ref || z != z_ref) {
        if (bad < 5)
          printf("mismatch group CPL=%d G=%d mode=%d window=%d: e %lld vs %lld, z %d vs %d\n", cpl, G, mode, w, e,
                 e_ref, z, z_ref);
        ++bad;
      }
    }
  }
  *total += n_win;
  printf("group CPL=%d%s G=%d fpw=%d: %lld windows, %d mismatches\n", cpl, CPLT > 0 ? " (compile-time)" : "", G, fpw,
         n_win, bad);
  return bad;
}

int main(int argc, char** argv) {
  const int n_cases = argc > 1 ? atoi(argv[1]) : 70;
  long long total = 0;
  int bad = 0;
  bad += run<5>(n_cases, &total);     //  4 kHz
  bad += run<10>(n_cases, &total);    //  8 kHz
  bad += run<15>(n_cases, &total);    // 12 kHz
  bad += run<20>(n_cases, &total);    // 16 kHz
  bad += run<30>(n_cases, &total);    // 24 kHz
  bad += run<40>(n_cases, &total);    // 32 kHz
  bad += run<60>(n_cases, &total);    // 48 kHz
  // the (CPL, G) pairs b2i_vad_launch picks for 16-byte aligned batches the lane-per-window kernel does not take
  bad += run_group<5>(5, 4, n_cases, &total);      // 16 kHz (B2_VAD_LAYOUT=group)
  bad += run_group<15>(15, 4, n_cases, &total);    // 48 kHz
  bad += run_group<0>(5, 2, n_cases, &total);      //  8 kHz (B2_VAD_LAYOUT=group)
  bad += run_group<0>(15, 2, n_cases, &total);     // 24 kHz
  bad += run_group<0>(5, 8, n_cases, &total);      // 32 kHz
  bad += run_group<0>(15, 8, n_cases, &total);     // 96 kHz
  bad += run_group<0>(1, 32, n_cases, &total);     // 25.6 kHz
  bad += run_group<0>(17, 2, n_cases, &total);     // 27.2 kHz: the 32-bit partial sums are flushed every 16 chunks
  if (bad) {
    printf("FAILED %d\n", bad);
    return 1;
  }
  printf("ok %lld\n", total);
  return 0;
}
