// CPU run of the rasterisers' cue arithmetic (ffsubsync_b200/csrc/raster_math.cuh): the same
// __host__ __device__ functions raster_cues_kernel and raster_bits_kernel call, record by record.
// Test infrastructure (the build container has no GPU); tests/test_raster_cpu.py drives it.
//
// usage: raster_emul in.bin out.bin
// in.bin : records of float64 start, end, ratio, start_seconds ; int64 sample_rate, n
// out.bin: records of float64 scaled start, scaled end ; int64 first, last (after slice clamping)
#include <stdio.h>
#include <stdint.h>

#include <vector>

#include "../../ffsubsync_b200/csrc/raster_math.cuh"

struct In {
  double start, end, ratio, start_seconds;
  int64_t sample_rate, n;
};
struct Out {
  double scaled_start, scaled_end;
  int64_t first, last;
};

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "rb");
  if (!f) return 3;
  std::vector<In> in;
  In r;
  while (fread(&r, sizeof(In), 1, f) == 1) in.push_back(r);
  fclose(f);
  std::vector<Out> out(in.size());
  for (size_t i = 0; i < in.size(); ++i) {
    const In& c = in[i];
    long long first, last;
    b2_cue_bounds(c.start, c.end, c.ratio, c.start_seconds, (int)c.sample_rate, c.n, first, last);
    out[i] = Out{b2_scaled_seconds(c.start, c.ratio), b2_scaled_seconds(c.end, c.ratio), first, last};
  }
  f = fopen(argv[2], "wb");
  if (!f) return 3;
  if (!out.empty() && fwrite(out.data(), sizeof(Out), out.size(), f) != out.size()) return 4;
  fclose(f);
  return 0;
}
