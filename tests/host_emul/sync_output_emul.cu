// CPU run of try_sync's epilogue arithmetic (ffsubsync_b200/csrc/sync_output.cuh): the same
// __host__ __device__ functions apply_sync_kernel calls, one track with one cue time per record.
// Test infrastructure (the build container has no GPU); tests/test_sync_output_cpu.py drives it.
//
// usage: sync_output_emul in.bin out.bin
// in.bin : records of float64 t, ratio, gss_ratio, best_score, apply_offset_seconds, min_score, max_offset_seconds,
//          max_framerate_deviation, suppress_threshold ; int64 best_offset, best_k, sample_rate, gate, has_suppress,
//          has_gss   (the grid is the single ratio: best_k 0 picks it, 1 the search point with has_gss)
// out.bin: records of float64 scale, offset_seconds ; int64 status, shift_us, synced_us, scaled_us (t at the ratio)
#include <stdio.h>
#include <stdint.h>

#include <vector>

#include "../../ffsubsync_b200/csrc/sync_output.cuh"

struct In {
  double t, ratio, gss_ratio, best_score, apply, min_score, max_off, max_dev, suppress;
  int64_t best_offset, best_k, sample_rate, gate, has_suppress, has_gss;
};
struct Out {
  double scale, offset_seconds;
  int64_t status, shift_us, synced_us, scaled_us;
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
    const B2SyncRule rule = b2_sync_rule((int)c.sample_rate, c.apply, (int)c.gate, c.min_score, c.max_off, c.max_dev,
                                         (int)c.has_suppress, c.suppress);
    const B2SyncTrack d = b2_sync_decide(c.best_score, (int)c.best_offset, (int)c.best_k, &c.ratio, 1,
                                         c.has_gss != 0, c.gss_ratio, rule);
    out[i] = Out{d.scale, d.offset_seconds, d.status, d.shift_us, b2_synced_us(c.t, d), b2_scaled_us(c.t, c.ratio)};
  }
  f = fopen(argv[2], "wb");
  if (!f) return 3;
  if (!out.empty() && fwrite(out.data(), sizeof(Out), out.size(), f) != out.size()) return 4;
  fclose(f);
  return 0;
}
