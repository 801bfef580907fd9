// CPU run of the GSS rounds' host-and-device arithmetic (ffsubsync_b200/csrc/job_plan.cuh, raster_math.cuh):
// the same __host__ __device__ functions gss_step_kernel and b2i_align_launch call.  Test infrastructure (the
// build container has no GPU); tests/test_gss_sync_cpu.py drives it.
//
// usage: gss_emul MODE in.bin out.bin
//   step : in  int64 lanes, n; float64 lo, hi; then per lane n + 1 float64 scores (round r's score)
//          out float64 invphi, invphi2; int64 kGssEvals; then per lane n + 1 points, final lo, hi
//   plan : in  records int64 R, S, max_offset_samples, quirk_mask
//          out records int64 kind, N, lo, hi, o_lo, o_hi, masked_offset
//   len  : in  records float64 max_end, ratio; int64 sample_rate
//          out int64 length per record
#include <stdio.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../ffsubsync_b200/csrc/job_plan.cuh"

template <class T>
static std::vector<T> read_all(const char* path) {
  std::vector<T> v;
  FILE* f = fopen(path, "rb");
  if (!f) return v;
  T r;
  while (fread(&r, sizeof(T), 1, f) == 1) v.push_back(r);
  fclose(f);
  return v;
}

template <class T>
static int write_all(const char* path, const std::vector<T>& v) {
  FILE* f = fopen(path, "wb");
  if (!f) return 3;
  if (!v.empty() && fwrite(v.data(), sizeof(T), v.size(), f) != v.size()) return 4;
  fclose(f);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const char* mode = argv[1];
  if (!strcmp(mode, "step")) {
    const std::vector<double> in = read_all<double>(argv[2]);
    if (in.size() < 4) return 5;
    long long lanes, n;
    memcpy(&lanes, &in[0], 8);
    memcpy(&n, &in[1], 8);
    const double lo = in[2], hi = in[3];
    std::vector<double> out{kGssInvPhi, kGssInvPhi2, 0.0};
    const long long ev = kGssEvals;
    memcpy(&out[2], &ev, 8);
    for (long long l = 0; l < lanes; ++l) {
      const double* sc = &in[4 + l * (n + 1)];
      B2GssLane s;
      for (long long r = 0; r <= n; ++r)   // the objective is the negated score, as in gss_step_kernel
        out.push_back(b2_gss_step(s, (int)r, r > 0 ? -sc[r - 1] : 0.0, lo, hi));
      double a, b;
      b2_gss_finish(s, -sc[n], a, b);
      out.push_back(a);
      out.push_back(b);
    }
    return write_all(argv[3], out);
  }
  if (!strcmp(mode, "plan")) {
    struct In { long long R, S, mo; uint64_t mask; };
    struct Out { long long kind, N, lo, hi, o_lo, o_hi, masked_offset; };
    const std::vector<In> in = read_all<In>(argv[2]);
    std::vector<Out> out;
    for (const In& c : in) {
      const B2JobPlan p = b2_plan_job(c.R, c.S, c.mo, c.mask);
      out.push_back(Out{p.kind, p.N, p.lo, p.hi, p.o_lo, p.o_hi, p.masked_offset});
    }
    return write_all(argv[3], out);
  }
  if (!strcmp(mode, "len")) {
    struct In { double max_end, ratio; long long sample_rate; };
    const std::vector<In> in = read_all<In>(argv[2]);
    std::vector<long long> out;
    for (const In& c : in) out.push_back(b2_signal_length(c.max_end, c.ratio, (int)c.sample_rate));
    return write_all(argv[3], out);
  }
  return 2;
}
