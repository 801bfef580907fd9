// CPU run of the PGS reference arithmetic (ffsubsync_b200/csrc/raster_math.cuh b2_pgs_bounds / b2_pgs_length) and of
// the batched sync calls' planner with PGS references (csrc/sync_plan.h).  Test infrastructure (the build container
// has no GPU); tests/test_pgs_ref_cpu.py drives it.
//
// usage: pgs_emul bounds in.bin out.bin
//   in : int64 count, int32 sample_rate, int64 n, then count x (start, end, start_seconds) float64
//   out: count x (first, last, b2_pgs_length(end)) int64
// usage: pgs_emul plan in.txt out.txt
//   in : "name n v0 .. v(n-1)" per line as for plan_emul; arrays pcm_off track_video cue_start cue_end cue_off
//        ratios ref_is_subs ref_cue_start ref_cue_end ref_cue_off ref_is_pgs pgs_start pgs_end pgs_off, scalars
//        who sample_rate detector label auditok_label start_seconds gss lane
//   out: "status s", "err <message>", then the plan's reference tables
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <vector>

#include "../../ffsubsync_b200/csrc/sync_plan.h"

static bool g_lane = false;
static bool lane_eligible(const int64_t*, int, int) { return g_lane; }

static int run_bounds(const char* in_path, const char* out_path) {
  FILE* f = fopen(in_path, "rb");
  if (!f) return 3;
  int64_t count, n;
  int32_t sr;
  if (fread(&count, 8, 1, f) != 1 || fread(&sr, 4, 1, f) != 1 || fread(&n, 8, 1, f) != 1) return 3;
  std::vector<double> t((size_t)count * 3);
  if (fread(t.data(), 8, t.size(), f) != t.size()) return 3;
  fclose(f);
  std::vector<int64_t> out((size_t)count * 3);
  for (int64_t i = 0; i < count; ++i) {
    long long first, last;
    b2_pgs_bounds(t[3 * i], t[3 * i + 1], t[3 * i + 2], sr, n, first, last);
    out[3 * i] = first;
    out[3 * i + 1] = last;
    out[3 * i + 2] = b2_pgs_length(t[3 * i + 1], sr);
  }
  FILE* o = fopen(out_path, "wb");
  if (!o) return 4;
  fwrite(out.data(), 8, out.size(), o);
  fclose(o);
  return 0;
}

static int run_plan(const char* in_path, const char* out_path) {
  FILE* f = fopen(in_path, "r");
  if (!f) return 3;
  std::map<std::string, std::vector<std::string>> in;
  char name[64];
  long n;
  while (fscanf(f, "%63s %ld", name, &n) == 2) {
    std::vector<std::string>& v = in[name];
    char tok[512];
    for (long i = 0; i < n && fscanf(f, "%511s", tok) == 1; ++i) v.push_back(tok);
  }
  fclose(f);
  std::vector<std::vector<int64_t>> i64s;
  std::vector<std::vector<double>> f64s;
  std::vector<std::vector<int32_t>> i32s;
  std::vector<std::vector<uint8_t>> u8s;
  i64s.reserve(8);
  f64s.reserve(8);
  i32s.reserve(2);
  u8s.reserve(4);
  auto has = [&](const char* k) { return in.count(k) != 0; };
  auto i64 = [&](const char* k, int64_t d = 0) { return has(k) ? strtoll(in[k][0].c_str(), nullptr, 10) : d; };
  auto f64 = [&](const char* k, double d = 0.0) { return has(k) ? strtod(in[k][0].c_str(), nullptr) : d; };
  auto arr = [&](auto& store, const char* k, auto conv) -> decltype(store.back().data()) {
    if (!has(k)) return nullptr;
    store.emplace_back();
    for (const std::string& s : in[k]) store.back().push_back(conv(s));
    store.back().push_back({});
    return store.back().data();
  };
  auto as_i = [](const std::string& s) { return strtoll(s.c_str(), nullptr, 10); };
  auto as_f = [](const std::string& s) { return strtod(s.c_str(), nullptr); };
  static int16_t pcm_dummy[8];
  static double d_dummy[1];
  static int32_t i_dummy[1];
  const std::string who = has("who") ? in["who"][0] : "sync_tracks_pgs";
  SyncRequest r{};
  r.who = who.c_str();
  r.pcm = pcm_dummy;
  r.pcm_off = arr(i64s, "pcm_off", as_i);
  r.V = (int)in["pcm_off"].size() - 1;
  r.track_video = arr(i32s, "track_video", as_i);
  r.T = (int)in["track_video"].size();
  r.frame_rate = 16000;
  r.sample_rate = (int)i64("sample_rate", 100);
  r.detector = (int)i64("detector", B2_DETECTOR_ENERGY_ZCR);
  r.energy.non_speech_label = (float)f64("label");
  r.energy.z_lo = r.energy.z_hi = -1;
  r.auditok.non_speech_label = f64("auditok_label");
  r.auditok.energy_threshold_db = 50.0;
  r.auditok.min_length = 20.0;
  r.auditok.max_length = 500;
  r.auditok.max_continuous_silence = 25.0;
  r.refs.is_subs = arr(u8s, "ref_is_subs", as_i);
  r.refs.cue_start_s = arr(f64s, "ref_cue_start", as_f);
  r.refs.cue_end_s = arr(f64s, "ref_cue_end", as_f);
  r.refs.cue_off = arr(i64s, "ref_cue_off", as_i);
  r.pgs.is_pgs = arr(u8s, "ref_is_pgs", as_i);
  r.pgs.start_s = arr(f64s, "pgs_start", as_f);
  r.pgs.end_s = arr(f64s, "pgs_end", as_f);
  r.pgs.off = arr(i64s, "pgs_off", as_i);
  r.cue_start_s = arr(f64s, "cue_start", as_f);
  r.cue_end_s = arr(f64s, "cue_end", as_f);
  r.cue_off = arr(i64s, "cue_off", as_i);
  r.ratios = arr(f64s, "ratios", as_f);
  r.K = (int)in["ratios"].size();
  r.start_seconds = f64("start_seconds");
  r.max_offset_samples = 6000;
  r.best_score = d_dummy;
  r.best_offset = r.best_k = i_dummy;
  r.search = i64("gss") != 0;
  r.gss_ratio = r.search ? d_dummy : nullptr;
  r.memspace = B2_HOST;
  g_lane = i64("lane") != 0;
  SyncPipeEnv env{132, b2_ctx::kEvents - 2, nullptr, nullptr, lane_eligible};
  SyncPlan p;
  const int st = plan_sync(r, env, &p);
  FILE* o = fopen(out_path, "w");
  if (!o) return 4;
  fprintf(o, "status %d\nerr %s\n", st, p.err.c_str());
  auto put = [&](const char* k, const auto& v) {
    fprintf(o, "%s", k);
    for (const auto& x : v) fprintf(o, " %lld", (long long)x);
    fprintf(o, "\n");
  };
  put("ref_off", p.ref_off);
  put("sub_video", p.sub_video);
  put("pgs_video", p.pgs_video);
  put("ch_out", p.ch.out);
  put("tok_off", p.ch.tok_off);
  put("ref_packed", p.ref_packed);
  put("audio_samples", std::vector<int64_t>{p.audio_samples});
  fprintf(o, "two_level %d %.9g\n", (int)p.two_level, (double)p.ref_label);
  fclose(o);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const std::string mode = argv[1];
  if (mode == "bounds") return run_bounds(argv[2], argv[3]);
  if (mode == "plan") return run_plan(argv[2], argv[3]);
  return 2;
}
