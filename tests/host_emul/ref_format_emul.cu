// CPU run of the batched sync calls' planner (ffsubsync_b200/csrc/sync_plan.h) for the reference format: which
// sub-batches have their VAD write the reference as packed bits (plan_ref_format, with the aligner's own path
// choice from align_path.h).  Test infrastructure (the build container has no GPU); tests/test_ref_packed_cpu.py
// drives it.  The request is read as plan_emul.cu reads it, with the aligner's environment on top.
//
// usage: ref_format_emul in.txt out.txt
//   in : one field of the request per line, "name n v0 .. v(n-1)"; a missing array is a null pointer.
//        Arrays: pcm_off track_video cue_start cue_end cue_off ratios ref_is_subs ref_cue_start ref_cue_end
//        ref_cue_off.  Scalars (n = 1): who frame_rate sample_rate detector label energy_threshold z_lo z_hi
//        auditok_label energy_threshold_db min_length max_length max_continuous_silence chunk_samples
//        start_seconds max_offset_samples outputs (1: best_* given) all (1: all_* given) gss (1: the search
//        runs) gss_ratio (1: given; default: gss) pcm (1: pcm given) sm_count subbatches vad_sms (as the
//        environment strings) lane (the lane kernel's eligibility) align_path ref_packed (as the environment
//        strings) capture (1: a nominations capture is on) fused (0: float subtitle signals).
//   out: "status s", "err <message>", the tables the reference format is decided on, and "ref_packed" (one flag
//        per sub-batch).
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <vector>

#include "../../ffsubsync_b200/csrc/sync_plan.h"

static bool g_lane = false;
static bool lane_eligible(const int64_t*, int, int) { return g_lane; }

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "r");
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
  auto has = [&](const char* k) { return in.count(k) != 0; };
  auto i64 = [&](const char* k, int64_t d = 0) { return has(k) ? strtoll(in[k][0].c_str(), nullptr, 10) : d; };
  auto f64 = [&](const char* k, double d = 0.0) { return has(k) ? strtod(in[k][0].c_str(), nullptr) : d; };
  auto arr = [&](auto& store, const char* k, auto conv) -> decltype(store.back().data()) {
    if (!has(k)) return nullptr;
    store.emplace_back();
    for (const std::string& s : in[k]) store.back().push_back(conv(s));
    store.back().push_back({});   // one spare element: an empty array is still not null
    return store.back().data();
  };
  auto as_i = [](const std::string& s) { return strtoll(s.c_str(), nullptr, 10); };
  auto as_f = [](const std::string& s) { return strtod(s.c_str(), nullptr); };
  i64s.reserve(8);
  f64s.reserve(8);
  i32s.reserve(2);
  u8s.reserve(2);
  static int16_t pcm_dummy[8];
  static double d_dummy[1];
  static int32_t i_dummy[1];
  const std::string who = has("who") ? in["who"][0] : "sync_tracks";
  const int64_t* pcm_off = arr(i64s, "pcm_off", as_i);
  const int64_t* cue_off = arr(i64s, "cue_off", as_i);
  const int64_t* ref_cue_off = arr(i64s, "ref_cue_off", as_i);
  const int32_t* track_video = arr(i32s, "track_video", as_i);
  const bool outputs = i64("outputs", 1) != 0, all = i64("all") != 0;
  SyncRequest r{};
  r.who = who.c_str();
  r.pcm = i64("pcm", 1) ? pcm_dummy : nullptr;
  r.pcm_off = pcm_off;
  r.V = has("pcm_off") ? (int)in["pcm_off"].size() - 1 : (int)i64("V");
  r.track_video = track_video;
  r.T = has("cue_off") ? (int)in["cue_off"].size() - 1 : (int)i64("T");
  if (track_video) r.T = (int)in["track_video"].size();
  r.frame_rate = (int)i64("frame_rate", 16000);
  r.sample_rate = (int)i64("sample_rate", 100);
  r.detector = (int)i64("detector", B2_DETECTOR_ENERGY_ZCR);
  r.energy.non_speech_label = (float)f64("label");
  r.energy.energy_threshold = i64("energy_threshold");
  r.energy.z_lo = (int)i64("z_lo", -1);
  r.energy.z_hi = (int)i64("z_hi", -1);
  r.auditok.non_speech_label = f64("auditok_label");
  r.auditok.energy_threshold_db = f64("energy_threshold_db", 50.0);
  r.auditok.min_length = f64("min_length", 20.0);
  r.auditok.max_length = i64("max_length", 500);
  r.auditok.max_continuous_silence = f64("max_continuous_silence", 25.0);
  r.auditok.chunk_samples = i64("chunk_samples");
  r.refs.is_subs = arr(u8s, "ref_is_subs", as_i);
  r.refs.cue_start_s = arr(f64s, "ref_cue_start", as_f);
  r.refs.cue_end_s = arr(f64s, "ref_cue_end", as_f);
  r.refs.cue_off = ref_cue_off;
  r.cue_start_s = arr(f64s, "cue_start", as_f);
  r.cue_end_s = arr(f64s, "cue_end", as_f);
  r.cue_off = cue_off;
  r.ratios = arr(f64s, "ratios", as_f);
  r.K = has("ratios") ? (int)in["ratios"].size() : 0;
  r.start_seconds = f64("start_seconds");
  r.max_offset_samples = i64("max_offset_samples", 6000);
  r.best_score = outputs ? d_dummy : nullptr;
  r.best_offset = r.best_k = outputs ? i_dummy : nullptr;
  r.all_score = all ? d_dummy : nullptr;
  r.all_offset = all ? i_dummy : nullptr;
  r.search = i64("gss") != 0;
  r.gss_ratio = i64("gss_ratio", r.search) ? d_dummy : nullptr;
  r.memspace = B2_HOST;
  g_lane = i64("lane") != 0;
  const std::string subbatches = has("subbatches") ? in["subbatches"][0] : "";
  const std::string vad_sms = has("vad_sms") ? in["vad_sms"][0] : "";
  SyncPipeEnv env{(int)i64("sm_count", 132), b2_ctx::kEvents - 2,
                  has("subbatches") ? subbatches.c_str() : nullptr, has("vad_sms") ? vad_sms.c_str() : nullptr,
                  lane_eligible};
  const std::string align_path = has("align_path") ? in["align_path"][0] : "";
  const std::string ref_packed = has("ref_packed") ? in["ref_packed"][0] : "";
  env.align_path = has("align_path") ? align_path.c_str() : nullptr;
  env.ref_packed = has("ref_packed") ? ref_packed.c_str() : nullptr;
  env.capture = i64("capture") != 0;
  env.fused = i64("fused", 1) != 0;
  SyncPlan p;
  const int st = plan_sync(r, env, &p);
  FILE* o = fopen(argv[2], "w");
  if (!o) return 4;
  fprintf(o, "status %d\nerr %s\n", st, p.err.c_str());
  auto put = [&](const char* k, const auto& v) {
    fprintf(o, "%s", k);
    for (const auto& x : v) fprintf(o, " %lld", (long long)x);
    fprintf(o, "\n");
  };
  put("cut", p.cut);
  put("trk_off", p.trk_off);
  put("ref_off", p.ref_off);
  put("sub_off", p.sub_off);
  put("ref_packed", p.ref_packed);
  fprintf(o, "two_level %d %.9g\n", (int)p.two_level, (double)p.ref_label);
  fclose(o);
  return 0;
}
