// CPU run of b2_ingest_sync_refs' host half (ffsubsync_b200/csrc/ingest_plan.h and sync_plan.h): a session's pushes
// through IngestStreams and the per-stream IngestPlanner, the pushed-reference-video check, the flush, and plan_sync
// on the request with ingested references (SyncRequest::ready) and the text / PGS / signal tables, as api.cu builds it
// before it launches anything.  Test infrastructure (the build container has no GPU); tests/test_ingest_refs_cpu.py
// drives it.
//
// usage: ingest_refs_emul in.txt out.txt
//   in : one field per line, "name n v0 .. v(n-1)"; a missing array is a null pointer.
//        Scalars: V frame_rate sample_rate detector label chunk_samples start_seconds max_offset_samples gss speech_out
//        lane.  Arrays: push_video push_bytes (one b2_ingest_push chunk each, of push_bytes[i] bytes) seg_video
//        seg_total seg_off seg_start (b2_ingest_segments) track_video cue_start cue_end cue_off ratios ref_is_subs
//        ref_cue_start ref_cue_end ref_cue_off ref_is_pgs pgs_start pgs_end pgs_off ref_is_sig sig_off (the values x
//        are not read: a dummy).
//   out: "status s", "err <message>", then "name n v0 .." for ref_off, sub_video, pgs_video, sig_video, seg_video,
//        ref_packed and "two_level t ref_label".
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <vector>

#include "../../ffsubsync_b200/csrc/ingest_plan.h"

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
  i64s.reserve(16);
  f64s.reserve(16);
  i32s.reserve(8);
  u8s.reserve(8);
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
  FILE* o = fopen(argv[2], "w");
  if (!o) return 4;
  auto done = [&](int st, const std::string& err) {
    fprintf(o, "status %d\nerr %s\n", st, err.c_str());
    fclose(o);
    return 0;
  };

  // b2_ingest_begin: the detector arguments, checked by plan_references on a call without videos
  const int V = (int)i64("V");
  static const int64_t no_pcm[1] = {0};
  SyncRequest det{};
  det.who = "ingest_begin";
  det.pcm_off = no_pcm;
  det.frame_rate = (int)i64("frame_rate", 16000);
  det.sample_rate = (int)i64("sample_rate", 100);
  det.detector = (int)i64("detector", B2_DETECTOR_ENERGY_ZCR);
  const double label = f64("label");
  det.energy = {(float)label, 0, -1, -1};
  det.auditok = {label, 50.0, 20.0, 25.0, 500, i64("chunk_samples")};
  SyncPlan dp;
  dp.auditok = det.detector == B2_DETECTOR_AUDITOK;
  if (const int st = plan_references(det, &dp)) return done(st, dp.err);
  IngestStreams ss;
  ss.begin(V);
  IngestPlanner pl;
  pl.begin(V, dp.fpw, dp.auditok, dp.call, 50.0);
  const int32_t* seg_video = arr(i32s, "seg_video", as_i);
  if (seg_video) {
    const int P = (int)in["seg_video"].size();
    if (const int st = ss.declare(det, P, seg_video, arr(f64s, "seg_total", as_f), arr(i64s, "seg_off", as_i),
                                  arr(i64s, "seg_start", as_i)))
      return done(st, ss.err);
    pl.add_streams(ss.streams() - V);
  }
  std::vector<IngestSpan> spans;
  std::vector<IngestChunk> chunks;
  const int64_t* push_video = arr(i64s, "push_video", as_i);
  const int64_t* push_bytes = arr(i64s, "push_bytes", as_i);
  for (size_t i = 0; push_video && i < in["push_video"].size(); ++i) {
    const int k = ss.route("ingest_push", (int)i, (int)push_video[i], false, 0);
    if (k < 0) return done(B2_ERR_BAD_ARG, ss.err);
    pl.push(k, push_bytes[i], &spans, &chunks);
  }

  // b2_ingest_sync_refs
  SyncRequest r = det;
  const bool gss = i64("gss") != 0;
  r.who = gss ? "ingest_sync_refs (search)" : "ingest_sync_refs";
  r.V = V;
  r.refs = {arr(u8s, "ref_is_subs", as_i), arr(f64s, "ref_cue_start", as_f), arr(f64s, "ref_cue_end", as_f), nullptr,
            V > 0 ? arr(i64s, "ref_cue_off", as_i) : nullptr};
  r.pgs = {arr(u8s, "ref_is_pgs", as_i), arr(f64s, "pgs_start", as_f), arr(f64s, "pgs_end", as_f),
           V > 0 ? arr(i64s, "pgs_off", as_i) : nullptr};
  static double x_dummy[1];
  const int64_t* sig_off = arr(i64s, "sig_off", as_i);
  r.sig = {arr(u8s, "ref_is_sig", as_i), sig_off ? x_dummy : nullptr, V > 0 ? sig_off : nullptr};
  if (const int st = ingest_refs_check(r, &ss, pl)) return done(st, ss.err);
  for (int k = 0; k < ss.streams(); ++k)
    if (ss.live(k)) pl.finish(k, &spans, &chunks);
  // the session's buffer: every stream's frames back to back
  std::vector<int64_t> at(ss.streams(), 0);
  for (int k = 1; k < ss.streams(); ++k) at[k] = at[k - 1] + pl.frames[k - 1];
  const int P = (int)ss.video.size();
  std::vector<int64_t> seg_off(1, 0), seg_start, seg_at, seg_len;
  for (int i = 0; i < P; ++i) {
    for (int64_t j = ss.first[i]; j < ss.first[i + 1]; ++j)
      if (!ss.dropped[j]) {
        seg_start.push_back(ss.start[j]);
        seg_at.push_back(at[V + j]);
        seg_len.push_back(pl.frames[V + j]);
      }
    seg_off.push_back((int64_t)seg_start.size());
  }
  const std::vector<int64_t> no_range(seg_start.size() + 1, 0);
  std::vector<int64_t> pcm_off(V + 1, 0);
  r.pcm = nullptr;
  r.pcm_off = pcm_off.data();
  r.track_video = arr(i32s, "track_video", as_i);
  r.T = has("track_video") ? (int)in["track_video"].size() : 0;
  r.cue_start_s = arr(f64s, "cue_start", as_f);
  r.cue_end_s = arr(f64s, "cue_end", as_f);
  r.cue_off = arr(i64s, "cue_off", as_i);
  r.ratios = arr(f64s, "ratios", as_f);
  r.K = has("ratios") ? (int)in["ratios"].size() : 0;
  r.start_seconds = f64("start_seconds");
  r.max_offset_samples = i64("max_offset_samples", 6000);
  static double d_dummy[1];
  static int32_t i_dummy[1];
  r.best_score = d_dummy;
  r.best_offset = r.best_k = i_dummy;
  r.search = gss;
  r.gss_ratio = gss ? d_dummy : nullptr;
  r.memspace = B2_HOST;
  static float ref_dummy[1];
  r.ready = {ref_dummy, at.data(), pl.frames.data(), seg_at.data(), seg_len.data()};
  if (ss.declared)
    r.seg = {P, ss.video.data(), ss.total.data(), seg_off.data(), seg_start.data(), no_range.data(), no_range.data()};
  g_lane = i64("lane") != 0;
  SyncPipeEnv env{132, b2_ctx::kEvents - 2, nullptr, nullptr, lane_eligible};
  env.speech_out = i64("speech_out") != 0;
  SyncPlan p;
  const int st = plan_sync(r, env, &p);
  fprintf(o, "status %d\nerr %s\n", st, p.err.c_str());
  auto put = [&](const char* k, const auto& v) {
    fprintf(o, "%s", k);
    for (const auto& x : v) fprintf(o, " %lld", (long long)x);
    fprintf(o, "\n");
  };
  put("ref_off", p.ref_off);
  put("sub_video", p.sub_video);
  put("pgs_video", p.pgs_video);
  put("sig_video", p.sig_video);
  put("seg_video", p.seg_video);
  put("ref_packed", p.ref_packed);
  fprintf(o, "two_level %d %.9g\n", (int)p.two_level, (double)p.ref_label);
  fclose(o);
  return 0;
}
