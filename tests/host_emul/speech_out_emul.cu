// CPU run of the speech output (ffsubsync_b200/csrc/speech_out.cuh, speech_out.cu's speech_out_kernel) and of the
// batched sync calls' planner with the output set (csrc/sync_plan.h, SyncPipeEnv::speech_out).  Test infrastructure
// (the build container has no GPU); tests/test_speech_out_cpu.py drives it.
//
// usage: speech_out_emul kernel in.bin out.bin
//   in : int32 n, int64 n_words, then n + 1 int64 off, n times (int64 src, float32 low, int32 packed), then n_words
//        uint32 words of the reference buffer (float32 frames or packed bits)
//   out: off[n] float64 frames, every one written by the kernel's loop nest run thread by thread (tiles of
//        kSpeechTile frames, kSpeechThreads threads, each thread's video found by bisection and then advanced)
// usage: speech_out_emul plan in.txt out.txt
//   in : "name n v0 .. v(n-1)" per line as for seg_ref_emul's plan mode, plus "speech_out 1" (the output is set)
//   out: "status s", "err <message>", then ref_off, cut, ref_packed, trk_off and the video lists
#include <stdio.h>
#include <stdlib.h>

#include <map>
#include <string>
#include <vector>

#include "../../ffsubsync_b200/csrc/speech_out.cuh"
#include "../../ffsubsync_b200/csrc/sync_plan.h"

static int run_kernel(const char* in_path, const char* out_path) {
  FILE* f = fopen(in_path, "rb");
  if (!f) return 3;
  int32_t n;
  int64_t nw;
  if (fread(&n, 4, 1, f) != 1 || fread(&nw, 8, 1, f) != 1) return 3;
  std::vector<long long> off((size_t)n + 1);
  std::vector<B2SpeechVideo> vids((size_t)n + 1);
  if (fread(off.data(), 8, (size_t)n + 1, f) != (size_t)n + 1) return 3;
  for (int i = 0; i < n; ++i) {
    int64_t src;
    float low;
    int32_t packed;
    if (fread(&src, 8, 1, f) != 1 || fread(&low, 4, 1, f) != 1 || fread(&packed, 4, 1, f) != 1) return 3;
    vids[i] = B2SpeechVideo{(long long)src, low, packed};
  }
  std::vector<uint32_t> words((size_t)nw + 1);
  if (nw && fread(words.data(), 4, (size_t)nw, f) != (size_t)nw) return 3;
  fclose(f);
  const float* ref = reinterpret_cast<const float*>(words.data());
  const long long total = n > 0 ? off[n] : 0;
  std::vector<double> out((size_t)total, -12345.0);
  std::vector<uint8_t> hits((size_t)total, 0);
  const long long tiles = (total + kSpeechTile - 1) / kSpeechTile;
  for (long long t = 0; t < tiles; ++t)
    for (int tid = 0; tid < kSpeechThreads; ++tid) {
      long long fr = t * kSpeechTile + tid;
      if (fr >= total) continue;
      int i = b2_speech_video(off.data(), n, fr);
      for (int k = 0; k < (int)(kSpeechTile / kSpeechThreads); ++k, fr += kSpeechThreads) {
        if (fr >= total) break;
        while (off[i + 1] <= fr) ++i;
        out[(size_t)fr] = b2_speech_frame(ref, vids[i], fr - off[i]);
        ++hits[(size_t)fr];
      }
    }
  for (long long fr = 0; fr < total; ++fr)
    if (hits[(size_t)fr] != 1) return 5;   // every frame written exactly once
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
  i64s.reserve(16);
  f64s.reserve(16);
  i32s.reserve(4);
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
  static double x_dummy[1];
  static int32_t i_dummy[1];
  const std::string who = has("who") ? in["who"][0] : "sync_tracks_seg";
  SyncRequest r{};
  r.who = who.c_str();
  r.pcm = pcm_dummy;
  r.pcm_off = arr(i64s, "pcm_off", as_i);
  r.V = (int)in["pcm_off"].size() - 1;
  r.track_video = arr(i32s, "track_video", as_i);
  r.T = (int)in["track_video"].size();
  r.frame_rate = (int)i64("frame_rate", 16000);
  r.sample_rate = (int)i64("sample_rate", 100);
  r.detector = (int)i64("detector", B2_DETECTOR_ENERGY_ZCR);
  r.energy.non_speech_label = (float)f64("label");
  r.energy.z_lo = r.energy.z_hi = -1;
  r.auditok.chunk_samples = i64("chunk_samples");
  r.auditok.non_speech_label = f64("label");
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
  r.sig.is_sig = arr(u8s, "ref_is_sig", as_i);
  r.sig.x = x_dummy;   // the planner never reads the values
  r.sig.off = arr(i64s, "sig_off", as_i);
  r.seg.video = arr(i32s, "seg_video", as_i);
  r.seg.n = has("seg_video") ? (int)in["seg_video"].size() : 0;
  r.seg.total = arr(f64s, "seg_total", as_f);
  r.seg.off = arr(i64s, "seg_off", as_i);
  r.seg.start = arr(i64s, "seg_start", as_i);
  r.seg.lo = arr(i64s, "seg_lo", as_i);
  r.seg.hi = arr(i64s, "seg_hi", as_i);
  r.cue_start_s = arr(f64s, "cue_start", as_f);
  r.cue_end_s = arr(f64s, "cue_end", as_f);
  r.cue_off = arr(i64s, "cue_off", as_i);
  r.ratios = arr(f64s, "ratios", as_f);
  r.K = (int)in["ratios"].size();
  r.start_seconds = f64("start_seconds");
  r.max_offset_samples = 6000;
  r.best_score = d_dummy;
  r.best_offset = r.best_k = i_dummy;
  r.memspace = B2_HOST;
  SyncPipeEnv env{132, b2_ctx::kEvents - 2, nullptr, nullptr, [](const int64_t*, int, int) { return false; }};
  env.speech_out = i64("speech_out") != 0;
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
  put("cut", p.cut);
  put("ref_packed", p.ref_packed);
  put("trk_off", p.trk_off);
  put("sub_video", p.sub_video);
  put("pgs_video", p.pgs_video);
  put("sig_video", p.sig_video);
  put("seg_video", p.seg_video);
  fclose(o);
  return 0;
}

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const std::string mode = argv[1];
  if (mode == "kernel") return run_kernel(argv[2], argv[3]);
  if (mode == "plan") return run_plan(argv[2], argv[3]);
  return 2;
}
