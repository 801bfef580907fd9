// CPU run of the sampled-segment reference (ffsubsync_b200/csrc/seg_ref.cuh, seg_ref.cu's seg_ref_kernel) and of
// the batched sync calls' planner with segment references (csrc/sync_plan.h).  Test infrastructure (the build
// container has no GPU); tests/test_seg_ref_cpu.py drives it.
//
// usage: seg_ref_emul kernel in.bin out.bin
//   in : int64 L, int64 n_runs, int64 n_scratch, int32 packed, then n_runs int64 run_lo, n_runs int64 run_src and
//        n_scratch float32 scratch frames
//   out: int64 first frame > 0 (-1: none), then L float32 frames, or ceil(L/32) uint32 words when packed
//   The kernel's loop nest run thread by thread: chunks of kSegChunkFrames, warps of kSegUnits units of 32 lanes, each
//   lane's run found by bisection and then advanced, every ballot built from the lanes' predicates.
// usage: seg_ref_emul plan in.txt out.txt
//   in : "name n v0 .. v(n-1)" per line as for sig_ref_emul, plus seg_video seg_total seg_off seg_start seg_lo seg_hi
//        and the scalars frame_rate chunk_samples; "lane 3" takes the library's own lane test (vad_layout.h, reading
//        B2_VAD_LAYOUT from the environment as the library does)
//   out: "status s", "err <message>", then the plan's reference and segment tables, and "seg_kernel k G cpl": the
//        energy kernel (vad_layout.h VadKernel) the segments' detector launch takes, with its lanes per window
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../ffsubsync_b200/csrc/seg_ref.cuh"
#include "../../ffsubsync_b200/csrc/sig_ref.cuh"
#include "../../ffsubsync_b200/csrc/sync_plan.h"
#include "../../ffsubsync_b200/csrc/vad_layout.h"

static int g_lane = 0;
static bool lane_eligible(const int64_t* off, int n, int fpw) {
  // "lane" 1: every table eligible; 2: eligible when every non-empty range starts at a multiple of 8; 3: the
  // library's test (b2i_vad_lane_eligible)
  if (g_lane == 3) return vad_layout(off, nullptr, n, fpw, getenv("B2_VAD_LAYOUT")).kernel == kVadLane;
  if (!g_lane) return false;
  for (int b = 0; b < n; ++b)
    if (off[b + 1] > off[b] && off[b] % 8 != 0 && g_lane > 1) return false;
  return true;
}

static int run_kernel(const char* in_path, const char* out_path) {
  FILE* f = fopen(in_path, "rb");
  if (!f) return 3;
  int64_t L, nr, ns;
  int32_t packed;
  if (fread(&L, 8, 1, f) != 1 || fread(&nr, 8, 1, f) != 1 || fread(&ns, 8, 1, f) != 1 || fread(&packed, 4, 1, f) != 1)
    return 3;
  std::vector<long long> lo((size_t)nr + 1), src((size_t)nr + 1);
  std::vector<float> scr((size_t)ns + 1);
  if ((nr && (fread(lo.data(), 8, (size_t)nr, f) != (size_t)nr || fread(src.data(), 8, (size_t)nr, f) != (size_t)nr)) ||
      (ns && fread(scr.data(), 4, (size_t)ns, f) != (size_t)ns))
    return 3;
  fclose(f);
  std::vector<float> frames((size_t)L, -12345.0f);
  std::vector<uint32_t> words((size_t)((L + 31) / 32), 0xdeadbeefu);
  unsigned long long speech = kSigNoBadFrame;
  const long long chunks = (L + kSegChunkFrames - 1) / kSegChunkFrames;
  const int r1 = (int)nr;
  for (long long c = 0; c < chunks; ++c)
    for (int warp = 0; warp < kSegThreads / 32; ++warp) {
      const long long f0 = c * kSegChunkFrames + (long long)warp * (kSegUnits * 32);
      if (f0 >= L) continue;
      int r[32];
      for (int lane = 0; lane < 32; ++lane) {   // bisection for the lane's first frame
        int a = 0, b = r1 - 1;
        while (a < b) {
          const int mid = (a + b + 1) >> 1;
          if (lo[mid] <= f0 + lane) a = mid;
          else b = mid - 1;
        }
        r[lane] = a;
      }
      long long speech_at = -1;
      for (int u = 0; u < kSegUnits; ++u) {
        uint32_t pos = 0, word = 0;
        for (int lane = 0; lane < 32; ++lane) {
          const long long fr = f0 + u * 32 + lane;
          const bool in = fr < L;
          float v = 0.0f;
          if (in) {
            r[lane] = b2_seg_run(lo.data(), r[lane], r1, fr);
            v = b2_seg_frame(scr.data(), lo.data(), src.data(), r[lane], fr);
          }
          if (in && v > 0.0f) pos |= 1u << lane;
          if (in && v == 1.0f) word |= 1u << lane;
          if (!packed && in) frames[(size_t)fr] = v;
        }
        if (pos && speech_at < 0) speech_at = f0 + u * 32 + __builtin_ctz(pos);
        if (packed && f0 + u * 32 < L) words[(size_t)((f0 >> 5) + u)] = word;
      }
      if (speech_at >= 0) speech = std::min(speech, (unsigned long long)speech_at);
    }
  FILE* o = fopen(out_path, "wb");
  if (!o) return 4;
  const int64_t sp = speech == kSigNoBadFrame ? -1 : (int64_t)speech;
  fwrite(&sp, 8, 1, o);
  if (packed) fwrite(words.data(), 4, words.size(), o);
  else fwrite(frames.data(), 4, frames.size(), o);
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
  r.sig.is_sig = arr(u8s, "ref_is_sig", as_i);
  r.sig.x = i64("x_null") ? nullptr : x_dummy;   // the planner never reads the values
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
  r.search = i64("gss") != 0;
  r.gss_ratio = r.search ? d_dummy : nullptr;
  r.memspace = B2_HOST;
  g_lane = (int)i64("lane");
  const std::string subbatches = has("subbatches") ? in["subbatches"][0] : "";
  SyncPipeEnv env{132, b2_ctx::kEvents - 2, has("subbatches") ? subbatches.c_str() : nullptr, nullptr, lane_eligible};
  const std::string ref_packed = has("ref_packed") ? in["ref_packed"][0] : "";
  if (has("ref_packed")) env.ref_packed = ref_packed.c_str();
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
  put("sig_video", p.sig_video);
  put("ch_out", p.ch.out);
  put("ch_first", p.ch.first);
  put("tok_off", p.ch.tok_off);
  put("cut", p.cut);
  put("trk_off", p.trk_off);
  put("sub_off", p.sub_off);
  put("ref_packed", p.ref_packed);
  put("audio_samples", std::vector<int64_t>{p.audio_samples});
  put("seg_video", p.seg_video);
  put("det_end", p.det_end);
  put("item_start", p.item_start);
  put("item_end", p.item_end);
  put("item_out", p.item_out);
  put("item_tail", p.item_tail);
  put("item_first", p.item_first);
  put("run_first", p.run_first);
  put("run_lo", p.run_lo);
  put("run_src", p.run_src);
  put("stage_lo", p.stage_lo);
  put("stage_hi", p.stage_hi);
  put("n_sub", std::vector<int>{p.n_sub});
  fprintf(o, "two_level %d %.9g\n", (int)p.two_level, (double)p.ref_label);
  if (st == 0 && p.fpw > 0) {   // the segments' detector launch: b2i_vad_launch over item_start / item_end
    const VadLayout lay = vad_layout(p.item_start.data(), p.item_end.data(), (int)p.item_end.size(), p.fpw,
                                     getenv("B2_VAD_LAYOUT"));
    fprintf(o, "seg_kernel %d %d %d\n", lay.kernel, lay.G, lay.cpl);
  }
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
