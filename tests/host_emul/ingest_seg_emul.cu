// CPU run of the batched ingest session's streams with sampled segments (ffsubsync_b200/csrc/ingest_plan.h): the
// IngestStreams routing and refusals of b2_ingest_segments / _push / _push_segments / _drop_segment, and the
// per-stream IngestPlanner they feed, as api.cu runs them before it stages anything.  Test infrastructure (the build
// container has no GPU); tests/test_ingest_seg_cpu.py drives it.
//
// usage: ingest_seg_emul in.txt out.txt
//   in : "V fpw auditok chunk_samples energy_threshold_db sample_rate", then one operation per line:
//        "S P video_0 .. total_0 .. off_0 .. off_P start_0 .." (b2_ingest_segments), "p n v_0 nb_0 .. v_n-1 nb_n-1"
//        (b2_ingest_push), "q n v_0 j_0 nb_0 .." (b2_ingest_push_segments), "d v j" (b2_ingest_drop_segment) or "f"
//        (the sync's flush of every live stream).
//   out: per operation "op i status", "e message" when refused, its spans "s stream s0 s1 frame tail" and completed
//        detector calls "c stream f0 f1", then "w" and every video's windows; at the end "streams N" and per stream
//        "k live frames".
#include <stdio.h>

#include "../../ffsubsync_b200/csrc/ingest_plan.h"

template <class T>
static bool read_all(FILE* f, const char* fmt, std::vector<T>* x) {
  for (auto& e : *x)
    if (fscanf(f, fmt, &e) != 1) return false;
  return true;
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "r");
  if (!f) return 3;
  int V, fpw, auditok, sr;
  long long chunk;
  double db;
  if (fscanf(f, "%d %d %d %lld %lf %d", &V, &fpw, &auditok, &chunk, &db, &sr) != 6) return 4;
  FILE* o = fopen(argv[2], "w");
  if (!o) return 5;
  SyncRequest det{};
  det.sample_rate = sr;
  det.frame_rate = sr * fpw;
  IngestStreams st;
  st.begin(V);
  IngestPlanner pl;
  pl.begin(V, fpw, auditok != 0, chunk, db);
  char op[8];
  int i = 0;
  while (fscanf(f, "%7s", op) == 1) {
    std::vector<IngestSpan> spans;
    std::vector<IngestChunk> chunks;
    int status = 0;
    std::string msg;
    if (op[0] == 'S') {
      int P;
      if (fscanf(f, "%d", &P) != 1) return 6;
      std::vector<int32_t> vid(P);
      std::vector<double> tot(P);
      std::vector<int64_t> off(P + 1);
      std::vector<long long> off_in(P + 1);
      if (!read_all(f, "%d", &vid) || !read_all(f, "%lf", &tot) || !read_all(f, "%lld", &off_in)) return 10;
      off.assign(off_in.begin(), off_in.end());
      std::vector<long long> start(off[P] > off[0] ? off[P] - off[0] : 0);
      if (!read_all(f, "%lld", &start)) return 11;
      status = st.declare(det, P, vid.data(), tot.data(), off.data(), (const int64_t*)start.data() - off[0]);
      if (status) msg = st.err;
      else pl.add_streams(st.streams() - V);
    } else if (op[0] == 'p' || op[0] == 'q') {
      const bool seg = op[0] == 'q';
      int n;
      if (fscanf(f, "%d", &n) != 1) return 7;
      std::vector<int> vid(n), k(n);
      std::vector<long long> j(n, 0), nb(n);
      for (int c = 0; c < n; ++c) {
        if (fscanf(f, "%d", &vid[c]) != 1 || (seg && fscanf(f, "%lld", &j[c]) != 1) || fscanf(f, "%lld", &nb[c]) != 1)
          return 8;
      }
      for (int c = 0; c < n && !status; ++c) {   // every chunk is routed before any is pushed, as api.cu does
        k[c] = st.route(seg ? "ingest_push_segments" : "ingest_push", c, vid[c], seg, j[c]);
        if (k[c] < 0) {
          status = 1;
          msg = st.err;
        }
      }
      for (int c = 0; c < n && !status; ++c) st.touched[vid[c]] = 1;
      for (int c = 0; c < n && !status; ++c) pl.push(k[c], nb[c], &spans, &chunks);
    } else if (op[0] == 'd') {
      int v;
      long long j;
      if (fscanf(f, "%d %lld", &v, &j) != 2) return 9;
      const int k = st.segment("ingest_drop_segment", -1, v, j);
      if (k < 0) {
        status = 1;
        msg = st.err;
      } else {
        st.dropped[k - V] = 1;
      }
    } else {
      for (int k = 0; k < st.streams(); ++k)
        if (st.live(k)) pl.finish(k, &spans, &chunks);
    }
    fprintf(o, "op %d %d\n", i++, status);
    if (status) fprintf(o, "e %s\n", msg.c_str());
    for (const IngestSpan& s : spans)
      fprintf(o, "s %d %lld %lld %lld %lld\n", s.video, (long long)s.s0, (long long)s.s1, (long long)s.frame,
              (long long)s.tail);
    for (const IngestChunk& c : chunks) fprintf(o, "c %d %lld %lld\n", c.video, (long long)c.f0, (long long)c.f1);
    fprintf(o, "w");
    for (int v = 0; v < V; ++v) fprintf(o, " %lld", (long long)st.windows(pl, v));
    fprintf(o, "\n");
  }
  fclose(f);
  fprintf(o, "streams %d\n", st.streams());
  for (int k = 0; k < st.streams(); ++k) fprintf(o, "k %d %lld\n", (int)st.live(k), (long long)pl.frames[k]);
  fclose(o);
  return 0;
}
