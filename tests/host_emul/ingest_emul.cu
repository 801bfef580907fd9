// CPU run of the batched ingest session's span planner (ffsubsync_b200/csrc/ingest_plan.h): the same IngestPlanner
// b2_ingest_push and b2_ingest_sync_tracks run before they stage anything.  Test infrastructure (the build container
// has no GPU); tests/test_ingest_cpu.py drives it.
//
// usage: ingest_emul in.txt out.txt
//   in : "V fpw auditok chunk_samples energy_threshold_db", then one operation per line: "p v n_bytes" (a push of
//        n_bytes bytes to video v) or "f v" (the end of video v's stream).
//   out: per operation "op i", then its spans "s v s0 s1 frame tail" and completed detector calls "c v f0 f1"; at the
//        end "frames f_0 .. f_(V-1)" and "base b_0 .. b_(V-1)".
#include <stdio.h>

#include "../../ffsubsync_b200/csrc/ingest_plan.h"

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  FILE* f = fopen(argv[1], "r");
  if (!f) return 3;
  int V, fpw, auditok;
  long long chunk;
  double db;
  if (fscanf(f, "%d %d %d %lld %lf", &V, &fpw, &auditok, &chunk, &db) != 5) return 4;
  FILE* o = fopen(argv[2], "w");
  if (!o) return 5;
  IngestPlanner pl;
  pl.begin(V, fpw, auditok != 0, chunk, db);
  char op[8];
  int v, i = 0;
  while (fscanf(f, "%7s %d", op, &v) == 2) {
    std::vector<IngestSpan> spans;
    std::vector<IngestChunk> chunks;
    if (op[0] == 'p') {
      long long nb;
      if (fscanf(f, "%lld", &nb) != 1) return 6;
      pl.push(v, nb, &spans, &chunks);
    } else {
      pl.finish(v, &spans, &chunks);
    }
    fprintf(o, "op %d\n", i++);
    for (const IngestSpan& s : spans)
      fprintf(o, "s %d %lld %lld %lld %lld\n", s.video, (long long)s.s0, (long long)s.s1, (long long)s.frame,
              (long long)s.tail);
    for (const IngestChunk& c : chunks) fprintf(o, "c %d %lld %lld\n", c.video, (long long)c.f0, (long long)c.f1);
  }
  fclose(f);
  fprintf(o, "frames");
  for (int w = 0; w < V; ++w) fprintf(o, " %lld", (long long)pl.frames[w]);
  fprintf(o, "\nbase");
  for (int w = 0; w < V; ++w) fprintf(o, " %lld", (long long)pl.base[w]);
  fprintf(o, "\n");
  fclose(o);
  return 0;
}
