"""Sampled segments through the batched ingest session (``--multi-segment-sync`` in a session: b2_ingest_segments /
b2_ingest_push_segments, ``IngestSession.push_segment``) at the bench shape: 256 two-hour videos, 8 x 60 s segments
each (MultiSegmentVideoSpeechTransformer._segment_starts), one track per video, K = 5 grid ratios, +-60 s, at 16 kHz
and at 48 kHz.  Each segment is pushed in the reference's 100 s reads (one read holds a 60 s segment), round-robin
over the videos.

    python tools/segment_ingest_bench.py [--videos 256] [--seconds 7200] [--rates 16000,48000] [--repeats 2]

The segments' PCM is a pool of distinct 60 s pieces of synthetic speech, video v's segment j being
pool[(7 v + 3 j) mod pool].  One JSON line per measurement, with the GPU's name and power limit read in the same run:
- ``push``: the segments' bytes over the host time from the first push until the device finished the last push's
  detector (``ingest_GBps``), and over the time the push calls took to return;
- ``sync``: the host time of the sync call after the last push (flush, assembly of the sparse references, the chain,
  results copied back);
- ``memory``: device memory in use over cudaMemGetInfo's reading before the first session (peak, and after the sync);
- ``whole_call``: the same videos through b2_sync_tracks_seg (B2_HOST) from the pieces held back to back in host
  memory (``host_GB`` of them): its host time, and whether its results equal the session's.
Repeat 0 is the warm-up; the later repeats are the steady state.  Needs an H100."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tracks_bench import gpu_info  # noqa: E402

SAMPLE_RATE = 100
SEGMENTS, DURATION = 8, 60


def pool_pieces(frame_rate, n, seed):
    """n pieces of 60 s of synthetic PCM at frame_rate (voiced / silent / hiss runs of 0.37 s)."""
    from oracle import vad_oracle as vo
    fpw = frame_rate // SAMPLE_RATE
    rng = np.random.RandomState(seed)
    nw = DURATION * SAMPLE_RATE
    out = []
    for i in range(n):
        cls = np.repeat(rng.choice([0, 1, 2], size=nw // 37 + 1, p=[0.45, 0.45, 0.1]), 37)[:nw].astype(np.uint8)
        out.append(vo.synth_pcm(cls, fpw, seed=seed * 1000 + i))
    return out


def run(rate, args, torch):
    from ffsubsync_b200.batch import BatchSynchronizer, ingest_segment_table, segment_table
    from ffsubsync_b200.synth import BENCH_RATIOS, synthetic_cues
    V = args.videos
    pool = pool_pieces(rate, args.pool, 11 + rate)
    piece = lambda v, j: pool[(7 * v + 3 * j) % len(pool)]
    bs = BatchSynchronizer(list(BENCH_RATIOS[:5]), frame_rate=rate, max_offset_seconds=60.0, device=0)
    table = ingest_segment_table([args.seconds] * V, np.arange(V), SEGMENTS, DURATION)
    S = int(table["seg_off"][1])
    cs, ce, co = [], [], [0]
    for v in range(V):
        s, e = synthetic_cues(1000 + v, args.seconds)
        cs.append(s)
        ce.append(e)
        co.append(co[-1] + len(s))
    cs, ce, co = np.concatenate(cs), np.concatenate(ce), np.array(co, np.int64)
    tv = np.arange(V, dtype=np.int32)
    base = dict(frame_rate=rate, videos=V, seconds=args.seconds, segments=S, segment_seconds=DURATION,
                K=len(BENCH_RATIOS[:5]))
    free0, total = torch.cuda.mem_get_info()
    used = [total - free0]
    res = None
    for rep in range(args.repeats):
        s = bs.ingest(V, expect_samples=np.full(V, DURATION * rate, np.int64), segments=table)
        nbytes, push_s = 0, 0.0
        t0 = time.perf_counter()
        for j in range(S):
            for v in range(V):
                p = piece(v, j)
                a = time.perf_counter()
                s.push_segment(v, j, p)
                push_s += time.perf_counter() - a
                nbytes += p.nbytes
        free, _ = torch.cuda.mem_get_info()
        used.append(total - free)
        bs.handle.synchronize()
        t1 = time.perf_counter()
        res = s.sync_tracks(tv, cs, ce, co)
        t2 = time.perf_counter()
        free, _ = torch.cuda.mem_get_info()
        used.append(total - free)
        r = dict(base, repeat=rep)
        print(json.dumps(dict(r, event="push", bytes=nbytes, ingest_s=round(t1 - t0, 3),
                              ingest_GBps=round(nbytes / (t1 - t0) / 1e9, 2), push_return_s=round(push_s, 3),
                              push_return_GBps=round(nbytes / push_s / 1e9, 2), pushes=S * V)), flush=True)
        print(json.dumps(dict(r, event="sync", last_push_to_results_ms=round((t2 - t1) * 1e3, 2))), flush=True)
        print(json.dumps(dict(r, event="memory", peak_GB=round((max(used) - used[0]) / 1e9, 3),
                              after_GB=round((used[-1] - used[0]) / 1e9, 3),
                              note="device memory in use over what it was before the first session")), flush=True)
    # the same videos through the whole call, from the pieces held back to back
    pcm = np.concatenate([piece(v, j) for v in range(V) for j in range(S)])
    pcm_off = np.arange(V + 1, dtype=np.int64) * S * len(pool[0])
    whole = segment_table(pcm_off, rate, None, [args.seconds] * V, SEGMENTS, DURATION,
                          piece_samples=[[len(pool[0])] * S] * V)
    times = []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        want = bs.sync_host_tracks(pcm, pcm_off, tv, cs, ce, co, **whole)
        times.append(time.perf_counter() - t0)
    eq = all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(res, want))
    print(json.dumps(dict(base, event="whole_call", host_GB=round(pcm.nbytes / 1e9, 2),
                          call_ms=[round(t * 1e3, 1) for t in times], equal=bool(eq))), flush=True)
    del pcm
    return eq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--rates", default="16000,48000")
    ap.add_argument("--pool", type=int, default=12)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("segment_ingest_bench: no CUDA device (this measurement runs on the GPU only)")
    print(json.dumps(dict(gpu_info(), event="gpu")), flush=True)
    ok = all([run(int(r), args, torch) for r in args.rates.split(",")])
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
