"""The batched ingest session (b2_ingest_*, ``BatchSynchronizer.ingest``) at the bench shape: 256 two-hour videos, one
track each, K = 5 grid ratios, +-60 s, at 16 kHz and at 48 kHz, the host PCM pushed in the reference's 100 s reads
round-robin across videos.

    python tools/ingest_bench.py [--videos 256] [--seconds 7200] [--rates 16000,48000] [--check-videos 4]
                                 [--repeats 2]

The PCM is generated on the host by seed: a pool of distinct 100 s pieces of synthetic speech (--pool of them),
video v's piece i being pool[(7 v + 3 i) mod pool] - so the pushes move the full 59 GB (16 kHz) or 177 GB (48 kHz)
while the host holds only the pool.  One JSON line per measurement, with the GPU's name and power limit read in the
same run:
- ``push``: bytes pushed over the host time from the first push until the device finished the last push's detector
  (``ingest_GBps``), and over the time the push calls took to return (``push_return_GBps``); the B2_HOST whole-call
  path's host-to-device rate on this machine is the comparison (51 GB/s measured for it before, H100 80 GB);
- ``sync``: the host time of the sync call after the last push (flush, the chain, results copied back);
- ``sync_profile``: the device time of each kernel and copy of repeat 0's sync step under torch.profiler - among them
  ``ref_bits_kernel``, which packs the float references into the run path's bits at sync, and the copy of the
  references into the chain's buffer;
- ``memory``: the device memory in use over cudaMemGetInfo's reading before the first session, after every round of
  pushes and after the results (peak and after);
- ``equal``: the results of the first --check-videos videos against b2_sync_tracks over their whole PCM.
Every measurement repeats ``--repeats`` times on full-size sessions; repeat 0 is the warm-up (first launches, the
chain's workspaces grown to full size, the profiler) and the later repeats are the steady state.
Needs an H100."""
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


def pool_pieces(frame_rate, n, seed):
    """n pieces of 100 s of synthetic PCM at frame_rate (voiced / silent / hiss runs of 0.37 s)."""
    from oracle import vad_oracle as vo
    fpw = frame_rate // SAMPLE_RATE
    rng = np.random.RandomState(seed)
    out = []
    for i in range(n):
        cls = np.repeat(rng.choice([0, 1, 2], size=10000 // 37 + 1, p=[0.45, 0.45, 0.1]), 37)[:10000].astype(np.uint8)
        out.append(vo.synth_pcm(cls, fpw, seed=seed * 1000 + i))
    return out


def piece(v, i, pool):
    return pool[(7 * v + 3 * i) % len(pool)]


def run(rate, args, bs_cls, torch):
    from ffsubsync_b200.synth import BENCH_RATIOS, synthetic_cues
    V, pieces_per_video = args.videos, int(round(args.seconds / 100.0))
    pool = pool_pieces(rate, args.pool, 7 + rate)
    ratios = list(BENCH_RATIOS[:5])
    bs = bs_cls(ratios, frame_rate=rate, max_offset_seconds=60.0, device=0)
    cs, ce, co = [], [], [0]
    for v in range(V):
        s, e = synthetic_cues(1000 + v, args.seconds)
        cs.append(s)
        ce.append(e)
        co.append(co[-1] + len(s))
    cs, ce, co = np.concatenate(cs), np.concatenate(ce), np.array(co, np.int64)
    tv = np.arange(V, dtype=np.int32)
    expect = np.full(V, pieces_per_video * len(pool[0]), np.int64)
    base = dict(frame_rate=rate, videos=V, seconds=args.seconds, K=len(ratios))
    free0, total = torch.cuda.mem_get_info()
    used = [total - free0]
    # repeat 0 is the warm-up: module load, first launches and the first full-size growth of the chain's workspaces;
    # its sync step is also profiled (device times of the step's kernels and copies)
    for rep in range(args.repeats):
        s = bs.ingest(V, expect_samples=expect)
        nbytes = 0
        t0 = time.perf_counter()
        push_s = 0.0
        for i in range(pieces_per_video):
            for v in range(V):
                p = piece(v, i, pool)
                a = time.perf_counter()
                s.push(v, p)
                push_s += time.perf_counter() - a
                nbytes += p.nbytes
            free, _ = torch.cuda.mem_get_info()
            used.append(total - free)
        bs.handle.synchronize()
        t1 = time.perf_counter()
        if rep == 0:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                res = s.sync_tracks(tv, cs, ce, co)
            kernels = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    name = "memcpy DtoD" if "DtoD" in e.name or "Device -> Device" in e.name else e.name.split("<")[0]
                    kernels[name] = kernels.get(name, 0.0) + e.device_time_total / 1e3
            top = dict(sorted(((k, round(v, 3)) for k, v in kernels.items()), key=lambda x: -x[1])[:8])
            print(json.dumps(dict(base, event="sync_profile", note="device ms per kernel / copy of the sync step, "
                                  "repeat 0 under torch.profiler; ref_bits_kernel = packing the float references at "
                                  "sync, memcpy DtoD = the references copied into the chain's buffer",
                                  device_ms=top, device_total_ms=round(sum(kernels.values()), 3))), flush=True)
        else:
            res = s.sync_tracks(tv, cs, ce, co)
        t2 = time.perf_counter()
        free, _ = torch.cuda.mem_get_info()
        used.append(total - free)
        r = dict(base, repeat=rep)
        print(json.dumps(dict(r, event="push", bytes=nbytes, ingest_s=round(t1 - t0, 3),
                              ingest_GBps=round(nbytes / (t1 - t0) / 1e9, 2), push_return_s=round(push_s, 3),
                              push_return_GBps=round(nbytes / push_s / 1e9, 2), pushes=pieces_per_video * V)),
              flush=True)
        print(json.dumps(dict(r, event="sync", last_push_to_results_ms=round((t2 - t1) * 1e3, 2),
                              profiled=rep == 0)), flush=True)
        print(json.dumps(dict(r, event="memory", peak_GB=round((max(used) - used[0]) / 1e9, 3),
                              after_GB=round((used[-1] - used[0]) / 1e9, 3), whole_pcm_GB=round(nbytes / 1e9, 1),
                              note="device memory in use over what it was before the first session")), flush=True)
    # the first check-videos videos through the non-streamed call over their whole PCM
    n = args.check_videos
    pcm = np.concatenate([piece(v, i, pool) for v in range(n) for i in range(pieces_per_video)])
    pcm_off = np.arange(n + 1, dtype=np.int64) * pieces_per_video * len(pool[0])
    want = bs.sync_host_tracks(pcm, pcm_off, tv[:n], cs[: co[n]], ce[: co[n]], co[: n + 1])
    eq = all(np.array_equal(np.asarray(a)[:n], np.asarray(b)) for a, b in zip(res, want))
    print(json.dumps(dict(base, event="equal", videos_checked=n, equal=bool(eq),
                          best_k=[int(x) for x in res[2][:n]])), flush=True)
    del pcm
    return eq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--rates", default="16000,48000")
    ap.add_argument("--pool", type=int, default=12)
    ap.add_argument("--check-videos", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    if not torch.cuda.is_available():
        sys.exit("ingest_bench: no CUDA device (this measurement runs on the GPU only)")
    print(json.dumps(dict(gpu_info(), event="gpu")), flush=True)
    ok = all([run(int(r), args, BatchSynchronizer, torch) for r in args.rates.split(",")])
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
