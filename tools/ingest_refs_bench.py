"""References that need no audio in the batched ingest session (b2_ingest_sync_refs, ``IngestSession.sync_tracks`` with
text streams, PGS intervals and stored signals) at the BASELINE configs[2] shape: 256 two-hour videos, 16 kHz, one
track per video, K = 5 grid ratios, +-60 s, the reference's 100 s pushes round-robin over the pushed videos.

    python tools/ingest_refs_bench.py [--videos 256] [--seconds 7200] [--repeats 2] [--check-videos 8] [--arm A]

Two arms, each a session of the same V videos under the ``subs_then_energy_zcr`` synchroniser, each run in a process
of its own (``--arm`` runs one in this process), so that no arm's device memory reading holds what another arm's
sessions, workspaces or equality check left allocated:
- ``audio``: every video pushed;
- ``mixed``: the even videos pushed, the odd ones taking a reference that needs no audio, in turn an embedded text
  stream, PGS display intervals and a stored ``--serialize-speech`` signal, each built from a cue list of the bench
  corpus (ffsubsync_b200.synth.synthetic_cues; the signal is that list rasterised at 100 Hz, 1.0 on a cue and 0.0
  elsewhere).
The PCM is a pool of distinct 100 s pieces of synthetic speech (--pool of them), video v's piece i being
pool[(7 v + 3 i) mod pool].  One JSON line per measurement, with the GPU's name and power limit read in the same run:
- ``push``: the bytes pushed over the host time from the first push until the device finished the last push's
  detector (``ingest_GBps``);
- ``sync``: the host time of the sync call after the last push (flush, the reference videos' references, the chain,
  results copied back);
- ``memory``: device memory in use over cudaMemGetInfo's reading before the arm's first session (peak, and after the
  sync; the arm's equality check runs after its last reading);
- ``equal``: the first --check-videos videos' results against b2_sync_tracks_seg (no segments) over their PCM back to
  back and the same reference tables.
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

from ingest_bench import piece, pool_pieces  # noqa: E402
from tracks_bench import gpu_info  # noqa: E402

FRAME_RATE, SAMPLE_RATE = 16000, 100
PIECE_SECONDS = 100


def kind_of(v, arm):
    """"audio", "text", "pgs" or "sig" of video v in an arm."""
    if arm == "audio" or v % 2 == 0:
        return "audio"
    return ("text", "pgs", "sig")[(v // 2) % 3]


def references(videos, arm, seconds):
    """The sync methods' keyword arguments giving the listed videos (indices within the list) their references."""
    from ffsubsync_b200.synth import synthetic_cues
    text_s, text_e, text_o, text_v = [], [], [0], []
    pgs_s, pgs_e, pgs_o, pgs_v = [], [], [0], []
    sig, sig_o, sig_v = [], [0], []
    n_frames = int(seconds * SAMPLE_RATE)
    for i, v in enumerate(videos):
        k = kind_of(v, arm)
        if k == "audio":
            continue
        s, e = synthetic_cues(5000 + v, seconds)
        if k == "text":
            text_s.append(s)
            text_e.append(e)
            text_o.append(text_o[-1] + len(s))
            text_v.append(i)
        elif k == "pgs":
            pgs_s.append(s)
            pgs_e.append(e)
            pgs_o.append(pgs_o[-1] + len(s))
            pgs_v.append(i)
        else:
            x = np.zeros(n_frames, np.float64)
            for a, b in zip(s, e):
                x[int(a * SAMPLE_RATE): int(b * SAMPLE_RATE)] = 1.0
            sig.append(x)
            sig_o.append(sig_o[-1] + len(x))
            sig_v.append(i)
    kw = {}
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0)   # noqa: E731
    if text_v:
        kw.update(ref_cue_start=cat(text_s), ref_cue_end=cat(text_e), ref_cue_off=np.array(text_o, np.int64),
                  ref_stream_video=np.array(text_v, np.int64))
    if pgs_v:
        kw.update(pgs_start=cat(pgs_s), pgs_end=cat(pgs_e), pgs_off=np.array(pgs_o, np.int64),
                  pgs_video=np.array(pgs_v, np.int64))
    if sig_v:
        kw.update(sig=cat(sig), sig_off=np.array(sig_o, np.int64), sig_video=np.array(sig_v, np.int64))
    return kw


def run_arm(arm, bs, pool, tracks, args, torch, used):
    from ffsubsync_b200 import _native
    tv, cs, ce, co = tracks
    V = args.videos
    per_video = int(round(args.seconds / PIECE_SECONDS))
    pushed = [v for v in range(V) if kind_of(v, arm) == "audio"]
    refs = references(range(V), arm, args.seconds)
    base = dict(arm=arm, frame_rate=FRAME_RATE, videos=V, pushed_videos=len(pushed), seconds=args.seconds, K=5,
                reference_videos={k: sum(kind_of(v, arm) == k for v in range(V)) for k in ("text", "pgs", "sig")})
    expect = np.array([per_video * len(pool[0]) if kind_of(v, arm) == "audio" else 0 for v in range(V)], np.int64)
    res = None
    for rep in range(args.repeats):
        s = bs.ingest(V, expect_samples=expect)
        nbytes = 0
        t0 = time.perf_counter()
        for i in range(per_video):
            for v in pushed:
                p = piece(v, i, pool)
                s.push(v, p)
                nbytes += p.nbytes
        free, total = torch.cuda.mem_get_info()
        used.append(total - free)
        bs.handle.synchronize()
        t1 = time.perf_counter()
        res = s.sync_tracks(tv, cs, ce, co, **refs)
        t2 = time.perf_counter()
        free, total = torch.cuda.mem_get_info()
        used.append(total - free)
        r = dict(base, repeat=rep)
        print(json.dumps(dict(r, event="push", bytes=nbytes, ingest_s=round(t1 - t0, 3),
                              ingest_GBps=round(nbytes / (t1 - t0) / 1e9, 2), pushes=per_video * len(pushed))),
              flush=True)
        print(json.dumps(dict(r, event="sync", last_push_to_results_ms=round((t2 - t1) * 1e3, 2))), flush=True)
        print(json.dumps(dict(r, event="memory", peak_GB=round((max(used) - used[0]) / 1e9, 3),
                              after_GB=round((used[-1] - used[0]) / 1e9, 3),
                              note="device memory in use over what it was before the arm's first session")), flush=True)
    # the first n videos through the whole call (b2_sync_tracks_seg without segments) over their PCM back to back
    n = args.check_videos
    lens = [per_video * len(pool[0]) if kind_of(v, arm) == "audio" else 0 for v in range(n)]
    pcm = np.concatenate([piece(v, i, pool) for v in range(n) if kind_of(v, arm) == "audio"
                          for i in range(per_video)] + [np.zeros(0, np.int16)])
    pcm_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    t_n = int(np.searchsorted(tv, n))
    ref_n, pgs_n, sig_n, _ = bs._all_refs(n, references(range(n), arm, args.seconds), on_device=False)
    no_seg = (np.zeros(0, np.int32), np.zeros(0), np.zeros(1, np.int64), np.zeros(0, np.int64),
              np.zeros(0, np.int64), np.zeros(0, np.int64))
    want = bs._dispatch(pcm, pcm_off, tv[:t_n], cs[: co[t_n]], ce[: co[t_n]], co[: t_n + 1], None, ref_n, False,
                        pgs=pgs_n, sig=sig_n, seg=no_seg, memspace=_native.B2_HOST)
    eq = all(np.array_equal(np.asarray(a)[:t_n], np.asarray(b)) for a, b in zip(res[:3], want[:3]))
    print(json.dumps(dict(base, event="equal", videos_checked=n, equal=bool(eq))), flush=True)
    return eq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--pool", type=int, default=12)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--check-videos", type=int, default=8)
    ap.add_argument("--arm", choices=("audio", "mixed"), default=None, help="run one arm in this process")
    args = ap.parse_args()
    if args.arm is None:   # each arm in a fresh process: its memory baseline is the device as no arm left it
        import subprocess
        fails = 0
        for arm in ("audio", "mixed"):
            fails += subprocess.call([sys.executable, os.path.abspath(__file__), "--arm", arm] + sys.argv[1:]) != 0
        sys.exit(1 if fails else 0)
    import torch
    if not torch.cuda.is_available():
        sys.exit("ingest_refs_bench: no CUDA device (this measurement runs on the GPU only)")
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, synthetic_cues
    print(json.dumps(dict(gpu_info(), event="gpu")), flush=True)
    V = args.videos
    pool = pool_pieces(FRAME_RATE, args.pool, 7 + FRAME_RATE)
    bs = BatchSynchronizer(list(BENCH_RATIOS[:5]), frame_rate=FRAME_RATE, max_offset_seconds=60.0, device=0,
                           vad="subs_then_energy_zcr")
    cs, ce, co = [], [], [0]
    for v in range(V):
        s, e = synthetic_cues(1000 + v, args.seconds)
        cs.append(s)
        ce.append(e)
        co.append(co[-1] + len(s))
    tracks = (np.arange(V, dtype=np.int32), np.concatenate(cs), np.concatenate(ce), np.array(co, np.int64))
    free0, total = torch.cuda.mem_get_info()
    used = [total - free0]
    sys.exit(0 if run_arm(args.arm, bs, pool, tracks, args, torch, used) else 1)


if __name__ == "__main__":
    main()
