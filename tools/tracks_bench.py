"""Several subtitle tracks per video: one b2_sync_tracks call against the same tracks as (video, subtitle)
pairs through b2_sync_batch with every video's PCM copied once per track.

    python tools/tracks_bench.py [--videos 64] [--tracks 4] [--ratios 5] [--seconds 7200]
                                 [--steps 5] [--warmup 2] [--repeats 3] [--large-videos 256]

(a) V videos x T tracks through BatchSynchronizer.sync_device_tracks; (b) the same V*T pairs through
sync_device.  Both over the same seeded inputs (PCM synthesised on the device, 2 h per video), +-60 s,
resident calls back to back as in bench.py, timed alternately (a, b, a, b, ...) with CUDA events.  The
per-track outputs of (a) must equal those of (b); recovery of the planted (ratio, offset) is reported.  Then (a) alone at
--large-videos videos (b would need that many times T copies of 2 h PCM).  Prints one JSON line per
measurement and the GPU's name and power limit, read in the same run.  Needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FPW, SAMPLE_RATE, FRAME_RATE = 160, 100, 16000


def gpu_info():
    out = {}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, clk = (s.strip() for s in q.split(","))
        out.update(gpu=name, power_limit=pl, max_sm_clock=clk)
    except Exception as e:   # the name from torch still identifies the card
        out["nvidia_smi_error"] = str(e)
    import torch
    out.setdefault("gpu", torch.cuda.get_device_name(0))
    return out


def make_tracks(handle, V, T, duration_s, ratios, seed0, flip=0.10, hiss_fraction=0.05):
    """V videos; track i of video v is the video's master cue list at its own ratio and delay (planted).  A video's
    windows are voiced where its master list has speech, a fraction `flip` of them flipped, and `hiss_fraction` of
    the rest loud hiss (the random draws do not depend on the fractions, so the cue lists do not either)."""
    from ffsubsync_b200.synth import synthetic_cues
    n = int(duration_s * SAMPLE_RATE)
    cls = np.zeros(V * n, dtype=np.uint8)
    cs, ce, planted = [], [], []
    for v in range(V):
        seed = seed0 + v
        starts, ends = synthetic_cues(seed, duration_s)
        off = np.array([0, len(starts)], dtype=np.int64)
        mask = handle.rasterize(starts, ends, None, off, [1.0], 1, False, SAMPLE_RATE, 0.0)[0][:n] != 0
        rng = np.random.RandomState(seed + 100003)
        ref = np.zeros(n, dtype=bool)
        ref[: len(mask)] = mask
        ref ^= rng.rand(n) < flip
        hiss = rng.rand(n) < hiss_fraction
        cls[v * n:(v + 1) * n] = np.where(ref, 1, np.where(hiss, 2, 0))
        for _ in range(T):
            k, delta = int(rng.randint(len(ratios))), int(rng.randint(-3000, 3001))
            keep = rng.rand(len(starts)) >= 0.1
            st = (starts - delta / 100.0) / ratios[k]
            en = (ends - delta / 100.0) / ratios[k]
            keep &= st >= 0
            cs.append(np.round(st[keep], 3))
            ce.append(np.round(en[keep], 3))
            planted.append((k, delta))
    cue_off = np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64)
    return cls, n, np.concatenate(cs), np.concatenate(ce), cue_off, np.array(planted)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=64)
    ap.add_argument("--tracks", type=int, default=4)
    ap.add_argument("--ratios", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--large-videos", type=int, default=256)
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS

    if not torch.cuda.is_available():
        sys.exit("tracks_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = BENCH_RATIOS[: args.ratios]
    K = len(ratios)
    dev = torch.device("cuda", 0)
    bs = BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0)
    h = bs.handle
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    bs.use_torch_stream()
    T = args.tracks

    def corpus(V, seed0):
        cls, n, cs, ce, cue_off, planted = make_tracks(h, V, T, args.seconds, ratios, seed0)
        cls_d = torch.from_numpy(cls).to(dev)
        pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)
        h.synth_pcm(cls_d.data_ptr(), V * n, FPW, seed0, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
        torch.cuda.synchronize()
        del cls_d
        return pcm, n, cs, ce, cue_off, planted

    def timed(call, steps):
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        l0 = h.launch_count
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            call()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps, (h.launch_count - l0) / steps

    def run(V, with_pairs):
        pcm, n, cs, ce, cue_off, planted = corpus(V, 7 + 1000 * V)
        tv = np.repeat(np.arange(V, dtype=np.int32), T)
        pcm_off = np.arange(V + 1, dtype=np.int64) * n * FPW
        out_a = {k: torch.empty(V * T, dtype=dt, device=dev) for k, dt in
                 (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
        out_b = {k: torch.empty_like(v) for k, v in out_a.items()}

        def step_a():
            bs.sync_device_tracks(pcm, pcm_off, tv, cs, ce, cue_off, out=out_a, inputs_resident=True)

        calls = {"tracks": step_a}
        if with_pairs:
            pcm_b = pcm.view(V, 1, -1).expand(V, T, n * FPW).reshape(-1)   # every video's PCM once per track
            pcm_off_b = np.arange(V * T + 1, dtype=np.int64) * n * FPW

            def step_b():
                bs.sync_device(pcm_b, pcm_off_b, cs, ce, cue_off, out=out_b, inputs_resident=True)

            calls["pairs"] = step_b
        res = {name: [] for name in calls}
        for rep in range(args.repeats if with_pairs else 1):
            for name, fn in calls.items():
                ms, launches = timed(fn, args.steps)
                res[name].append((ms, launches))
        got_a = {k: v.cpu().numpy() for k, v in out_a.items()}
        planted_ok = bool((got_a["best_k"] == planted[:, 0]).all() and (got_a["best_offset"] == planted[:, 1]).all())
        equal = None
        if with_pairs:
            got_b = {k: v.cpu().numpy() for k, v in out_b.items()}
            equal = all(np.array_equal(got_a[k], got_b[k]) for k in got_a)
            assert equal, "per-track outputs of sync_device_tracks differ from sync_device on duplicated pairs"
        for name, rs in res.items():
            ms = [r[0] for r in rs]
            print(json.dumps(dict(info, event="measure", mode=name, videos=V, tracks_per_video=T, K=K,
                                  alignments=V * T * K, seconds_per_video=args.seconds, steps=args.steps,
                                  ms_per_step=[round(m, 3) for m in ms], ms_per_step_min=round(min(ms), 3),
                                  alignments_per_s=round(V * T * K / (min(ms) / 1e3), 1),
                                  launches_per_call=rs[-1][1], outputs_equal=equal, planted_ok=planted_ok)),
                  flush=True)
        del pcm
        if with_pairs:
            del pcm_b
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    run(args.videos, True)
    if args.large_videos:
        run(args.large_videos, False)


if __name__ == "__main__":
    main()
