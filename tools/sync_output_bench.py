"""Cost of try_sync's output step (b2_apply_sync) at the bench shape, against the sync step it follows and against
the host timedelta loop it replaces.

    python tools/sync_output_bench.py [--pairs 256] [--ratios 5] [--steps 5] [--warmup 2] [--repeats 20]
                                      [--host-tracks 256]

The workload is bench.py's: 256 two-hour pairs (synth.make_pairs, about 1 200 cues each), PCM synthesised on the
device, BatchSynchronizer.sync_device with +-60 s as resident calls back to back.  Timed with CUDA events on one
stream: the sync step alone, then apply_sync alone over that step's results with the gate and suppression on
(--skip-sync-on-low-quality, --apply-offset-seconds 0.25, --suppress-output-if-offset-less-than -30).  The host loop
is the reference's SubtitleScaler + SubtitleShifter arithmetic (timedelta per cue time) over --host-tracks of the
tracks, timed with the host clock.  The check: apply_sync's outputs equal oracle/sync_output_oracle.py on the same
results for every cue.  Prints one JSON line per measurement and the GPU's name and power limit, read in the same
run.  Needs an H100.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tracks_bench import FPW, FRAME_RATE, SAMPLE_RATE, gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--ratios", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--host-tracks", type=int, default=256)
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    from oracle import sync_output_oracle as so

    if not torch.cuda.is_available():
        sys.exit("sync_output_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    dev = torch.device("cuda", 0)
    ratios = list(BENCH_RATIOS[: args.ratios])
    B = args.pairs
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    bs = BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60)
    bs.use_torch_stream()
    h = bs.handle
    pairs = make_pairs([13 + b for b in range(B)], 7200.0, ratios, handle=h)
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(pairs.window_class).to(dev)
    pcm = torch.empty(n_win * FPW, dtype=torch.int16, device=dev)
    h.synth_pcm(cls_d.data_ptr(), n_win, FPW, 1234, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    del cls_d
    pcm_off = pairs.win_off * FPW
    cs, ce, co = pairs.cue_start, pairs.cue_end, pairs.cue_off
    n_cues = int(co[-1])
    rule = dict(skip_sync_on_low_quality=True, apply_offset_seconds=0.25, suppress_output_if_offset_less_than=-30.0)
    out = {"best_score": torch.empty(B, dtype=torch.float64, device=dev),
           "best_offset": torch.empty(B, dtype=torch.int32, device=dev),
           "best_k": torch.empty(B, dtype=torch.int32, device=dev)}

    def step():
        bs.sync_device(pcm, pcm_off, cs, ce, co, out=out, inputs_resident=True)

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(n):
            fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n

    for _ in range(args.warmup):
        step()
    step_ms = timed(step, args.steps)
    res = bs.apply_sync(out, cs, ce, co, **rule)   # warm-up of the epilogue (and its metadata arena)
    torch.cuda.synchronize(dev)
    apply_ms = timed(lambda: bs.apply_sync(out, cs, ce, co, **rule), args.repeats)
    res = {k: v.cpu().numpy() for k, v in bs.apply_sync(out, cs, ce, co, **rule).items()}
    torch.cuda.synchronize(dev)
    # device time of the kernel and of the cue upload alone (a separate, traced run: the calls above are
    # bound by the host's check-and-copy of the cue times)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            bs.apply_sync(out, cs, ce, co, **rule)
        torch.cuda.synchronize(dev)
    dev_us = {}
    for e in prof.key_averages():
        if "apply_sync_kernel" in e.key or "Memcpy HtoD" in e.key:
            t = getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0)
            dev_us["kernel_us" if "apply_sync_kernel" in e.key else "h2d_us"] = round(float(t), 2)
    got = [out[k].cpu().numpy() for k in ("best_score", "best_offset", "best_k")]
    want = so.apply_sync(*got, None, cs, ce, co, ratios, SAMPLE_RATE, apply_offset_seconds=0.25, gate=True,
                         suppress=-30.0)
    ok = all(np.array_equal(res[k], w, equal_nan=True)
             for k, w in zip(("synced_start_us", "synced_end_us", "offset_seconds", "scale", "status"), want))
    # the host loop the epilogue replaces: SubtitleScaler + SubtitleShifter per cue time, in Python
    from datetime import timedelta
    T_host = min(args.host_tracks, B)
    t0 = time.perf_counter()
    for t in range(T_host):
        scale = ratios[int(got[2][t])] if got[2][t] >= 0 else 1.0
        shift = timedelta(seconds=int(got[1][t]) / float(SAMPLE_RATE) + 0.25)
        for i in range(int(co[t]), int(co[t + 1])):
            timedelta(seconds=float(cs[i]) * scale) + shift
            timedelta(seconds=float(ce[i]) * scale) + shift
    host_s = (time.perf_counter() - t0) * B / T_host
    print(json.dumps(dict(info, event="measure", pairs=B, K=len(ratios), cues=n_cues, step_ms=round(step_ms, 3),
                          apply_sync_ms=round(apply_ms, 4), apply_sync_share_of_step=round(apply_ms / step_ms, 5),
                          apply_sync_device=dev_us,
                          host_timedelta_loop_s=round(host_s, 3), host_loop_tracks_timed=T_host,
                          statuses={str(k): int(v) for k, v in zip(*np.unique(res["status"], return_counts=True))},
                          equals_oracle=bool(ok))), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
