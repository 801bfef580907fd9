"""Cost of the speech output (``--serialize-speech``, b2_speech_output) of the batched sync calls at the bench shape:
256 two-hour videos at 16 kHz, one track each, K = 5 grid ratios, +-60 s, resident calls back to back as in bench.py.

    python tools/speech_out_bench.py [--videos 256] [--ratios 5] [--seconds 7200] [--steps 5] [--warmup 2]
                                     [--repeats 3] [--host-videos 16]

Measurements (one JSON line each, with the GPU's name and power limit read in the same run):
- ``sync``: ms per step of BatchSynchronizer.sync_device without and with ``speech_video`` = every video, alternated,
  ``--repeats`` runs each (CUDA events on one stream), and the launches per call;
- ``kernel``: speech_out_kernel's device time from a torch.profiler run of one call, the bytes it moves (8 B written
  per frame, 4 B or 1/8 B read) and their rate, next to the 3.35 TB/s data-sheet bound;
- ``serialize_only``: a call without tracks that writes every video's signal, against b2_vad_energy_zcr over the same
  PCM (the detector pass a caller would otherwise make), CUDA events;
- ``host``: sync_host over the first ``--host-videos`` videos (the whole corpus does not fit a host copy), without and
  with the output copied back, host clock around the blocking call;
- ``equal``: the outputs with and without the speech output, and the speech against b2_vad_energy_zcr widened.
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

from tracks_bench import FPW, FRAME_RATE, SAMPLE_RATE, gpu_info, make_tracks  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=256)
    ap.add_argument("--ratios", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-videos", type=int, default=16)
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS

    if not torch.cuda.is_available():
        sys.exit("speech_out_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = list(BENCH_RATIOS[: args.ratios])
    K, V = len(ratios), args.videos
    dev = torch.device("cuda", 0)
    bs = BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0)
    h = bs.handle
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    bs.use_torch_stream()

    cls, n, cs, ce, cue_off, _ = make_tracks(h, V, 1, args.seconds, ratios, 7 + 1000 * V, flip=0.0, hiss_fraction=0.0)
    cls_d = torch.from_numpy(cls).to(dev)
    pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)
    h.synth_pcm(cls_d.data_ptr(), V * n, FPW, 7, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    h.synchronize()
    pcm_off = np.arange(V + 1, dtype=np.int64) * n * FPW
    every = np.arange(V)
    outs = {arm: {k: torch.empty(V, dtype=dt, device=dev) for k, dt in
                  (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
            for arm in ("plain", "speech")}
    last = {}

    def events(fn, steps):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        l0 = h.launch_count
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps, (h.launch_count - l0) / steps

    def call(arm):
        def fn():
            r = bs.sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs[arm], inputs_resident=True,
                               speech_video=every if arm == "speech" else None)
            if arm == "speech":
                last["speech"], last["off"] = r["speech"], r["speech_off"]
        return fn

    res = {"plain": [], "speech": []}
    for _ in range(args.repeats):
        for arm in ("plain", "speech"):
            res[arm].append(events(call(arm), args.steps))
    frames = int(last["off"][-1])
    for arm, rs in res.items():
        ms = [r[0] for r in rs]
        print(json.dumps(dict(info, event="sync", arm=arm, pairs=V, K=K, seconds_per_pair=args.seconds,
                              max_offset_seconds=60, steps=args.steps, ms_per_step=[round(m, 3) for m in ms],
                              ms_per_step_min=round(min(ms), 3), spread_ms=round(max(ms) - min(ms), 3),
                              launches_per_call=rs[-1][1], speech_frames=frames if arm == "speech" else 0)),
              flush=True)

    # the kernel on its own, from a profiled call
    from torch.profiler import ProfilerActivity, profile
    with h.capture_reference(frames + 64, V) as cap:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call("speech")()
            torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "speech_out_kernel" in e.key)
    n_packed = int(sum(cap["ref_off"][v + 1] - cap["ref_off"][v] for v in range(V) if cap["packed"][v]))
    moved = 8 * frames + 4 * (frames - n_packed) + n_packed / 8
    print(json.dumps(dict(info, event="kernel", frames=frames, packed_frames=n_packed, bytes=int(moved),
                          speech_out_kernel_us=round(us, 1), gb_per_s=round(moved / (us * 1e-6) / 1e9, 1) if us else None,
                          datasheet_bound_us=round(moved / 3.35e12 * 1e6, 1))), flush=True)

    # equality: results with and without the output, the speech against the detector widened
    fpw = h.frames_per_window(FRAME_RATE, SAMPLE_RATE)
    det_off = np.concatenate([[0], np.cumsum((np.diff(pcm_off) + fpw - 1) // fpw)]).astype(np.int64)
    det = torch.empty(int(det_off[-1]), dtype=torch.float32, device=dev)

    def vad():
        h.vad_energy_zcr(pcm.data_ptr(), pcm_off, FRAME_RATE, SAMPLE_RATE, 0.0, bs.energy_threshold, -1, -1,
                         out=det.data_ptr(), memspace=_native.B2_DEVICE)
    vad()
    torch.cuda.synchronize()
    same = all(torch.equal(outs["plain"][k], outs["speech"][k]) for k in outs["plain"])
    speech_ok = bool(torch.equal(last["speech"], det.to(torch.float64)))
    print(json.dumps(dict(info, event="equal", results_equal=same, speech_equals_vad=speech_ok)), flush=True)

    # serialize-only: no tracks, every video's signal, against the detector pass over the same PCM
    empty = (np.zeros(0, np.int32), np.zeros(0), np.zeros(0), np.zeros(1, np.int64))

    def ser():
        last["ser"] = bs.sync_device_tracks(pcm, pcm_off, *empty, speech_video=every)["speech"]
    t_ser = [events(ser, args.steps)[0] for _ in range(args.repeats)]
    t_vad = [events(vad, args.steps)[0] for _ in range(args.repeats)]
    print(json.dumps(dict(info, event="serialize_only", ms_serialize_only=[round(t, 3) for t in t_ser],
                          ms_vad_energy_zcr=[round(t, 3) for t in t_vad],
                          equal=bool(torch.equal(last["ser"], det.to(torch.float64))))), flush=True)
    del last["ser"], det

    # B2_HOST with the copy back, on a subset
    Vh = min(args.host_videos, V)
    pcm_h = pcm[: Vh * n * FPW].cpu().numpy()
    off_h = pcm_off[: Vh + 1]
    sh = BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0)
    t = {"plain": [], "speech": []}
    for rep in range(args.repeats + 1):
        for arm in ("plain", "speech"):
            t0 = time.perf_counter()
            r = sh.sync_host(pcm_h, off_h, cs, ce, cue_off[: Vh + 1], speech_video=np.arange(Vh) if arm == "speech"
                             else None)
            if rep:
                t[arm].append((time.perf_counter() - t0) * 1e3)
    print(json.dumps(dict(info, event="host", videos=Vh, ms_plain=[round(x, 1) for x in t["plain"]],
                          ms_speech=[round(x, 1) for x in t["speech"]], speech_mb=round(r[-1][-1] * 8 / 1e6, 1))),
          flush=True)


if __name__ == "__main__":
    main()
