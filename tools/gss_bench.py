"""Cost of the golden-section search (--gss) inside the batched sync: the bench shape with and without it.

    python tools/gss_bench.py [--videos 256] [--ratios 5] [--seconds 7200] [--steps 5] [--warmup 2] [--repeats 3]

(a) BatchSynchronizer(grid).sync_device and (b) BatchSynchronizer(grid + [None]).sync_device (b2_sync_tracks_gss
through the identity track map) over the same seeded pairs (PCM synthesised on the device, 2 h per pair, one
subtitle per video at a planted grid ratio and delay), +-60 s, resident calls back to back as in bench.py, timed
alternately (a, b, a, b, ...) with CUDA events on one stream.  Reports ms per step, kernel launches per call, and
whether (b) equals the composition of public entry points it replaces: b2_vad_energy_zcr -> b2_sync_tracks with
per-ratio outputs -> gss_align_batch on the VAD signals -> the reference's combine (gss_batch.combine_gss); and
whether (b)'s grid answer equals (a)'s wherever the search does not win.  Prints one JSON line per measurement and
the GPU's name and power limit, read in the same run.  Needs an H100.
"""
import argparse
import json
import os
import sys

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
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.gss_batch import combine_gss, gss_align_batch
    from ffsubsync_b200.synth import BENCH_RATIOS

    if not torch.cuda.is_available():
        sys.exit("gss_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = list(BENCH_RATIOS[: args.ratios])
    K, V = len(ratios), args.videos
    dev = torch.device("cuda", 0)
    grid = BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0)
    gss = BatchSynchronizer(ratios + [None], FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0)
    h = grid.handle
    assert gss.handle is h
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    grid.use_torch_stream()

    cls, n, cs, ce, cue_off, planted = make_tracks(h, V, 1, args.seconds, ratios, 7 + 1000 * V)
    cls_d = torch.from_numpy(cls).to(dev)
    pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)
    h.synth_pcm(cls_d.data_ptr(), V * n, FPW, 7, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    torch.cuda.synchronize()
    del cls_d
    pcm_off = np.arange(V + 1, dtype=np.int64) * n * FPW
    out_a = {k: torch.empty(V, dtype=dt, device=dev) for k, dt in
             (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
    out_b = dict({k: torch.empty_like(v) for k, v in out_a.items()},
                 gss_ratio=torch.empty(V, dtype=torch.float64, device=dev))

    def step_a():
        grid.sync_device(pcm, pcm_off, cs, ce, cue_off, out=out_a, inputs_resident=True)

    def step_b():
        gss.sync_device(pcm, pcm_off, cs, ce, cue_off, out=out_b, inputs_resident=True)

    def timed(call):
        for _ in range(args.warmup):
            call()
        torch.cuda.synchronize()
        l0 = h.launch_count
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            call()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps, (h.launch_count - l0) / args.steps

    res = {"grid": [], "grid+gss": []}
    for _ in range(args.repeats):
        for name, fn in (("grid", step_a), ("grid+gss", step_b)):
            res[name].append(timed(fn))
    got_a = {k: v.cpu().numpy() for k, v in out_a.items()}
    got_b = {k: v.cpu().numpy() for k, v in out_b.items()}

    # the composition of public entry points the call replaces
    tv = np.arange(V, dtype=np.int32)
    c_bs = torch.empty(V, dtype=torch.float64, device=dev)
    c_bo, c_bk = torch.empty(V, dtype=torch.int32, device=dev), torch.empty(V, dtype=torch.int32, device=dev)
    c_as = torch.empty(V * K, dtype=torch.float64, device=dev)
    c_ao = torch.empty(V * K, dtype=torch.int32, device=dev)
    h.sync_tracks(pcm.data_ptr(), pcm_off, tv, FRAME_RATE, SAMPLE_RATE, 0.0, grid.energy_threshold, -1, -1, cs, ce,
                  None, cue_off, ratios, 0.0, grid.max_offset_samples, c_bs.data_ptr(), c_bo.data_ptr(),
                  c_bk.data_ptr(), c_as.data_ptr(), c_ao.data_ptr(), memspace=_native.B2_DEVICE)
    fpw = h.frames_per_window(FRAME_RATE, SAMPLE_RATE)
    ref_off = np.concatenate([[0], np.cumsum((np.diff(pcm_off) + fpw - 1) // fpw)]).astype(np.int64)
    ref = torch.empty(int(ref_off[-1]), dtype=torch.float32, device=dev)
    h.vad_energy_zcr(pcm.data_ptr(), pcm_off, FRAME_RATE, SAMPLE_RATE, 0.0, grid.energy_threshold, out=ref.data_ptr(),
                     memspace=_native.B2_DEVICE)
    h.synchronize()
    g = gss_align_batch(ref, ref_off, cs, ce, cue_off, None, grid.max_offset_samples, SAMPLE_RATE, 0.0, handle=h)
    w_bs, w_bo, w_bk, w_r, _, _ = combine_gss(c_bs.cpu().numpy(), c_bo.cpu().numpy(), c_bk.cpu().numpy(), g, K,
                                              grid.max_offset_samples)
    equal = bool(np.array_equal(got_b["best_score"], w_bs) and np.array_equal(got_b["best_offset"], w_bo)
                 and np.array_equal(got_b["best_k"], w_bk) and np.array_equal(got_b["gss_ratio"], w_r))
    grid_kept = got_b["best_k"] < K
    grid_same = bool(all(np.array_equal(got_a[k][grid_kept], got_b[k][grid_kept]) for k in got_a))
    planted_ok = bool((got_a["best_k"] == planted[:, 0]).all() and (got_a["best_offset"] == planted[:, 1]).all())
    for name, rs in res.items():
        ms = [r[0] for r in rs]
        print(json.dumps(dict(info, event="measure", mode=name, pairs=V, K=K, seconds_per_pair=args.seconds,
                              max_offset_seconds=60, steps=args.steps, ms_per_step=[round(m, 3) for m in ms],
                              ms_per_step_min=round(min(ms), 3), launches_per_call=rs[-1][1])), flush=True)
    print(json.dumps(dict(info, event="check", gss_equals_composition=equal, grid_answer_unchanged=grid_same,
                          gss_wins=int((got_b["best_k"] == K).sum()), grid_planted_ok=planted_ok,
                          extra_ms_per_step=round(min(r[0] for r in res["grid+gss"]) - min(r[0] for r in res["grid"]),
                                                  3))), flush=True)


if __name__ == "__main__":
    main()
