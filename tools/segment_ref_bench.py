"""Cost of sampled segments as references (``--multi-segment-sync``) in the batched sync: the bench shape with a
fraction p of the videos synced against 8 sampled 60 s segments (BatchSynchronizer's seg_* arguments from
batch.segment_table) instead of their whole audio, next to vad="energy_zcr" on every video's full PCM.

    python tools/segment_ref_bench.py [--videos 256] [--ratios 5] [--seconds 7200] [--steps 5] [--warmup 2]
                                      [--repeats 3] [--fractions 1,0.5,0] [--host-videos 16]

Every video has one subtitle track at a planted grid ratio and delay and 2 h of 16 kHz PCM (synthesised on the device,
voiced where its true cues are: tools/tracks_bench.make_tracks), resident in HBM.  For each p, every round(1/p)-th
video (all of them at p = 1) is a segment video whose segments are slices of its resident decode.  sync_device with
+-60 s, resident calls back to back as in bench.py, timed alternately against vad="energy_zcr" with CUDA events.

Per p also:
- B2_HOST: sync_host on the first --host-videos videos from a host copy of their PCM (the segment videos' full decode:
  only their segments cross PCIe), ms per call, and the bytes copied host-to-device;
- seg_ref_kernel's device time from a torch.profiler run of one device call;
- equals_composition: the call's per-ratio outputs against the composition of public entry points (b2_vad_energy_zcr
  over each segment, placed by the reference's rule, b2_vad_energy_zcr over the audio videos, b2_rasterize,
  b2_align_batch, b2_reduce_ratios), exact where the composition did not overflow its re-score budget.
Prints one JSON line per measurement and the GPU's name and power limit, read in the same run.  Needs an H100.
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

from tracks_bench import FPW, FRAME_RATE, SAMPLE_RATE, gpu_info, make_tracks  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=256)
    ap.add_argument("--ratios", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=7200.0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--fractions", default="1,0.5,0")
    ap.add_argument("--host-videos", type=int, default=16)
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer, segment_table
    from ffsubsync_b200.synth import BENCH_RATIOS

    if not torch.cuda.is_available():
        sys.exit("segment_ref_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = list(BENCH_RATIOS[: args.ratios])
    K, V = len(ratios), args.videos
    dev = torch.device("cuda", 0)
    syncs = {arm: BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0,
                                    vad="energy_zcr") for arm in ("energy_zcr", "segments")}
    h = syncs["energy_zcr"].handle
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    syncs["energy_zcr"].use_torch_stream()

    seed0 = 7 + 1000 * V
    cls, n, cs, ce, cue_off, planted = make_tracks(h, V, 1, args.seconds, ratios, seed0, flip=0.0, hiss_fraction=0.0)
    cls_d = torch.from_numpy(cls).to(dev)
    pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)
    h.synth_pcm(cls_d.data_ptr(), V * n, FPW, 7, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    h.synchronize()
    del cls_d
    pcm_off = (np.arange(V + 1) * n * FPW).astype(np.int64)
    tv = np.arange(V, dtype=np.int32)

    outs = {arm: {k: torch.empty(V, dtype=dt, device=dev) for k, dt in
                  (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
            for arm in syncs}

    def timed(arm, kw):
        def call():
            syncs[arm].sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs[arm], inputs_resident=True, **kw)
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

    Vh = min(args.host_videos, V)
    pcm_host = pcm[: Vh * n * FPW].cpu().numpy()
    for p in (float(x) for x in args.fractions.split(",")):
        segv = np.zeros(V, dtype=bool) if p <= 0 else (np.arange(V) % max(1, int(round(1.0 / p))) == 0)
        kw = segment_table(pcm_off, FRAME_RATE, videos=np.flatnonzero(segv)) if segv.any() else {}
        res = {"energy_zcr": [], "segments": []}
        for _ in range(args.repeats):
            res["energy_zcr"].append(timed("energy_zcr", {}))
            res["segments"].append(timed("segments", kw))
        for arm, rs in res.items():
            ms = [r[0] for r in rs]
            print(json.dumps(dict(info, event="measure", arm=arm, arm_of=p,
                                  segment_videos=int(segv.sum()) if arm == "segments" else 0, pairs=V, K=K,
                                  seconds_per_pair=args.seconds, max_offset_seconds=60, steps=args.steps,
                                  ms_per_step=[round(m, 3) for m in ms], ms_per_step_min=round(min(ms), 3),
                                  launches_per_call=rs[-1][1])), flush=True)
        # B2_HOST on the first Vh videos: time per call and the bytes the call copies to the device
        hv = segv[:Vh]
        hkw = segment_table(pcm_off[: Vh + 1], FRAME_RATE, videos=np.flatnonzero(hv)) if hv.any() else {}
        host_bytes = 2 * int(sum(n * FPW for v in range(Vh) if not hv[v]) + sum(
            hkw["seg_hi"][j] - hkw["seg_lo"][j] for j in range(len(hkw.get("seg_lo", [])))))
        host = {}
        for arm, kk in (("energy_zcr", {}), ("segments", hkw)):
            t = []
            for _ in range(args.repeats + 1):
                t0 = time.perf_counter()
                syncs[arm].sync_host(pcm_host, pcm_off[: Vh + 1], cs, ce, cue_off[: Vh + 1], **kk)
                t.append((time.perf_counter() - t0) * 1e3)
            host[arm] = t[1:]
        print(json.dumps(dict(info, event="host", arm_of=p, pairs=Vh, segment_videos=int(hv.sum()),
                              ms_per_call_energy_zcr=[round(x, 1) for x in host["energy_zcr"]],
                              ms_per_call_segments=[round(x, 1) for x in host["segments"]],
                              h2d_bytes_energy_zcr=2 * Vh * n * FPW, h2d_bytes_segments=host_bytes)), flush=True)
        if not segv.any():
            continue
        # seg_ref_kernel's time, and the call with per-ratio outputs against its composition
        from torch.profiler import ProfilerActivity, profile
        ss = syncs["segments"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ss.sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs["segments"], inputs_resident=True, **kw)
            torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "seg_ref_kernel" in e.key)
        timed_out = {k: v.cpu().numpy() for k, v in outs["segments"].items()}
        a_s = torch.empty(V * K, dtype=torch.float64, device=dev)
        a_o = torch.empty(V * K, dtype=torch.int32, device=dev)
        ss.sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs["segments"], all_out={"score": a_s, "offset": a_o},
                       **kw)
        torch.cuda.synchronize()
        call = {k: v.cpu().numpy() for k, v in outs["segments"].items()}
        fpw = h.frames_per_window(FRAME_RATE, SAMPLE_RATE)
        parts = []
        seg_of = {int(v): i for i, v in enumerate(kw["seg_video"])}
        for v in range(V):
            if v not in seg_of:
                d = torch.empty((n * FPW + fpw - 1) // fpw, dtype=torch.float32, device=dev)
                h.vad_energy_zcr(pcm[pcm_off[v]:].data_ptr(), [0, n * FPW], FRAME_RATE, SAMPLE_RATE, 0.0,
                                 ss.energy_threshold, -1, -1, out=d.data_ptr(), memspace=_native.B2_DEVICE)
                parts.append(d)
                continue
            i = seg_of[v]
            js = range(int(kw["seg_off"][i]), int(kw["seg_off"][i + 1]))
            L = int(float(kw["seg_total"][i]) * SAMPLE_RATE) + 2
            x = torch.zeros(L, dtype=torch.float32, device=dev)
            for j in js:
                a, b = int(pcm_off[v] + kw["seg_lo"][j]), int(pcm_off[v] + kw["seg_hi"][j])
                piece = pcm[a:b].contiguous()
                d = torch.empty(max((b - a + fpw - 1) // fpw, 1), dtype=torch.float32, device=dev)
                h.vad_energy_zcr(piece.data_ptr(), [0, b - a], FRAME_RATE, SAMPLE_RATE, 0.0, ss.energy_threshold,
                                 -1, -1, out=d.data_ptr(), memspace=_native.B2_DEVICE)
                s0 = int(kw["seg_start"][j]) * SAMPLE_RATE
                e = min(s0 + (b - a + fpw - 1) // fpw, L)
                if e > s0:
                    x[s0:e] = d[: e - s0]
                h.synchronize()
            parts.append(x)
        h.synchronize()
        ref_off = np.concatenate([[0], np.cumsum([len(q) for q in parts])]).astype(np.int64)
        ref = torch.cat(parts).contiguous()
        del parts
        lengths = h.rasterize_lengths(ce, cue_off, ratios, K, False, SAMPLE_RATE)
        sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
        h.rasterize(cs, ce, None, cue_off, ratios, K, False, SAMPLE_RATE, 0.0, out=sub.data_ptr(), out_off=sub_off,
                    memspace=_native.B2_DEVICE)
        score = torch.empty(V * K, dtype=torch.float64, device=dev)
        offset = torch.empty(V * K, dtype=torch.int32, device=dev)
        status = torch.empty(V * K, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        h.align_batch(ref.data_ptr(), ref_off, sub.data_ptr(), sub_off, V, K, ss.max_offset_samples,
                      score=score.data_ptr(), offset=offset.data_ptr(), status=status.data_ptr(),
                      memspace=_native.B2_DEVICE)
        h.synchronize()
        del ref, sub
        m_s, m_o, st = score.cpu().numpy(), offset.cpu().numpy(), status.cpu().numpy()
        bs_, bo_, bk_ = h.reduce_ratios(m_s, m_o, st, V, K, ss.max_offset_samples)
        overflow = (st & _native.ALIGN_CAND_OVERFLOW) != 0
        c_s, c_o = a_s.cpu().numpy(), a_o.cpu().numpy()
        per_ratio = bool(np.array_equal(c_s[~overflow], m_s[~overflow]) and np.array_equal(c_o[~overflow],
                                                                                          m_o[~overflow]))
        pair_exact = ~overflow.reshape(V, K).any(axis=1)
        best = all(np.array_equal(call[k][pair_exact], w[pair_exact])
                   for k, w in (("best_score", bs_), ("best_offset", bo_), ("best_k", bk_)))
        timed_equal = all(np.array_equal(timed_out[k], call[k]) for k in call)
        print(json.dumps(dict(info, event="check", arm_of=p, segment_videos=int(segv.sum()),
                              seg_ref_kernel_us=round(us, 1),
                              equals_composition=bool(per_ratio and best and timed_equal),
                              jobs=int(V * K), composition_overflow_jobs=int(overflow.sum()),
                              planted_k_fraction=float((call["best_k"] == planted[:, 0]).mean()),
                              planted_offset_fraction=float((call["best_offset"] == planted[:, 1]).mean()))),
              flush=True)


if __name__ == "__main__":
    main()
