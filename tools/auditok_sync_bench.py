"""Cost of the auditok detector inside the batched sync: the bench shape with vad="energy_zcr" and vad="auditok".

    python tools/auditok_sync_bench.py [--videos 256] [--ratios 5] [--seconds 7200] [--steps 5] [--warmup 2]
                                       [--repeats 3] [--flip 0.0] [--hiss 0.0] [--trace]

BatchSynchronizer(grid, vad=...).sync_device over the same seeded pairs (PCM synthesised on the device, 2 h per pair
at 16 kHz, one subtitle per video at a planted grid ratio and delay), +-60 s, resident calls back to back as in
bench.py, timed alternately (energy_zcr, auditok, energy_zcr, ...) with CUDA events on one stream.  Reports ms per
step and kernel launches per call.

The PCM is voiced exactly where each video's cue list has speech by default (--flip / --hiss add bench.py's random
flips and hiss).  With bench.py's 10 % flips and 5 % hiss the isolated valid blocks lie closer than auditok's 0.25 s
of tolerated silence, so its tokens chain over whole videos, the signal is nearly constant and no aligner has a
usable peak.

The check: one more auditok call with per-ratio outputs against the composition of public entry points it replaces,
b2_vad_auditok (100 s detector calls) -> float32 -> b2_rasterize -> b2_align_batch -> b2_reduce_ratios.  The
composition is exact for a (pair, ratio) unless it overflowed its re-score budget (B2_ALIGN_CAND_OVERFLOW); there
the call (which scores every offset exactly) must score at least as high.  equals_composition: every per-ratio
(score, offset) where the composition is exact equal, no overflowed one scored higher by the composition, best_*
equal on every pair without an overflowed ratio, and the timed resident calls' outputs equal to this call's.  The
counts of overflowed jobs and of those that still agree are printed beside it.  --trace: one chained
pair of calls per detector with B2_PIPE_TRACE=1 (the sub-batch timeline on stderr).  Prints one JSON line per
measurement and the GPU's name and power limit, read in the same run.  Needs an H100.
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
    ap.add_argument("--flip", type=float, default=0.0)
    ap.add_argument("--hiss", type=float, default=0.0)
    ap.add_argument("--trace", action="store_true")
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS

    if not torch.cuda.is_available():
        sys.exit("auditok_sync_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = list(BENCH_RATIOS[: args.ratios])
    K, V = len(ratios), args.videos
    dev = torch.device("cuda", 0)
    syncs = {vad: BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0, vad=vad)
             for vad in ("energy_zcr", "auditok")}
    h = syncs["energy_zcr"].handle
    assert syncs["auditok"].handle is h
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    syncs["energy_zcr"].use_torch_stream()

    cls, n, cs, ce, cue_off, planted = make_tracks(h, V, 1, args.seconds, ratios, 7 + 1000 * V, flip=args.flip,
                                                  hiss_fraction=args.hiss)
    cls_d = torch.from_numpy(cls).to(dev)
    pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)
    h.synth_pcm(cls_d.data_ptr(), V * n, FPW, 7, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    torch.cuda.synchronize()
    del cls_d
    pcm_off = np.arange(V + 1, dtype=np.int64) * n * FPW
    outs = {vad: {k: torch.empty(V, dtype=dt, device=dev) for k, dt in
                  (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
            for vad in syncs}

    def timed(vad):
        def call():
            syncs[vad].sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs[vad], inputs_resident=True)
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

    res = {vad: [] for vad in syncs}
    for _ in range(args.repeats):
        for vad in syncs:
            res[vad].append(timed(vad))
    got = {k: v.cpu().numpy() for k, v in outs["auditok"].items()}
    if args.trace:
        os.environ["B2_PIPE_TRACE"] = "1"
        for vad in syncs:
            for _ in range(2):
                syncs[vad].sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs[vad], inputs_resident=True)
            torch.cuda.synchronize()
        del os.environ["B2_PIPE_TRACE"]

    # the call with per-ratio outputs
    sa = syncs["auditok"]
    tv = np.arange(V, dtype=np.int32)
    c_out = [torch.empty(V, dtype=dt, device=dev) for dt in (torch.float64, torch.int32, torch.int32)]
    c_as = torch.empty(V * K, dtype=torch.float64, device=dev)
    c_ao = torch.empty(V * K, dtype=torch.int32, device=dev)
    h.sync_tracks_auditok(pcm.data_ptr(), pcm_off, tv, FRAME_RATE, SAMPLE_RATE, 0.0, cs, ce, None, cue_off, ratios,
                          0.0, sa.max_offset_samples, sa.chunk_samples, best_score=c_out[0].data_ptr(),
                          best_offset=c_out[1].data_ptr(), best_k=c_out[2].data_ptr(), all_score=c_as.data_ptr(),
                          all_offset=c_ao.data_ptr(), memspace=_native.B2_DEVICE)
    # the per-stage composition the call replaces
    ref, ref_off = sa._vad_auditok_device(pcm, pcm_off)
    lengths = h.rasterize_lengths(ce, cue_off, ratios, K, False, SAMPLE_RATE)
    sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
    h.rasterize(cs, ce, None, cue_off, ratios, K, False, SAMPLE_RATE, 0.0, out=sub.data_ptr(), out_off=sub_off,
                memspace=_native.B2_DEVICE)
    score = torch.empty(V * K, dtype=torch.float64, device=dev)
    offset = torch.empty(V * K, dtype=torch.int32, device=dev)
    status = torch.empty(V * K, dtype=torch.int32, device=dev)
    h.align_batch(ref.data_ptr(), ref_off, sub.data_ptr(), sub_off, V, K, sa.max_offset_samples,
                  score=score.data_ptr(), offset=offset.data_ptr(), status=status.data_ptr(), memspace=_native.B2_DEVICE)
    w = [torch.empty(V, dtype=dt, device=dev) for dt in (torch.float64, torch.int32, torch.int32)]
    h.reduce_ratios(score.data_ptr(), offset.data_ptr(), status.data_ptr(), V, K, sa.max_offset_samples,
                    best_score=w[0].data_ptr(), best_offset=w[1].data_ptr(), best_k=w[2].data_ptr(),
                    memspace=_native.B2_DEVICE)
    h.synchronize()
    torch.cuda.synchronize()
    keys = ("best_score", "best_offset", "best_k")
    call = {k: x.cpu().numpy() for k, x in zip(keys, c_out)}
    comp = {k: x.cpu().numpy() for k, x in zip(keys, w)}
    c_s, c_o = c_as.cpu().numpy(), c_ao.cpu().numpy()
    m_s, m_o, st = score.cpu().numpy(), offset.cpu().numpy(), status.cpu().numpy()
    overflow = (st & _native.ALIGN_CAND_OVERFLOW) != 0
    exact = ~overflow
    per_ratio_equal = bool(np.array_equal(c_s[exact], m_s[exact]) and np.array_equal(c_o[exact], m_o[exact]))
    not_below = bool(np.all(c_s[overflow] >= m_s[overflow]))
    pair_exact = ~overflow.reshape(V, K).any(axis=1)
    best_equal = all(np.array_equal(call[k][pair_exact], comp[k][pair_exact]) for k in keys)
    timed_equal = all(np.array_equal(got[k], call[k]) for k in keys)
    overflow_equal = int(np.sum((c_s[overflow] == m_s[overflow]) & (c_o[overflow] == m_o[overflow])))
    best_equal_all = all(np.array_equal(call[k], comp[k]) for k in keys)
    equal = bool(per_ratio_equal and not_below and best_equal and timed_equal)
    for vad, rs in res.items():
        ms = [r[0] for r in rs]
        print(json.dumps(dict(info, event="measure", vad=vad, pairs=V, K=K, seconds_per_pair=args.seconds,
                              max_offset_seconds=60, steps=args.steps, ms_per_step=[round(m, 3) for m in ms],
                              ms_per_step_min=round(min(ms), 3), launches_per_call=rs[-1][1])), flush=True)
    print(json.dumps(dict(info, event="check", equals_composition=equal, flip=args.flip, hiss=args.hiss,
                          jobs=int(V * K), composition_overflow_jobs=int(overflow.sum()),
                          per_ratio_equal_where_exact=per_ratio_equal, overflow_jobs_score_not_below=not_below,
                          best_equal_where_exact=bool(best_equal), best_equal_all_pairs=bool(best_equal_all),
                          overflow_jobs_equal=overflow_equal, timed_resident_equal_checked_call=bool(timed_equal),
                          auditok_planted_k_fraction=float((got["best_k"] == planted[:, 0]).mean()),
                          auditok_planted_offset_fraction=float((got["best_offset"] == planted[:, 1]).mean()),
                          extra_ms_per_step=round(min(r[0] for r in res["auditok"]) -
                                                  min(r[0] for r in res["energy_zcr"]), 3))), flush=True)


if __name__ == "__main__":
    main()
