"""Cost of serialized speech signals as references (``ffs ref.npz -i in.srt``) in the batched sync: the bench shape
with a fraction p of the videos synced against a stored signal (BatchSynchronizer's sig / sig_off / sig_video) instead
of their PCM, next to vad="energy_zcr" on every video.

    python tools/signal_ref_bench.py [--videos 256] [--ratios 5] [--seconds 7200] [--steps 5] [--warmup 2]
                                     [--repeats 3] [--fractions 1,0.5,0]

Every video has one subtitle track at a planted grid ratio and delay and PCM (synthesised on the device, 2 h at
16 kHz) voiced where its true cues are (tools/tracks_bench.make_tracks).  The stored signals are the corpus's own VAD
output (b2_vad_energy_zcr at label 0), as float64 the way np.load returns a --serialize-speech artefact, resident in
HBM.  For each p, every round(1/p)-th video (all of them at p = 1) takes its signal and an empty PCM range; the other
videos' PCM is packed back to back.  BatchSynchronizer.sync_device with +-60 s, resident calls back to back as in
bench.py, timed alternately against vad="energy_zcr" over the full PCM with CUDA events on one stream.  Reports ms per
step and kernel launches per call.

Per p > 0 also:
- the ingest kernel (sig_ref_kernel) from a torch.profiler run of one call: its device time, the bytes it moves
  (8 B read per frame, 4 B or 1/8 B written) and their rate;
- equals_composition: the call with per-ratio outputs against the composition of public entry points it replaces
  (the rule applied to each stored signal, b2_vad_energy_zcr for the audio videos, b2_rasterize, b2_align_batch,
  b2_reduce_ratios), exact where the composition did not overflow its re-score budget, not below it where it did,
  and the timed resident calls' outputs equal to that call's;
- equals_pcm_call: the timed call's outputs equal those of the energy_zcr call over the full PCM (its signals are
  that call's references).
Prints one JSON line per measurement and the GPU's name and power limit, read in the same run.  Needs an H100.
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
    ap.add_argument("--fractions", default="1,0.5,0")
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS

    if not torch.cuda.is_available():
        sys.exit("signal_ref_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = list(BENCH_RATIOS[: args.ratios])
    K, V = len(ratios), args.videos
    dev = torch.device("cuda", 0)
    syncs = {arm: BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0,
                                    vad="energy_zcr") for arm in ("energy_zcr", "signal")}
    h = syncs["energy_zcr"].handle
    assert syncs["signal"].handle is h
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    syncs["energy_zcr"].use_torch_stream()

    seed0 = 7 + 1000 * V
    cls, n, cs, ce, cue_off, planted = make_tracks(h, V, 1, args.seconds, ratios, seed0, flip=0.0, hiss_fraction=0.0)
    cls_d = torch.from_numpy(cls).to(dev)
    pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)

    def layout(sig):
        """PCM of the audio videos packed back to back (synthesised into pcm); returns pcm_off."""
        audio = np.flatnonzero(~sig)
        lens = np.where(sig, 0, n * FPW).astype(np.int64)
        if len(audio):
            src = cls_d.view(V, n)[torch.from_numpy(audio).to(dev)].reshape(-1).contiguous()
            h.synth_pcm(src.data_ptr(), len(audio) * n, FPW, 7, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
            h.synchronize()
        return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)

    # the stored signals: the corpus's own VAD output over the full PCM, as float64
    full_off = layout(np.zeros(V, dtype=bool))
    fpw = h.frames_per_window(FRAME_RATE, SAMPLE_RATE)
    det_off = np.concatenate([[0], np.cumsum((np.diff(full_off) + fpw - 1) // fpw)]).astype(np.int64)
    det = torch.empty(int(det_off[-1]), dtype=torch.float32, device=dev)
    h.vad_energy_zcr(pcm.data_ptr(), full_off, FRAME_RATE, SAMPLE_RATE, 0.0, syncs["energy_zcr"].energy_threshold,
                     -1, -1, out=det.data_ptr(), memspace=_native.B2_DEVICE)
    h.synchronize()
    stored = det.to(torch.float64)
    del det

    def sig_args(sig):
        sv = np.flatnonzero(sig)
        parts = [stored[det_off[v]: det_off[v + 1]] for v in sv]
        x = torch.cat(parts) if parts else torch.zeros(0, dtype=torch.float64, device=dev)
        off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        return dict(sig=x, sig_off=off, sig_video=sv)

    outs = {arm: {k: torch.empty(V, dtype=dt, device=dev) for k, dt in
                  (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
            for arm in syncs}

    def timed(arm, pcm_off, kw):
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

    no_sig = np.zeros(V, dtype=bool)
    for p in (float(x) for x in args.fractions.split(",")):
        sig = np.zeros(V, dtype=bool) if p <= 0 else (np.arange(V) % max(1, int(round(1.0 / p))) == 0)
        res = {"energy_zcr": [], "signal": []}
        for _ in range(args.repeats):
            res["energy_zcr"].append(timed("energy_zcr", layout(no_sig), {}))
            pcm_off = layout(sig)
            kw = sig_args(sig) if p > 0 else {}
            res["signal"].append(timed("signal", pcm_off, kw))
        for arm, rs in res.items():
            ms = [r[0] for r in rs]
            print(json.dumps(dict(info, event="measure", arm=arm, signal_fraction=p if arm != "energy_zcr" else 0.0,
                                  arm_of=p, signal_videos=int(sig.sum()) if arm != "energy_zcr" else 0, pairs=V, K=K,
                                  seconds_per_pair=args.seconds, max_offset_seconds=60, steps=args.steps,
                                  ms_per_step=[round(m, 3) for m in ms], ms_per_step_min=round(min(ms), 3),
                                  launches_per_call=rs[-1][1])), flush=True)
        if p <= 0:
            continue
        got = {k: v.cpu().numpy() for k, v in outs["signal"].items()}
        pcm_ref = {k: v.cpu().numpy() for k, v in outs["energy_zcr"].items()}
        ss = syncs["signal"]
        # the ingest kernel's time from a profiled call
        from torch.profiler import ProfilerActivity, profile
        frames = int(sum(det_off[v + 1] - det_off[v] for v in np.flatnonzero(sig)))
        with h.capture_reference(int(det_off[-1]) + 64, V) as cap:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                ss.sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs["signal"], inputs_resident=True, **kw)
                torch.cuda.synchronize()
        us = sum(e.device_time_total for e in prof.key_averages() if "sig_ref_kernel" in e.key)
        packed = cap["packed"][sig]
        n_packed = int(sum(det_off[v + 1] - det_off[v] for v in np.flatnonzero(sig) if cap["packed"][v]))
        moved = 8 * frames + 4 * (frames - n_packed) + n_packed / 8
        print(json.dumps(dict(info, event="ingest", signal_fraction=p, frames=frames, packed_videos=int(packed.sum()),
                              sig_ref_kernel_us=round(us, 1), bytes=int(moved),
                              gb_per_s=round(moved / (us * 1e-6) / 1e9, 1) if us > 0 else None)), flush=True)
        # the call with per-ratio outputs, and its composition of public entry points
        refs, pgs, sg, _ = ss._all_refs(V, dict(kw), on_device=True)
        tv = np.arange(V, dtype=np.int32)
        c_out = [torch.empty(V, dtype=dt, device=dev) for dt in (torch.float64, torch.int32, torch.int32)]
        c_as = torch.empty(V * K, dtype=torch.float64, device=dev)
        c_ao = torch.empty(V * K, dtype=torch.int32, device=dev)
        ss._dispatch(pcm, pcm_off, tv, cs, ce, cue_off, None, None, False, sig=sg,
                     best_score=c_out[0].data_ptr(), best_offset=c_out[1].data_ptr(), best_k=c_out[2].data_ptr(),
                     all_score=c_as.data_ptr(), all_offset=c_ao.data_ptr(), memspace=_native.B2_DEVICE)
        a_off = np.concatenate([[0], np.cumsum((np.diff(pcm_off) + fpw - 1) // fpw)]).astype(np.int64)
        a_det = torch.empty(max(int(a_off[-1]), 1), dtype=torch.float32, device=dev)
        h.vad_energy_zcr(pcm.data_ptr(), pcm_off, FRAME_RATE, SAMPLE_RATE, 0.0, ss.energy_threshold, -1, -1,
                         out=a_det.data_ptr(), memspace=_native.B2_DEVICE)
        h.synchronize()
        is_sig, x, voff = sg
        parts = [torch.where(x[voff[v]: voff[v + 1]] < 1.0, torch.zeros((), dtype=torch.float64, device=dev),
                             x[voff[v]: voff[v + 1]]).to(torch.float32) if is_sig[v]
                 else a_det[a_off[v]: a_off[v + 1]] for v in range(V)]
        ref_off = np.concatenate([[0], np.cumsum([len(q) for q in parts])]).astype(np.int64)
        ref = torch.cat(parts).contiguous()
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
        w = [torch.empty(V, dtype=dt, device=dev) for dt in (torch.float64, torch.int32, torch.int32)]
        h.reduce_ratios(score.data_ptr(), offset.data_ptr(), status.data_ptr(), V, K, ss.max_offset_samples,
                        best_score=w[0].data_ptr(), best_offset=w[1].data_ptr(), best_k=w[2].data_ptr(),
                        memspace=_native.B2_DEVICE)
        h.synchronize()
        torch.cuda.synchronize()
        keys = ("best_score", "best_offset", "best_k")
        call = {k: q.cpu().numpy() for k, q in zip(keys, c_out)}
        comp = {k: q.cpu().numpy() for k, q in zip(keys, w)}
        c_s, c_o = c_as.cpu().numpy(), c_ao.cpu().numpy()
        m_s, m_o, st = score.cpu().numpy(), offset.cpu().numpy(), status.cpu().numpy()
        overflow = (st & _native.ALIGN_CAND_OVERFLOW) != 0
        exact = ~overflow
        per_ratio_equal = bool(np.array_equal(c_s[exact], m_s[exact]) and np.array_equal(c_o[exact], m_o[exact]))
        not_below = bool(np.all(c_s[overflow] >= m_s[overflow]))
        pair_exact = ~overflow.reshape(V, K).any(axis=1)
        best_equal = all(np.array_equal(call[k][pair_exact], comp[k][pair_exact]) for k in keys)
        timed_equal = all(np.array_equal(got[k], call[k]) for k in keys)
        hit_k = got["best_k"] == planted[:, 0]
        hit_o = got["best_offset"] == planted[:, 1]
        print(json.dumps(dict(info, event="check", signal_fraction=p, signal_videos=int(sig.sum()),
                              equals_composition=bool(per_ratio_equal and not_below and best_equal and timed_equal),
                              equals_pcm_call=bool(all(np.array_equal(got[k], pcm_ref[k]) for k in keys)),
                              jobs=int(V * K), composition_overflow_jobs=int(overflow.sum()),
                              per_ratio_equal_where_exact=per_ratio_equal, overflow_jobs_score_not_below=not_below,
                              best_equal_where_exact=bool(best_equal),
                              timed_resident_equal_checked_call=bool(timed_equal),
                              planted_k_fraction=float(hit_k.mean()),
                              planted_offset_fraction=float(hit_o.mean()))), flush=True)


if __name__ == "__main__":
    main()
