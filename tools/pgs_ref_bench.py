"""Cost of PGS references (--pgs-ref-stream) in the batched sync: the bench shape with a fraction p of the videos synced
against their PGS display intervals (BatchSynchronizer's pgs_* arguments) next to vad="energy_zcr" on every video.

    python tools/pgs_ref_bench.py [--videos 256] [--ratios 5] [--seconds 7200] [--steps 5] [--warmup 2]
                                   [--repeats 3] [--fractions 0,0.5,1]

Every video has one subtitle track at a planted grid ratio and delay (tools/tracks_bench.make_tracks: the video's
true speech cues, scaled, delayed, 10 % dropped) and PCM (synthesised on the device, 2 h at 16 kHz) voiced where those
cues are.  For each p, every round(1/p)-th video (all of them at p = 1) gets a PGS reference - its true speech cues as
display intervals - and an empty PCM range; the other videos' PCM is packed back to back.  BatchSynchronizer.sync_device with
+-60 s, resident calls back to back as in bench.py, timed alternately against vad="energy_zcr" over the full PCM
(energy_zcr, PGS p, energy_zcr, ...) with CUDA events on one stream.  Reports ms per step and kernel launches per call.

The check, per p > 0: one more call with per-ratio outputs against the composition of public entry points it
replaces - b2_vad_energy_zcr for the audio videos, b2_rasterize_pgs for the PGS ones, one
reference per track, b2_rasterize of the tracks, b2_align_batch, b2_reduce_ratios.  The composition is exact for a
(pair, ratio) unless it overflowed its re-score budget (B2_ALIGN_CAND_OVERFLOW); there the call (which scores every
offset exactly) must score at least as high.  equals_composition: every per-ratio (score, offset) where the composition
is exact equal, no overflowed one scored higher by the composition, best_* equal on every pair without an overflowed
ratio, and the timed resident calls' outputs equal to this call's.  Planted ratio / delay recovery is reported for the
PGS-reference videos and for all.  Prints one JSON line per measurement and the GPU's name and power limit, read
in the same run.  Needs an H100.
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
    ap.add_argument("--fractions", default="0,0.5,1")
    args = ap.parse_args()

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, synthetic_cues

    if not torch.cuda.is_available():
        sys.exit("pgs_ref_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    ratios = list(BENCH_RATIOS[: args.ratios])
    K, V = len(ratios), args.videos
    dev = torch.device("cuda", 0)
    syncs = {arm: BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60, device=0,
                                    vad="energy_zcr") for arm in ("energy_zcr", "pgs")}
    h = syncs["energy_zcr"].handle
    assert syncs["pgs"].handle is h
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    syncs["energy_zcr"].use_torch_stream()

    seed0 = 7 + 1000 * V
    cls, n, cs, ce, cue_off, planted = make_tracks(h, V, 1, args.seconds, ratios, seed0, flip=0.0, hiss_fraction=0.0)
    true_cues = [synthetic_cues(seed0 + v, args.seconds) for v in range(V)]   # make_tracks' master lists
    cls_d = torch.from_numpy(cls).to(dev)
    pcm = torch.empty(V * n * FPW, dtype=torch.int16, device=dev)

    def layout(subs):
        """PCM of the audio videos packed back to back (synthesised into pcm); returns pcm_off."""
        audio = np.flatnonzero(~subs)
        lens = np.where(subs, 0, n * FPW).astype(np.int64)
        if len(audio):
            src = cls_d.view(V, n)[torch.from_numpy(audio).to(dev)].reshape(-1).contiguous()
            h.synth_pcm(src.data_ptr(), len(audio) * n, FPW, 7, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
            h.synchronize()
        return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)

    def streams(subs):
        sv = np.flatnonzero(subs)
        st = [true_cues[v] for v in sv]
        off = np.concatenate([[0], np.cumsum([len(s[0]) for s in st])]).astype(np.int64)
        return dict(pgs_start=np.concatenate([s[0] for s in st] + [np.zeros(0)]),
                    pgs_end=np.concatenate([s[1] for s in st] + [np.zeros(0)]), pgs_off=off, pgs_video=sv)

    outs = {vad: {k: torch.empty(V, dtype=dt, device=dev) for k, dt in
                  (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
            for vad in syncs}

    def timed(vad, pcm_off, kw):
        def call():
            syncs[vad].sync_device(pcm, pcm_off, cs, ce, cue_off, out=outs[vad], inputs_resident=True, **kw)
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

    no_subs = np.zeros(V, dtype=bool)
    for p in (float(x) for x in args.fractions.split(",")):
        subs = np.zeros(V, dtype=bool) if p <= 0 else (np.arange(V) % max(1, int(round(1.0 / p))) == 0)
        res = {"energy_zcr": [], "pgs": []}
        for _ in range(args.repeats):
            res["energy_zcr"].append(timed("energy_zcr", layout(no_subs), {}))
            pcm_off = layout(subs)
            res["pgs"].append(timed("pgs", pcm_off, streams(subs)))
        for vad, rs in res.items():
            ms = [r[0] for r in rs]
            print(json.dumps(dict(info, event="measure", arm=vad, pgs_fraction=p if vad != "energy_zcr" else 0.0,
                                  arm_of=p, pgs_videos=int(subs.sum()) if vad != "energy_zcr" else 0, pairs=V, K=K,
                                  seconds_per_pair=args.seconds, max_offset_seconds=60, steps=args.steps,
                                  ms_per_step=[round(m, 3) for m in ms], ms_per_step_min=round(min(ms), 3),
                                  launches_per_call=rs[-1][1])), flush=True)
        if p <= 0:
            continue
        got = {k: v.cpu().numpy() for k, v in outs["pgs"].items()}
        # the call with per-ratio outputs
        ss = syncs["pgs"]
        pgs = ss._pgs_refs(V, streams(subs))
        tv = np.arange(V, dtype=np.int32)
        c_out = [torch.empty(V, dtype=dt, device=dev) for dt in (torch.float64, torch.int32, torch.int32)]
        c_as = torch.empty(V * K, dtype=torch.float64, device=dev)
        c_ao = torch.empty(V * K, dtype=torch.int32, device=dev)
        ss._dispatch(pcm, pcm_off, tv, cs, ce, cue_off, None, None, False, pgs=pgs,
                     best_score=c_out[0].data_ptr(), best_offset=c_out[1].data_ptr(), best_k=c_out[2].data_ptr(),
                     all_score=c_as.data_ptr(), all_offset=c_ao.data_ptr(), memspace=_native.B2_DEVICE)
        # the composition: detector / raster reference per video, then the public aligner steps
        fpw = h.frames_per_window(FRAME_RATE, SAMPLE_RATE)
        det_off = np.concatenate([[0], np.cumsum((np.diff(pcm_off) + fpw - 1) // fpw)]).astype(np.int64)
        det = torch.empty(max(int(det_off[-1]), 1), dtype=torch.float32, device=dev)
        h.vad_energy_zcr(pcm.data_ptr(), pcm_off, FRAME_RATE, SAMPLE_RATE, 0.0, ss.energy_threshold, -1, -1,
                         out=det.data_ptr(), memspace=_native.B2_DEVICE)
        is_pgs, ps, pe, poff = pgs
        # b2_rasterize_pgs takes the PGS videos' lists only (an empty list is an error)
        pv = np.flatnonzero(is_pgs)
        p_off = np.concatenate([[0], np.cumsum(np.diff(poff)[pv])]).astype(np.int64)
        r_len = h.rasterize_pgs_lengths(pe, p_off, SAMPLE_RATE)
        r_off = np.concatenate([[0], np.cumsum(r_len)]).astype(np.int64)
        rsig = torch.empty(max(int(r_off[-1]), 1), dtype=torch.float32, device=dev)
        h.rasterize_pgs(ps, pe, p_off, SAMPLE_RATE, 0.0, out=rsig.data_ptr(), out_off=r_off,
                        memspace=_native.B2_DEVICE)
        slot = {int(v): i for i, v in enumerate(pv)}
        parts = [rsig[r_off[slot[v]]: r_off[slot[v] + 1]] if is_pgs[v] else det[det_off[v]: det_off[v + 1]]
                 for v in range(V)]
        ref_off = np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.int64)
        ref = torch.cat(parts)
        lengths = h.rasterize_lengths(ce, cue_off, ratios, K, False, SAMPLE_RATE)
        sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
        h.rasterize(cs, ce, None, cue_off, ratios, K, False, SAMPLE_RATE, 0.0, out=sub.data_ptr(), out_off=sub_off,
                    memspace=_native.B2_DEVICE)
        score = torch.empty(V * K, dtype=torch.float64, device=dev)
        offset = torch.empty(V * K, dtype=torch.int32, device=dev)
        status = torch.empty(V * K, dtype=torch.int32, device=dev)
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
        hit_k = got["best_k"] == planted[:, 0]
        hit_o = got["best_offset"] == planted[:, 1]
        print(json.dumps(dict(info, event="check", pgs_fraction=p, pgs_videos=int(subs.sum()),
                              equals_composition=bool(per_ratio_equal and not_below and best_equal and timed_equal),
                              jobs=int(V * K), composition_overflow_jobs=int(overflow.sum()),
                              per_ratio_equal_where_exact=per_ratio_equal, overflow_jobs_score_not_below=not_below,
                              best_equal_where_exact=bool(best_equal),
                              best_equal_all_pairs=bool(all(np.array_equal(call[k], comp[k]) for k in keys)),
                              timed_resident_equal_checked_call=bool(timed_equal),
                              planted_k_fraction_pgs=float(hit_k[subs].mean()),
                              planted_offset_fraction_pgs=float(hit_o[subs].mean()),
                              planted_k_fraction_all=float(hit_k.mean()),
                              planted_offset_fraction_all=float(hit_o.mean()))), flush=True)


if __name__ == "__main__":
    main()
