#!/usr/bin/env python
"""b2_sync_batch sub-batch pipeline (VAD of later sub-batches on a subset of the SMs, alignment on the rest):
one resident batch, a sweep over B2_SUBBATCHES x B2_VAD_SMS x B2_VAD_BATCH; every setting must reproduce the
unpipelined results bit for bit.

    python tools/pipeline_probe.py [pairs [n_combos]]
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffsubsync_b200 import _native  # noqa: E402
from ffsubsync_b200.batch import BatchSynchronizer  # noqa: E402
from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs  # noqa: E402

FPW, FR = 160, 16000
KNOBS = ("B2_SUBBATCHES", "B2_VAD_SMS", "B2_VAD_BATCH", "B2_VAD_LAYOUT", "B2_VAD_EVICT_FIRST", "B2_PIPE_TRACE")


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
    dev = torch.device("cuda", 0)
    bs = BatchSynchronizer(BENCH_RATIOS, FR, 100, 0.0, max_offset_seconds=60, device=0)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    bs.use_torch_stream()
    pairs = make_pairs([7000 + b for b in range(B)], 7200.0, BENCH_RATIOS, handle=bs.handle)
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(pairs.window_class).to(dev)
    pcm = torch.empty(n_win * FPW, dtype=torch.int16, device=dev)
    bs.handle.synth_pcm(cls_d.data_ptr(), n_win, FPW, 99, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    del cls_d
    pcm_off = pairs.win_off * FPW

    def run(env, steps=5, resident=False):
        for k in KNOBS:
            os.environ.pop(k, None)
        os.environ.update(env)
        kw = {"inputs_resident": True} if resident else {}
        out = {"best_score": torch.empty(B, dtype=torch.float64, device=dev),
               "best_offset": torch.empty(B, dtype=torch.int32, device=dev),
               "best_k": torch.empty(B, dtype=torch.int32, device=dev)}
        for _ in range(3):
            bs.sync_device(pcm, pcm_off, pairs.cue_start, pairs.cue_end, pairs.cue_off, out=out, **kw)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(steps):
            bs.sync_device(pcm, pcm_off, pairs.cue_start, pairs.cue_end, pairs.cue_off, out=out, **kw)
        b.record(stream)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps, {k: v.cpu().numpy().copy() for k, v in out.items()}

    ms0, ref = run({"B2_VAD_LAYOUT": "group"})
    ok0 = bool((ref["best_offset"] == pairs.true_offset).all() and (ref["best_k"] == pairs.true_k).all())
    print("pairs=%d lane-group kernel, no pipeline: %.3f ms/step (%.0f alignments/s), planted offsets ok=%s"
          % (B, ms0, B / ms0 * 1e3, ok0), flush=True)
    ms1, got = run({"B2_SUBBATCHES": "1"})
    same = all(np.array_equal(ref[k], got[k]) for k in ref)
    print("lane kernel, no pipeline: %.3f ms/step, identical=%s" % (ms1, same), flush=True)
    ms2, got = run({})
    same = all(np.array_equal(ref[k], got[k]) for k in ref)
    print("library defaults: %.3f ms/step (%.0f alignments/s, %.3f x), identical=%s"
          % (ms2, B / ms2 * 1e3, ms0 / ms2, same), flush=True)
    for steps in (5, 20):
        ms3, got = run({}, steps=steps, resident=True)
        same = all(np.array_equal(ref[k], got[k]) for k in ref)
        print("library defaults, B2_DEVICE_RESIDENT (calls chained), %d steps: %.3f ms/step (%.0f alignments/s, %.3f x), identical=%s"
              % (steps, ms3, B / ms3 * 1e3, ms0 / ms3, same), flush=True)
    if os.environ.get("PIPE_PROBE") == "resident":
        for env in ({"B2_VAD_SMS": "74"}, {"B2_VAD_SMS": "86"}, {"B2_SUBBATCHES": "2"}, {"B2_SUBBATCHES": "4"}):
            ms3, got = run(env, steps=20, resident=True)
            same = all(np.array_equal(ref[k], got[k]) for k in ref)
            print("resident, %s: %.3f ms/step (%.0f alignments/s, %.3f x), identical=%s"
                  % (env, ms3, B / ms3 * 1e3, ms0 / ms3, same), flush=True)
        return
    combos = []
    for sub, sms in ((2, 80), (3, 80), (4, 80)):
        combos.append({"B2_SUBBATCHES": str(sub), "B2_VAD_SMS": str(sms), "B2_VAD_BATCH": "5", "B2_VAD_EVICT_FIRST": "1"})
    if len(sys.argv) > 2:
        combos = combos[: int(sys.argv[2])]
    for env in combos:
        ms, got = run(env)
        same = all(np.array_equal(ref[k], got[k]) for k in ref)
        print("evict_first=%s sub=%2s vad_sms=%3s batch=%s: %.3f ms/step (%.0f alignments/s, %.3f x), identical=%s"
              % (env["B2_VAD_EVICT_FIRST"], env["B2_SUBBATCHES"], env["B2_VAD_SMS"], env["B2_VAD_BATCH"], ms, B / ms * 1e3,
                 ms0 / ms, same),
              flush=True)


if __name__ == "__main__":
    main()
