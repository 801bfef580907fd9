#!/usr/bin/env python
"""SM-partitioning probe (VERDICT r1 item 4): the HBM-bound VAD on X SMs (one 512-consumer CTA per
SM, ring filling its shared memory) next to the FP32/shared-memory-bound correlation kernels on the
other remaining SMs (neither kernel fits beside the other on one SM, so the block scheduler keeps them
apart), on two streams, the VAD stream at high priority.

    python tools/partition_probe.py [pairs]
Prints: VAD alone vs X; align alone vs CTA cap; both together vs X.
"""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffsubsync_b200 import _native  # noqa: E402
from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs  # noqa: E402

FPW, FR = 160, 16000


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 74
    dev = torch.device("cuda", 0)
    nsm = torch.cuda.get_device_properties(dev).multi_processor_count
    h1, h2 = _native.Handle(0), _native.Handle(0)
    s1, s2 = torch.cuda.Stream(priority=-1), torch.cuda.Stream()
    h1.set_stream(s1.cuda_stream)
    h2.set_stream(s2.cuda_stream)
    pairs = make_pairs(list(range(50, 50 + B)), 7200.0, BENCH_RATIOS, handle=h1)
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(pairs.window_class).to(dev)
    pcm = torch.empty(n_win * FPW, dtype=torch.int16, device=dev)
    h1.synth_pcm(cls_d.data_ptr(), n_win, FPW, 5, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    pcm_off = pairs.win_off * FPW
    ref = torch.empty(n_win, dtype=torch.float32, device=dev)
    ref2 = torch.empty(n_win, dtype=torch.float32, device=dev)
    K = len(BENCH_RATIOS)
    lengths = h1.rasterize_lengths(pairs.cue_end, pairs.cue_off, BENCH_RATIOS, K, False, 100)
    sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
    sc = torch.empty(B * K, dtype=torch.float64, device=dev)
    of = torch.empty(B * K, dtype=torch.int32, device=dev)
    st = torch.empty(B * K, dtype=torch.int32, device=dev)
    gb = (pcm.numel() * 2 + n_win * 4) / 1e9

    def vad(dst=ref2):
        h1.vad_energy_zcr(pcm.data_ptr(), pcm_off, FR, 100, 0.0, 100000, out=dst.data_ptr(),
                          memspace=_native.B2_DEVICE)

    def align():
        h2.align_batch(ref.data_ptr(), pairs.win_off, sub.data_ptr(), sub_off, B, K, 6000, score=sc.data_ptr(),
                       offset=of.data_ptr(), status=st.data_ptr(), memspace=_native.B2_DEVICE)

    vad(ref)
    h1.synchronize()
    h2.rasterize(pairs.cue_start, pairs.cue_end, None, pairs.cue_off, BENCH_RATIOS, K, False, 100, 0.0,
                 out=sub.data_ptr(), out_off=sub_off, memspace=_native.B2_DEVICE)
    for _ in range(2):
        align()
    torch.cuda.synchronize()

    def timed(fns, reps=4):
        for f in fns:
            f()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            for f in fns:
                f()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps * 1e3

    for k in ("B2_VAD_CONSUMERS", "B2_VAD_GRID", "B2_VAD_STAGES", "B2_VAD_CTAS_FORCE", "B2_CORR_MAX_CTAS"):
        os.environ.pop(k, None)
    tv0, ta0 = timed([vad]), timed([align])
    print("pairs=%d default: vad alone %.3f ms (%.0f GB/s), align alone %.3f ms, sum %.3f ms"
          % (B, tv0, gb / tv0 * 1e3, ta0, tv0 + ta0), flush=True)
    print("--- VAD alone, one CTA per SM on X SMs")
    for consumers, stages in (("512", "5"), ("512", "4"), ("256", "10"), ("256", "8")):
        for X in (nsm, 120, 100, 90, 80, 74, 64, 48):
            os.environ.update(B2_VAD_CONSUMERS=consumers, B2_VAD_STAGES=stages, B2_VAD_CTAS_FORCE="1",
                              B2_VAD_GRID=str(X))
            tv = timed([vad])
            print("vad consumers=%s stages=%s X=%3d: %.3f ms = %.0f GB/s = %.1f GB/s per SM"
                  % (consumers, stages, X, tv, gb / tv * 1e3, gb / tv * 1e3 / X), flush=True)
    for k in ("B2_VAD_CONSUMERS", "B2_VAD_GRID", "B2_VAD_STAGES", "B2_VAD_CTAS_FORCE"):
        os.environ.pop(k, None)
    print("--- both together: VAD on X SMs (512 consumers, 5 stages), correlation on the rest")
    for X in (60, 68, 74, 80, 86, 92, 100):
        os.environ.update(B2_VAD_CONSUMERS="512", B2_VAD_STAGES="5", B2_VAD_CTAS_FORCE="1", B2_VAD_GRID=str(X),
                          B2_CORR_MAX_CTAS=str(nsm - X))
        tv = timed([vad])
        ta = timed([align])
        tb = timed([vad, align])
        print("X=%3d: vad alone %.3f ms, align alone (ref_spectra on %d CTAs) %.3f ms, both %.3f ms  (default sum %.3f)"
              % (X, tv, nsm - X, ta, tb, tv0 + ta0), flush=True)


if __name__ == "__main__":
    main()
