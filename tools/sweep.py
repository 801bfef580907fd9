#!/usr/bin/env python
"""BASELINE configs[4]: signal-length x batch sweep, 1 GPU or (under torchrun) G GPUs.

    python tools/sweep.py > gpurun_out/sweep.md
    python tools/sweep.py --cells 120:4096,120:8192,10:8192
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29513 \
        tools/sweep.py --cells 120:4096,10:8192

For each duration T (minutes) and GLOBAL batch B: whole-path alignments/s (PCM resident, K = 5,
+-60 s window) and the VAD kernel's GB/s of algorithmic bytes against the measured HBM peak.  Pairs
are block-sharded over the ranks (B / G each); a shard that does not fit the PCM budget is processed
in WAVES over one resident wave of synthetic PCM (wave size printed: SURVEY.md section 8d asks for it).
Every cell checks the recovered offsets / ratios.  CUDA events on the launching stream, barrier on
both sides, max over ranks; 3 warm-up + 5 timed steps; one NCCL all-gather of the results per step.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffsubsync_b200 import _native, distributed  # noqa: E402
from ffsubsync_b200.batch import BatchSynchronizer  # noqa: E402
from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs  # noqa: E402

FPW, FR = 160, 16000
PCM_BUDGET = 55e9    # bytes of resident PCM per GPU (80 GB HBM; workspaces and signals need the rest)


def peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    return json.load(open(p))["hbm_gbs"] if os.path.exists(p) else 6650.0


def cell(minutes, B_global, bs, stream, rank, world, dev):
    dur = minutes * 60.0
    lo, hi = distributed.shard_pairs(B_global, rank, world)
    B = hi - lo
    per_pair = minutes * 60 * FR * 2
    wave = B
    while wave * per_pair > PCM_BUDGET:
        wave = (wave + 1) // 2
    n_waves = (B + wave - 1) // wave if B else 0
    wave = max(wave, 1)
    pairs = make_pairs([1000 * minutes + lo + b for b in range(wave)], dur, BENCH_RATIOS, handle=bs.handle)
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(pairs.window_class).to(dev)
    pcm = torch.empty(n_win * FPW, dtype=torch.int16, device=dev)
    bs.handle.synth_pcm(cls_d.data_ptr(), n_win, FPW, 99, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    del cls_d
    pcm_off = pairs.win_off * FPW
    out = {"best_score": torch.empty(wave, dtype=torch.float64, device=dev),
           "best_offset": torch.empty(wave, dtype=torch.int32, device=dev),
           "best_k": torch.empty(wave, dtype=torch.int32, device=dev)}
    packed = torch.zeros((max(B, 1), 3), dtype=torch.float64, device=dev)

    def step():
        for w in range(n_waves):
            bs.sync_device(pcm, pcm_off, pairs.cue_start, pairs.cue_end, pairs.cue_off, out=out)
            n = min(wave, B - w * wave)
            packed[w * wave:w * wave + n, 0] = out["best_score"][:n]
            packed[w * wave:w * wave + n, 1] = out["best_offset"][:n].to(torch.float64)
            packed[w * wave:w * wave + n, 2] = out["best_k"][:n].to(torch.float64)
        if world > 1:
            distributed.gather_pair_results(packed[:B], B_global, rank, world)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    ok = bool((out["best_offset"].cpu().numpy() == pairs.true_offset).all()
              and (out["best_k"].cpu().numpy() == pairs.true_k).all()) if B else True
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if world > 1:
        torch.distributed.barrier()
    stream.synchronize()
    a.record(stream)
    for _ in range(5):
        step()
    b.record(stream)
    torch.cuda.synchronize()
    ms = distributed.max_over_ranks(a.elapsed_time(b) / 5, dev)
    ok = distributed.max_over_ranks(0.0 if ok else 1.0, dev) == 0.0
    sig = torch.empty(n_win, dtype=torch.float32, device=dev)
    a.record(stream)
    for _ in range(5):
        bs.handle.vad_energy_zcr(pcm.data_ptr(), pcm_off, FR, 100, 0.0, 100000, out=sig.data_ptr(),
                                 memspace=_native.B2_DEVICE)
    b.record(stream)
    torch.cuda.synchronize()
    vad_ms = a.elapsed_time(b) / 5
    vad_gbs = (n_win * (2 * FPW + 4)) / (vad_ms * 1e-3) / 1e9
    del pcm, sig
    return B_global / (ms * 1e-3), ms, vad_gbs, ok, wave, n_waves


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", default="", help="comma separated minutes:batch; default: the full 1-GPU grid")
    args = ap.parse_args()
    rank, world, local_rank = distributed.init_from_env("nccl")
    distributed.bind_to_gpu_numa(local_rank)
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    bs = BatchSynchronizer(BENCH_RATIOS, FR, 100, 0.0, max_offset_seconds=60, device=local_rank)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    bs.use_torch_stream()
    pk = peak()
    if args.cells:
        cells = [tuple(int(v) for v in c.split(":")) for c in args.cells.split(",")]
    else:
        cells = [(m, B) for m in (10, 30, 60, 120, 240) for B in (1, 8, 64, 512, 4096, 8192)]
    if rank == 0:
        print("| T | N (reference FFT size) | GPUs | B (global) | per-GPU wave x waves | alignments/s | ms/step | "
              "VAD GB/s per GPU | VAD frac of %.0f GB/s | offsets ok |" % pk)
        print("|---|---|---|---|---|---|---|---|---|---|", flush=True)
    for minutes, B in cells:
        if B < world:
            continue
        n_fft = 1 << int(np.ceil(np.log2(2 * minutes * 6000)))
        rate, ms, gbs, ok, wave, n_waves = cell(minutes, B, bs, stream, rank, world, dev)
        if rank == 0:
            print("| %d min | 2^%d | %d | %d | %d x %d | %.0f | %.3f | %.0f | %.2f | %s |"
                  % (minutes, int(np.log2(n_fft)), world, B, wave, n_waves, rate, ms, gbs, gbs / pk, ok), flush=True)
        torch.cuda.empty_cache()
    if world > 1:
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
