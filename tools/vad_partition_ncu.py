#!/usr/bin/env python
"""Launches the VAD kernel in its SM-partitioned shape (one 512-consumer CTA per SM on X SMs) so that
ncu can show why an SM cannot go faster.

    B2_VAD_CONSUMERS=512 B2_VAD_CTAS_FORCE=1 B2_VAD_STAGES=5 B2_VAD_GRID=74 \
      ncu --set full --clock-control none -k regex:vad_energy -s 2 -c 1 -o gpurun_out/r2_vad_x74 python tools/vad_partition_ncu.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffsubsync_b200 import _native  # noqa: E402


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    h = _native.Handle(0)
    n_win = B * 720000
    cls = torch.from_numpy(np.random.RandomState(0).randint(0, 3, n_win).astype(np.uint8)).cuda()
    pcm = torch.empty(n_win * 160, dtype=torch.int16, device="cuda")
    h.synth_pcm(cls.data_ptr(), n_win, 160, 5, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    out = torch.empty(n_win, dtype=torch.float32, device="cuda")
    off = np.arange(B + 1, dtype=np.int64) * 720000 * 160
    for _ in range(4):
        h.vad_energy_zcr(pcm.data_ptr(), off, 16000, 100, 0.0, 100000, out=out.data_ptr(), memspace=_native.B2_DEVICE)
    h.synchronize()


if __name__ == "__main__":
    main()
