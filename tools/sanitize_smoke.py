#!/usr/bin/env python
"""Small run of every kernel of the library for compute-sanitizer (memcheck / racecheck / synccheck):

    compute-sanitizer --tool racecheck python tools/sanitize_smoke.py

Sizes are tiny (the sanitizer slows kernels 10-100x) but cover: the TMA/mbarrier rings of both VAD
kernels (lane-group: vector path, generic path, ragged tails; lane-per-window: multi-signal batches,
one CTA reusing its ring many times); the auditok energy + tokenizer scan; both rasterisers;
boundaries; blend; the correlation kernels (float and bit-mask subtitle signals, a multi-block job,
the split-block small batch path), the run path (reference bits, run correlation), candidate selection, exact re-score, pick and the ratio
reduction; b2_sync_batch with and without the sub-batch pipeline; b2_sync_tracks_auditok (grid and search);
b2_sync_tracks_seg (overlapping and misaligned segments, both detectors, packed and float references, a video
without speech; ranges ending mid-buffer off a 16-byte boundary on the lane-per-window kernel, empty and sub-window
items, a range ending at the last sample of a buffer whose length is no multiple of 8).  Results are checked against the
oracle so that a run under the sanitizer is also a parity run.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ffsubsync_b200 import _native  # noqa: E402
from ffsubsync_b200.aligners import FFTAligner, MaxScoreAligner  # noqa: E402
from ffsubsync_b200.batch import BatchSynchronizer  # noqa: E402
from ffsubsync_b200.synth import BENCH_RATIOS, synthetic_cues  # noqa: E402
from oracle import aligner_oracle as ao  # noqa: E402
from oracle import auditok_oracle as au  # noqa: E402
from oracle import raster_oracle as ro  # noqa: E402
from oracle import vad_oracle as vo  # noqa: E402


def main():
    h = _native.get_handle(0)
    rng = np.random.RandomState(0)
    # ---- VAD: vector path, generic path (441-sample windows), ragged tail
    for fr in (16000, 44100):
        fpw = vo.frames_per_window(fr, 100)
        pcm = vo.synth_pcm(rng.randint(0, 3, 700).astype(np.uint8), fpw, seed=3)[: 700 * fpw - 5]
        got, _ = h.vad_energy_zcr(pcm, [0, len(pcm)], fr, 100, 0.0, 100000)
        assert np.array_equal(got.astype(np.float64), vo.energy_zcr_detect(pcm, 100, fr, 0.0)), fr
    # lane-per-window kernel (16 kHz and 8 kHz, aligned multi-signal batch, ragged last window) against the
    # lane-group kernel on the same input
    for fr in (16000, 8000):
        fpw = vo.frames_per_window(fr, 100)
        pcm = vo.synth_pcm(rng.randint(0, 3, 2600).astype(np.uint8), fpw, seed=5)[: 2600 * fpw - 3]
        offs = [0, fpw * 1000, fpw * 1800, len(pcm)]
        want = np.concatenate([vo.energy_zcr_detect(pcm[a:b], 100, fr, 0.0) for a, b in zip(offs[:-1], offs[1:])])
        for env in ({}, {"B2_VAD_LAYOUT": "group"}, {"B2_VAD_BATCH": "2", "B2_VAD_STAGES": "4"}):
            os.environ.update(env)
            got, _ = h.vad_energy_zcr(pcm, offs, fr, 100, 0.0, 100000)
            for k in env:
                os.environ.pop(k)
            assert np.array_equal(got.astype(np.float64), want), (fr, env)
    # ---- auditok: energy + tokenizer
    amp = np.repeat(rng.choice([0.8, 1.2], 60), rng.choice([3, 30, 120], 60))[:2000]
    pcm = np.round(rng.randn(len(amp) * 160) * 316.2 * np.repeat(amp, 160)).astype(np.int16)[:-9]
    got, _ = h.vad_auditok(pcm, [0, len(pcm)], 16000, 100, 0.25, chunk_samples=160 * 700)
    want = np.concatenate([au.auditok_detect_fast(pcm[i:i + 160 * 700].tobytes(), 100, 16000, 0.25)
                           for i in range(0, len(pcm), 160 * 700)])
    assert np.array_equal(got, want)
    # ---- rasterisers, boundaries, blend
    starts, ends = synthetic_cues(5, 300.0)
    sig, off = h.rasterize(starts, ends, None, [0, len(starts)], BENCH_RATIOS, 5, False, 100, 0.0)
    for k, r in enumerate(BENCH_RATIOS):
        assert np.array_equal(sig[off[k]:off[k + 1]].astype(np.float64) != 0, ro.rasterize(starts, ends, None, 100, 0, r)[0] != 0)
    first, last = h.first_last_nonzero(sig, off)
    assert first[0] >= 0 and last[0] > first[0]
    h.blend_signals(sig[:1000], sig[1000:2000], 2, 0.6, 0.4)
    # ---- aligner: multi-block float path, split-block small batch, ratio reduction
    ref = (rng.rand(60000) > 0.6).astype(float)
    sub = np.concatenate([np.zeros(321), ref])[:60000]
    got = FFTAligner(max_offset_samples=6000).fit_transform(ref, sub, get_score=True)
    want = ao.fft_align(ref, sub, 6000)
    assert got[1] == want[1] == -321 and abs(got[0] - want[0]) <= 1e-5 * abs(want[0])
    (s2, o2), _ = MaxScoreAligner(FFTAligner, None, 100, 60).fit_transform(ref, [sub, sub[::-1].copy()])
    assert o2 == -321
    # ---- whole path (bit-mask subtitle signals), with and without the sub-batch pipeline
    n_win = 30000
    cls = np.zeros(n_win, np.uint8)
    mask = ro.rasterize(starts, ends, None, 100, 0, 1.0)[0] != 0
    cls[200:200 + len(mask)] = mask[: n_win - 200]
    pcm = vo.synth_pcm(np.concatenate([cls, cls]), 160, seed=9)
    bs = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=60, device=0)
    cue_off = [0, len(starts), 2 * len(starts)]
    args = (pcm, [0, n_win * 160, 2 * n_win * 160], np.tile(starts, 2), np.tile(ends, 2), cue_off)
    base = bs.sync_host(*args)
    assert list(base[1]) == [200, 200] and list(base[2]) == [0, 0], base
    # sub-batch pipeline: VAD on the internal stream; with B2_VAD_SMS=1 the second sub-batch's VAD is one
    # lane-per-window CTA that reuses its ring for all 938 tiles of its 30 000 windows
    for env in ({"B2_SUBBATCHES": "2"}, {"B2_SUBBATCHES": "2", "B2_VAD_SMS": "1"}):
        os.environ.update(env)
        piped = bs.sync_host(*args)
        for k in env:
            os.environ.pop(k)
        assert all(np.array_equal(a, b) for a, b in zip(base, piped)), env
    # the run path (the default for these cue-mode calls) against the overlap-save FFT path, per ratio too
    for env in ({"B2_ALIGN_PATH": "runs"}, {"B2_ALIGN_PATH": "tiled"}):
        os.environ.update(env)
        other = bs.sync_host(*args)
        for k in env:
            os.environ.pop(k)
        assert all(np.array_equal(a, b) for a, b in zip(base, other)), env
    j_all = h.sync_batch(pcm, [0, n_win * 160, 2 * n_win * 160], 16000, 100, 0.0, 100000, -1, -1, np.tile(starts, 2),
                         np.tile(ends, 2), None, cue_off, BENCH_RATIOS, 0.0, 6000, want_all=True)
    os.environ["B2_ALIGN_PATH"] = "tiled"
    j_fft = h.sync_batch(pcm, [0, n_win * 160, 2 * n_win * 160], 16000, 100, 0.0, 100000, -1, -1, np.tile(starts, 2),
                         np.tile(ends, 2), None, cue_off, BENCH_RATIOS, 0.0, 6000, want_all=True)
    os.environ.pop("B2_ALIGN_PATH")
    assert all(np.array_equal(a, b) for a, b in zip(j_all, j_fft))
    # ---- the auditok detector inside the batched sync (energy pass + in-place tokenizer), grid and search, against
    # the per-stage composition (the reference signal is two-level at label 0, so the run path may read it)
    chunk = 160 * 7000
    ba = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=60, device=0, vad="auditok")
    got = h.sync_tracks_auditok(pcm, args[1], [0, 1], 16000, 100, 0.0, args[2], args[3], None, cue_off, BENCH_RATIOS,
                                0.0, 6000, chunk, want_all=True)
    ref64, ref_off = h.vad_auditok(pcm, args[1], 16000, 100, 0.0, chunk_samples=chunk)
    sub, sub_off = h.rasterize(args[2], args[3], None, cue_off, BENCH_RATIOS, 5, False, 100, 0.0)
    sc, of, stt = h.align_batch(ref64.astype(np.float32), ref_off, sub, sub_off, 2, 5, 6000)
    assert np.array_equal(got[3], sc) and np.array_equal(got[4], of)
    g = h.sync_tracks_auditok(pcm, args[1], [0, 1], 16000, 100, 0.0, args[2], args[3], None, cue_off, BENCH_RATIOS,
                              0.0, 6000, chunk, gss=True)
    assert np.isfinite(g[5]).all()
    ba.sync_host(*args)
    # ---- sampled segments (b2_sync_tracks_seg): overlapping 20 s segments of both videos' full decodes, one set off a
    # multiple of 8 samples (the lane-group kernel), against the composition of public calls; a silent third video
    from ffsubsync_b200.batch import segment_table
    n_pcm = int(args[1][2])
    pcm3 = np.concatenate([pcm, np.zeros(30 * 16000, np.int16)])
    off3 = np.array([0, int(args[1][1]), n_pcm, n_pcm + 30 * 16000], np.int64)
    tab = segment_table(off3, 16000, segment_count=3, segment_duration=20)
    cue3 = np.concatenate([cue_off, [cue_off[-1] + (cue_off[1] - cue_off[0])]])
    starts3, ends3 = np.concatenate([args[2], args[2][: cue_off[1]]]), np.concatenate([args[3], args[3][: cue_off[1]]])
    for det, shift in (("energy_zcr", 0), ("auditok", 0), ("energy_zcr", 3)):
        t = dict(tab, seg_lo=np.minimum(tab["seg_lo"] + shift, tab["seg_hi"]))
        bseg = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=60, device=0, vad=det)
        for env in ({}, {"B2_REF_PACKED": "0"}):
            os.environ.update(env)
            got = bseg._dispatch(pcm3, off3, np.arange(3, dtype=np.int32), starts3, ends3, cue3, None, None, False,
                                 seg=bseg._seg_refs(3, t), want_all=True, memspace=_native.B2_HOST)
            for k in env:
                os.environ.pop(k)
            assert got[2][2] == _native.B2_BEST_K_NO_SPEECH, got[2]
            ref, ref_off = bseg._reference_signals(pcm3, off3, seg=bseg._seg_refs(3, t))
            sub, sub_off = h.rasterize(starts3, ends3, None, cue3, BENCH_RATIOS, 5, False, 100, 0.0)
            sc, of, stt = h.align_batch(ref, ref_off, sub, sub_off, 3, 5, 6000)
            assert np.array_equal(got[3][:10], sc[:10]) and np.array_equal(got[4][:10], of[:10]), (det, shift, env)
    # segments on the lane-per-window kernel that end mid-buffer off a 16-byte boundary, an empty and sub-window
    # items, and a range ending at the last sample of a buffer of 16 s + 13 samples, against the segment oracle
    from oracle import segment_oracle as so
    x = rng.randint(-32768, 32768, 16000 * 16 + 13).astype(np.int16)
    lo = [0, 8008, 16000, 16800, 17600, 32000, len(x) - 4005]
    hi = [3205, 8008, 16100, 16959, 17761, 33607, len(x)]
    starts = [0, 2, 3, 4, 5, 6, 8]
    tok = dict(min_length=1, max_length=10 ** 6, max_continuous_silence=0)
    for det, kw in (("energy_zcr", dict(energy_threshold=0, z_lo=0, z_hi=160)), ("auditok", dict(chunk_samples=1000,
                                                                                                **tok))):
        with h.capture_reference(2000, 1) as cap:
            h.sync_tracks_seg(x, [0, len(x)], [0], 16000, 100, 0.0 if det == "auditok" else 0.5, [0], [10.0], [0, 7],
                              starts, lo, hi, starts3[:5], ends3[:5], None, [0, 5], [1.0], 0.0, 200,
                              detector=_native.B2_DETECTOR_AUDITOK if det == "auditok" else 0, **kw)
        want = so.segment_reference(x, 10.0, starts, lo, hi, 100, detector=det, frame_rate=16000,
                                    non_speech_label=0.0 if det == "auditok" else 0.5, **kw).astype(np.float32)
        assert cap["ref_off"][1] == len(want), det
        if cap["packed"][0]:   # auditok at label 0: two-level, the run path's bits
            from oracle import sig_oracle
            got = cap["ref"][: (len(want) + 31) // 32].view(np.uint32)
            assert np.array_equal(got, sig_oracle.packed_words(want)), det
        else:
            assert np.array_equal(cap["ref"][: len(want)], want), det
    h.synchronize()
    print("sanitize_smoke ok")


if __name__ == "__main__":
    main()
