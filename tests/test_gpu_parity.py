"""GPU parity tests (run on an H100): the CUDA path, called through the C ABI / the
reference-shaped Python API, against the oracle and the committed golden fixtures.

Bars: integer/index results bit-exact; correlation scores within 1e-5 relative (north_star)."""
import math
from datetime import timedelta

import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

SCORE_RTOL = 1e-5


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _score_ok(got, want):
    if math.isinf(want) or math.isinf(got):
        return got == want
    return abs(got - want) <= SCORE_RTOL * max(abs(want), 1e-3) + 1e-6


# =============================================================================== VAD (K1)

@pytest.mark.parametrize("frame_rate", [16000, 48000, 44100, 8000, 32000])
@pytest.mark.parametrize("label", [0.0, 0.5])
def test_vad_matches_oracle(handle, frame_rate, label):
    from ffsubsync_b200.speech_transformers import _make_energy_zcr_detector
    fpw = vo.frames_per_window(frame_rate, 100)
    rng = np.random.RandomState(frame_rate % 97)
    cls = rng.randint(0, 3, 3000).astype(np.uint8)
    pcm = vo.synth_pcm(cls, fpw, seed=11)
    # perturb a few windows so energies land near the threshold and the band edges
    pcm[: fpw * 50] = (pcm[: fpw * 50].astype(np.int32) * rng.uniform(0.02, 0.2)).astype(np.int16)
    det = _make_energy_zcr_detector(100, frame_rate, label)
    for cut in (len(pcm), len(pcm) - 7, fpw * 10 + 1, 3, 0):
        chunk = pcm[:cut].tobytes()
        want = vo.energy_zcr_detect(chunk, 100, frame_rate, label)
        got = det(np.frombuffer(chunk, np.uint8)) if cut else det(b"")
        assert got.dtype == np.float64 and np.array_equal(got, want), (frame_rate, cut)


def test_vad_batch_ragged_and_thresholds(handle):
    rng = np.random.RandomState(5)
    fpw = 160
    sigs = [vo.synth_pcm(rng.randint(0, 3, n).astype(np.uint8), fpw, seed=n)[: n * fpw - r]
            for n, r in ((400, 0), (1, 0), (37, 5), (0, 0), (256, 159), (64, 1))]
    sigs = [s if len(s) else np.zeros(0, np.int16) for s in sigs]
    off = np.concatenate([[0], np.cumsum([len(s) for s in sigs])])
    for thr, zlo, zhi in ((100000, -1, -1), (10, 0, 200), (100000, 2, 3), (5 * 10**7, 0, 160)):
        out, out_off = handle.vad_energy_zcr(np.concatenate(sigs), off, 16000, 100, 0.25, thr, zlo, zhi)
        for b, s in enumerate(sigs):
            want = vo.energy_zcr_detect(s, 100, 16000, 0.25, thr, None if zlo < 0 else zlo,
                                        None if zhi < 0 else zhi)
            assert np.array_equal(out[out_off[b]:out_off[b + 1]].astype(np.float64), want), (b, thr)


def test_vad_full_scale_samples(handle):
    # int16 extremes: energy needs 64-bit accumulation (160 * 32768^2 > 2^32)
    pcm = np.full(160 * 4, -32768, dtype=np.int16)
    pcm[160:320] = 32767
    pcm[320:480:2] = 32767
    out, _ = handle.vad_energy_zcr(pcm, [0, len(pcm)], 16000, 100, 0.0, 100000, 0, 160)
    assert np.array_equal(out.astype(np.float64), vo.energy_zcr_detect(pcm, 100, 16000, 0.0, 100000, 0, 160))


# (frame_rate, samples per signal): up to 8 two-hour signals, where every CTA of the lane-per-window kernel
# reuses its ring many times
_LANE_CASES = {"%d-%dx%d" % (fr, b, nw): (fr, [nw * (fr // 100)] * b) for fr, b, nw in (
    (16000, 1, 64), (16000, 1, 65), (16000, 1, 640), (16000, 1, 5000), (16000, 3, 20000), (16000, 2, 200000),
    (16000, 8, 720000), (8000, 2, 100000))}
# window counts that are no multiple of a tile, partial last windows, an empty signal and a buffer end that is
# not 16-byte aligned; every signal starts 16-byte aligned, so the lane-per-window kernel still takes the batch
_LANE_CASES["16000-ragged"] = (16000, [160 * 1000 + 88, 0, 160 * 37 - 72, 160 * 4001, 160 + 8, 160 * 777 - 5])


@pytest.mark.parametrize("frame_rate, lengths", list(_LANE_CASES.values()), ids=list(_LANE_CASES))
def test_vad_lane_kernel_equals_lane_group_kernel(handle, monkeypatch, frame_rate, lengths):
    """The default VAD (lane-per-window kernel at 8 and 16 kHz) and the lane-group kernel
    (B2_VAD_LAYOUT=group) give bit-identical windows on the same device PCM, and both equal plain
    torch arithmetic on that PCM."""
    import torch
    from ffsubsync_b200 import _native
    fpw = frame_rate // 100
    pcm_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    n_out = sum(-(-n // fpw) for n in lengths)
    n_syn = -(-int(pcm_off[-1]) // fpw)
    cls = torch.from_numpy(np.random.RandomState(n_syn % 9973).randint(0, 3, n_syn).astype(np.uint8)).cuda()
    pcm = torch.empty(n_syn * fpw, dtype=torch.int16, device="cuda")
    lane, group = (torch.full((n_out,), -7.0, dtype=torch.float32, device="cuda") for _ in range(2))
    torch.cuda.synchronize()   # the handle launches on its own stream
    handle.synth_pcm(cls.data_ptr(), n_syn, fpw, 5, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    handle.vad_energy_zcr(pcm.data_ptr(), pcm_off, frame_rate, 100, 0.5, 100000, out=lane.data_ptr(),
                          memspace=_native.B2_DEVICE)
    monkeypatch.setenv("B2_VAD_LAYOUT", "group")
    handle.vad_energy_zcr(pcm.data_ptr(), pcm_off, frame_rate, 100, 0.5, 100000, out=group.data_ptr(),
                          memspace=_native.B2_DEVICE)
    handle.synchronize()
    assert torch.equal(lane, group)
    want = []
    for a, b in zip(pcm_off[:-1].tolist(), pcm_off[1:].tolist()):
        n_full = (b - a) // fpw
        x = pcm[a:a + n_full * fpw].view(n_full, fpw)
        e = x.to(torch.int64).square().sum(1)
        z = ((x[:, 1:] < 0) != (x[:, :-1] < 0)).sum(1)
        speech = (e >= fpw * 100000) & (z <= (3 * fpw) // 8)
        want.append(speech.float() * 0.5 + 0.5)   # 1.0 or the non-speech label 0.5
        if (b - a) % fpw:
            want.append(torch.full((1,), 0.5, device="cuda"))   # partial last window: non-speech
    assert torch.equal(lane, torch.cat(want))


def test_device_memspace_is_ordered_on_the_callers_stream(handle):
    """B2_DEVICE calls only enqueue work on the stream given to b2_set_stream; torch ops queued on
    the same stream right after must see the results (no host synchronisation in between).  Covers
    an explicit torch stream and torch's default stream (handle 0 -> cudaStreamLegacy)."""
    import torch
    from ffsubsync_b200 import _native
    cls = np.random.RandomState(9).randint(0, 3, 200000).astype(np.uint8)
    want = vo.energy_zcr_detect(vo.synth_pcm(cls, 160, seed=4), 100, 16000, 0.0)
    try:
        for stream in (torch.cuda.Stream(), torch.cuda.default_stream()):
            with torch.cuda.stream(stream):
                handle.set_stream(stream.cuda_stream)
                cls_d = torch.from_numpy(cls).cuda()
                pcm = torch.empty(len(cls) * 160, dtype=torch.int16, device="cuda")
                out = torch.full((len(cls),), -7.0, dtype=torch.float32, device="cuda")
                handle.synth_pcm(cls_d.data_ptr(), len(cls), 160, 4, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
                handle.vad_energy_zcr(pcm.data_ptr(), [0, pcm.numel()], 16000, 100, 0.0, 100000,
                                      out=out.data_ptr(), memspace=_native.B2_DEVICE)
                total = out.double().sum()      # queued behind our kernels on the same stream
                got = out.cpu().numpy()
            assert np.array_equal(got.astype(np.float64), want) and float(total) == want.sum()
    finally:
        handle.set_stream(None)


def test_fused_detector_blend_kats(handle):
    """The reference's tests/test_vad_fused.py:21-54 with stub constituents: min / max / 0.6-0.4
    blend, default strategy, common-length clip, unknown strategy."""
    from ffsubsync_b200.speech_transformers import VideoSpeechTransformer, _make_fused_detector

    def stubs(first, second):
        return (lambda *a: (lambda seg: np.asarray(first, dtype=float)),
                lambda *a: (lambda seg: np.asarray(second, dtype=float)))

    # the reference weights silero (here: first) 0.6 and webrtc (second) 0.4
    silero, webrtc = [1.0, 0.0, 0.0], [1.0, 1.0, 0.0]
    assert list(_make_fused_detector(100, 48000, 0.0, "intersection", stubs(silero, webrtc))(b"")) == [1.0, 0.0, 0.0]
    assert list(_make_fused_detector(100, 48000, 0.0, "union", stubs(silero, webrtc))(b"")) == [1.0, 1.0, 0.0]
    assert np.allclose(_make_fused_detector(100, 48000, 0.0, "weighted", stubs([0.0, 1.0], [1.0, 0.0]))(b""), [0.4, 0.6])
    assert np.allclose(_make_fused_detector(100, 48000, 0.0, factories=stubs([0.0], [1.0]))(b""), [0.4])
    assert len(_make_fused_detector(100, 48000, 0.0, "union", stubs([1.0, 1.0], [1.0, 1.0, 1.0]))(b"")) == 2
    with pytest.raises(ValueError, match="unknown fused VAD strategy"):
        _make_fused_detector(100, 48000, 0.0, "bogus")
    # real constituents on PCM: energy/ZCR (0.6) + energy-only (0.4); loud hiss passes only the latter
    cls = np.array([0, 1, 2, 1, 0, 2], dtype=np.uint8)
    pcm = vo.synth_pcm(cls, 160, seed=8).tobytes()
    t = VideoSpeechTransformer("fused", 100, 16000, 0.0).fit(pcm)
    assert np.allclose(t.transform(), [0.0, 1.0, 0.4, 1.0, 0.0, 0.4])
    assert list(VideoSpeechTransformer("fused:intersection", 100, 16000, 0.0).fit(pcm).transform()) == [0, 1, 0, 1, 0, 0]
    rng = np.random.RandomState(1)
    a, b = rng.rand(100003).astype(np.float32), rng.rand(100003).astype(np.float32)
    got = handle.blend_signals(a, b, 2, 0.6, 0.4)
    assert np.array_equal(got, (0.6 * a.astype(np.float64) + 0.4 * b.astype(np.float64)).astype(np.float32))


def test_synth_pcm_matches_numpy_replay(handle):
    cls = np.random.RandomState(2).randint(0, 3, 500).astype(np.uint8)
    got = handle.synth_pcm(cls, len(cls), 160, seed=77)
    assert np.array_equal(got, vo.synth_pcm(cls, 160, seed=77))


def test_video_speech_transformer_chunk_protocol(handle):
    """Chunked reads + progress callbacks as in the reference's loop (100 s per chunk)."""
    from ffsubsync_b200.speech_transformers import VideoSpeechTransformer
    fr = 16000
    cls = np.random.RandomState(3).randint(0, 2, 25000).astype(np.uint8)  # 250 s
    pcm = vo.synth_pcm(cls, 160, seed=5)
    seen = []
    t = VideoSpeechTransformer("energy_zcr", 100, fr, 0.0, progress_handler=seen.append)
    t.fit(pcm.tobytes() + b"\x01")  # odd trailing byte is ignored
    want = vo.energy_zcr_detect(pcm.tobytes(), 100, fr, 0.0)
    assert np.array_equal(t.transform(), want)
    assert [round(p.processed_seconds) for p in seen] == [100, 200, 250]
    assert seen[-1].fraction == 1.0
    with pytest.raises(ValueError, match="unknown vad"):
        VideoSpeechTransformer("webrtc", 100, fr, 0.0).fit(b"\0\0")
    with pytest.raises(ValueError, match="Unable to detect speech"):
        VideoSpeechTransformer("energy", 100, fr, 0.0).fit(b"")


def test_more_than_65535_signals_in_one_call(handle):
    """The rasterisers index signals with grid.y (limit 65 535): larger batches are split into
    several launches.  66 000 one-cue signals through b2_rasterize, and 33 000 pairs x 2 ratios
    through b2_sync_batch (bit-mask path), spot-checked against the oracle."""
    rs = np.random.RandomState(4)
    J = 66000
    st = rs.uniform(0.0, 0.5, J)
    en = st + rs.uniform(0.05, 0.4, J)
    out, off = handle.rasterize(st, en, None, np.arange(J + 1), [1.0], 1, False, 100, 0.0)
    for j in list(range(0, J, 1777)) + [65534, 65535, 65536, J - 1]:
        want = ro.rasterize(st[j:j + 1], en[j:j + 1], None, 100, 0, 1.0)[0]
        assert np.array_equal(out[off[j]:off[j + 1]].astype(np.float64), want), j
    B, fpw, nwin = 33000, 160, 12
    cls = np.zeros(B * nwin, np.uint8)
    delta = rs.randint(0, 4, B)
    for b in range(B):                                   # speech windows [3+d, 7+d) of 12
        cls[b * nwin + 3 + delta[b]: b * nwin + 7 + delta[b]] = 1
    pcm = handle.synth_pcm(cls, len(cls), fpw, 3)
    cs, ce = np.full(B, 0.03), np.full(B, 0.07)          # subtitle speech frames [3, 7)
    ratios = [1.0, 0.5]
    bs, bo, bk, a_s, a_o = handle.sync_batch(pcm, np.arange(B + 1) * nwin * fpw, 16000, 100, 0.0, 100000,
                                             -1, -1, cs, ce, None, np.arange(B + 1), ratios, 0.0, 8,
                                             want_all=True)
    for b in list(range(0, B, 997)) + [32767, 32768, B - 1]:
        ref_sig = vo.energy_zcr_detect(pcm[b * nwin * fpw:(b + 1) * nwin * fpw], 100, 16000, 0.0)
        # tiny signals tie exactly at several offsets: the oracle's exact-arithmetic argmax is the
        # defined answer (DESIGN.md section 2)
        results = [ao.exact_align(ref_sig, ro.rasterize(cs[b:b + 1], ce[b:b + 1], None, 100, 0, r)[0], 8)
                   for r in ratios]
        wk = ao.max_score_select(results, 8)
        assert (bk[b], bo[b]) == (wk, results[wk][1]), b
        assert [int(a_o[2 * b]), int(a_o[2 * b + 1])] == [results[0][1], results[1][1]]
        assert _score_ok(bs[b], results[wk][0])


def test_align_batch_more_than_65535_tiled_jobs(handle):
    """b2_align_batch on the overlap-save path with 17 000 pairs x 4 ratios = 68 000 (pair, ratio) jobs:
    every per-job launch indexes jobs with grid.x (grid.y stops at 65 535).  Random binary signals of a
    few hundred frames, so the float64 correlation rounds to the exact integer scores; every job against
    the oracle's argmax (ties -> largest offset)."""
    rs = np.random.RandomState(65536)
    B, K, mos = 17000, 4, 150
    refs = [(rs.rand(rs.randint(300, 400)) > 0.5).astype(np.float32) for _ in range(B)]
    subs = [(rs.rand(rs.randint(200, 300)) > 0.5).astype(np.float32) for _ in range(B * K)]
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])])
    sub_off = np.concatenate([[0], np.cumsum([len(s) for s in subs])])
    score, off, st = handle.align_batch(np.concatenate(refs), ref_off, np.concatenate(subs), sub_off, B, K, mos)
    assert len(off) == B * K and np.all(st == 0)
    for j, sub in enumerate(subs):
        conv = np.round(ao.correlation(refs[j // K], sub))
        N, S = len(conv), len(sub)
        lo, hi = ao.surviving_index_range(N, S, mos)
        idx = lo + int(np.argmax(conv[lo:hi]))
        assert (off[j], score[j]) == (N - 1 - idx - S, conv[idx]), j


def test_vad_stream_matches_per_chunk_detection(handle):
    """b2_vad_stream_*: every pushed chunk is detected like one detector call (ceil(n/fpw) windows,
    partial last window non-speech, odd trailing byte dropped); the ring (3 slots) wraps, chunk
    sizes change, results come back in push order."""
    from ffsubsync_b200 import _native
    fr, fpw = 16000, 160
    cls = np.random.RandomState(31).randint(0, 3, 9000).astype(np.uint8)
    raw = vo.synth_pcm(cls, fpw, seed=3).tobytes()
    sizes = [320 * 700, 320 * 700 + 1, 7, 0, 320 * 2100 + 38, 320, 320 * 1500 - 5, 2, 320 * 900, 1]
    chunks, pos = [], 0
    for n in sizes:
        chunks.append(raw[pos:pos + n])
        pos += n
    chunks.append(raw[pos:])
    want = np.concatenate([vo.energy_zcr_detect(c[:len(c) // 2 * 2], 100, fr, 0.25) for c in chunks if len(c) >= 2])
    handle.vad_stream_begin(fr, 100, 0.25, 100000)
    with pytest.raises(_native.NativeError, match="already open"):
        handle.vad_stream_begin(fr, 100, 0.25, 100000)
    for i, c in enumerate(chunks):
        handle.vad_stream_push(np.frombuffer(c, np.uint8) if i % 2 else c)
    got = handle.vad_stream_end()
    assert got.dtype == np.float32 and np.array_equal(got.astype(np.float64), want)
    with pytest.raises(_native.NativeError, match="not open"):
        handle.vad_stream_push(b"\0\0")
    handle.vad_stream_begin(fr, 100, 0.0, 100000)        # empty stream, and a second use of the handle
    assert len(handle.vad_stream_end()) == 0
    # band parameters are honoured (energy-only variant)
    handle.vad_stream_begin(fr, 100, 0.0, 100000, 0, fpw)
    handle.vad_stream_push(raw)
    assert np.array_equal(handle.vad_stream_end().astype(np.float64),
                          vo.energy_zcr_detect(raw, 100, fr, 0.0, 100000, 0, fpw))


def test_multi_segment_transformer_batched_vs_threads_vs_oracle(handle, tmp_path):
    """MultiSegmentVideoSpeechTransformer on raw PCM: the one-launch batched path, the reference's
    thread-pool path (one VideoSpeechTransformer per window, -ss/-t emulated on the raw PCM) and the
    oracle VAD placed by hand must agree; the sparse signal then aligns like the full one."""
    from ffsubsync_b200.speech_transformers import MultiSegmentVideoSpeechTransformer
    fr, dur = 16000, 333.37
    n_win = int(dur * 100)
    cls = np.repeat(np.random.RandomState(21).randint(0, 2, n_win // 25 + 1), 25)[:n_win].astype(np.uint8)
    pcm = vo.synth_pcm(cls, 160, seed=7)
    pcm = np.concatenate([pcm, np.full(59, 9000, np.int16)])       # ragged tail (partial last window)
    total = len(pcm) / fr
    full = vo.energy_zcr_detect(pcm.tobytes(), 100, fr, 0.0)

    def make(**kw):
        return MultiSegmentVideoSpeechTransformer("energy_zcr", 100, fr, 0.0, segment_count=5,
                                                  segment_duration=40, **kw)

    batched = make().fit(pcm).transform()
    want = np.zeros(int(total * 100) + 2)
    t = make()
    starts = t._segment_starts(total)
    assert len(starts) == 5
    for s in starts:
        seg = vo.energy_zcr_detect(pcm[s * fr:(s + 40) * fr].tobytes(), 100, fr, 0.0)
        end = min(s * 100 + len(seg), len(want))
        want[s * 100:end] = seg[:end - s * 100]
    assert np.array_equal(batched, want)
    for s in starts:                                                # windows sit at their true positions
        assert np.array_equal(batched[s * 100:s * 100 + 4000], full[s * 100:s * 100 + 4000])
    # thread-pool path: instance-level extractor forces it; .pcm file source
    path = str(tmp_path / "ref.pcm")
    pcm.tofile(path)
    t2 = make(parallel_workers=3)
    t2._extract_segment_speech = lambda fname, start: MultiSegmentVideoSpeechTransformer._extract_segment_speech(t2, fname, start)
    assert np.array_equal(t2.fit(path).transform(), want)
    assert np.array_equal(make().fit(path).transform(), want)      # batched from the file (memmap)
    fused = MultiSegmentVideoSpeechTransformer("fused:union", 100, fr, 0.0, segment_count=5,
                                               segment_duration=40).fit(pcm).transform()
    assert np.all((fused > 0) >= (want > 0)) and len(fused) == len(want)   # union with energy-only: superset
    # the sparse reference recovers a planted shift like the full reference does
    from ffsubsync_b200.aligners import FFTAligner
    sub = np.concatenate([np.zeros(321), full])[:len(full)]
    assert FFTAligner(6000).fit_transform(batched, sub) == -321
    assert FFTAligner(6000).fit_transform(full, sub) == -321


# ========================================================================= rasteriser (K2, K7)

def test_raster_matches_reference_fixtures(handle, golden, gf):
    done = 0
    for c in golden["raster"]:
        starts, ends = cases.synthetic_cues(c["seed"], c["duration"])
        out, off = handle.rasterize(starts, ends, None, [0, len(starts)], [c["ratio"]], 1, False, 100,
                                    float(c["start_seconds"]))
        assert len(out) == c["length"] == off[-1], c["ratio"]
        levels, rs, re_ = cases.run_lengths(out)
        assert rs == c["run_starts"] and re_ == c["run_stops"], (c["seed"], c["ratio"])
        assert [np.float32(v) for v in c["levels"]] == [np.float32(v) for v in levels]
        done += 1
    assert done >= 30


def test_raster_batch_k_ratios_and_boundaries(handle):
    grid = cases.ratio_grid()
    cue_sets = [cases.synthetic_cues(s, d) for s, d in ((1, 300.0), (2, 45.0), (3, 900.0))]
    starts = np.concatenate([c[0] for c in cue_sets])
    ends = np.concatenate([c[1] for c in cue_sets])
    cue_off = np.concatenate([[0], np.cumsum([len(c[0]) for c in cue_sets])])
    keep = (np.arange(len(starts)) % 7 != 3).astype(np.uint8)
    out, off = handle.rasterize(starts, ends, keep, cue_off, grid, len(grid), False, 100, 0.0)
    first, last = handle.first_last_nonzero(out, off)
    for b, (st, en) in enumerate(cue_sets):
        kb = keep[cue_off[b]:cue_off[b + 1]].astype(bool)
        for k, r in enumerate(grid):
            want, _, sf, ef = ro.rasterize(st, en, kb, 100, 0, r)
            j = b * len(grid) + k
            got = out[off[j]:off[j + 1]]
            assert len(got) == len(want)
            assert np.array_equal(got != 0, want != 0)
            assert np.allclose(got[got != 0], np.float32(min(1.0 / r, 1.0)))
            assert (first[j], last[j]) == (sf, ef)


def test_subtitle_speech_transformer_kat(handle, golden, gf):
    """tests/test_subtitles.py fake_srt timings through the reference-shaped classes."""
    from ffsubsync_b200.sklearn_shim import make_pipeline
    from ffsubsync_b200.speech_transformers import SubtitleSpeechTransformer
    from ffsubsync_b200.subtitle_transformers import Cue, SubtitleScaler
    k = golden["raster_kat"]
    for c in k["cases"]:
        subs = [Cue(timedelta(seconds=k["starts"][i]), timedelta(seconds=k["ends"][i]), k["contents"][i])
                for i in c["cue_idx"]]
        tr = SubtitleSpeechTransformer(sample_rate=c["sample_rate"], start_seconds=c["start_seconds"])
        x = tr.fit(subs).transform()
        assert x.dtype == np.float64 and len(x) == c["length"]
        assert cases.run_lengths(x) == (c["levels"], c["run_starts"], c["run_stops"])
        assert tr.max_time_ == gf(c["max_time"])
        assert (tr.start_frame_, tr.end_frame_) == (c["start_frame"], c["end_frame"])
    # scaler + transformer == fused oracle for a non-unit ratio, incl. the float64 level
    starts, ends = cases.synthetic_cues(21, 120.0)
    subs = [Cue(timedelta(seconds=s), timedelta(seconds=e), "hi") for s, e in zip(starts, ends)]
    r = 25.0 / 24.0
    pipe = make_pipeline(SubtitleScaler(r), SubtitleSpeechTransformer(100, 0, r))
    got = pipe.fit_transform(subs)
    want, max_time, sf, ef = ro.rasterize(starts, ends, None, 100, 0, r)
    assert np.array_equal(got, want) and pipe[-1].num_frames == ef - sf


# ============================================================================== aligner (K3-K5)

def test_align_kats(handle, golden, gf):
    from ffsubsync_b200.aligners import FFTAligner, MaxScoreAligner
    for sub, ref, off in [("111001", "11001", -1), ("1001", "1001", 0), ("10010", "01001", 1)]:
        assert FFTAligner().fit_transform(ref, sub) == off
        assert MaxScoreAligner(FFTAligner).fit_transform(ref, sub)[0][1] == off
        assert MaxScoreAligner(FFTAligner()).fit_transform(ref, sub)[0][1] == off
    for c in golden["kats"]:
        score, off = FFTAligner(c["mos"]).fit_transform(c["ref"], c["sub"], get_score=True)
        want = gf(c["score"])
        # exact ties (e.g. the all-negative case) are decided by float64 round-off in the
        # reference; the GPU path breaks them like np.argmax on exact values
        es, eo = ao.exact_align(c["ref"], c["sub"], c["mos"])
        assert off == eo, c
        assert _score_ok(score, want), (score, want)
        if abs(es - want) < 1e-6 and off != c["offset"]:
            pytest.fail("offset differs from the reference without a tie: %r" % (c,))


def test_align_empty_inputs_raise(handle):
    from ffsubsync_b200.aligners import FailedToFindAlignmentException, FFTAligner
    for ref, sub in ((np.array([]), np.array([1, 0, 1])), (np.array([1, 0, 1]), np.array([])),
                     (np.array([]), np.array([]))):
        with pytest.raises(FailedToFindAlignmentException, match="empty speech data"):
            FFTAligner().fit(ref, sub)


def test_align_small_cases_batched(handle, golden, gf):
    """240 random small cases (binary / two-level / float signals x mask regimes) in few calls."""
    by_mos = {}
    for c in golden["small"]:
        by_mos.setdefault(c["mos"], []).append(c)
    n_checked = n_tie = 0
    for mos, group in by_mos.items():
        refs, subs = [], []
        for c in group:
            ref, sub, m = cases.small_align_case(c["seed"])
            refs.append(ref)
            subs.append(sub)
        ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])])
        sub_off = np.concatenate([[0], np.cumsum([len(s) for s in subs])])
        score, offset, status = handle.align_batch(np.concatenate(refs), ref_off, np.concatenate(subs),
                                                   sub_off, len(group), 1, mos)
        for i, c in enumerate(group):
            want = gf(c["score"])
            # the GPU path is exact on the float32 values it is handed
            es, eo = ao.exact_align(refs[i].astype(np.float32), subs[i].astype(np.float32), mos)
            assert offset[i] == eo, (c, offset[i], eo)
            assert _score_ok(score[i], es)
            if offset[i] != c["offset"]:
                # only legitimate when the reference's own maximum is a float64 near-tie
                assert abs(ao.exact_score(refs[i], subs[i], c["offset"]) - es) < 1e-6, c
                n_tie += 1
            else:
                assert _score_ok(score[i], want)
            n_checked += 1
    assert n_checked == 240 and n_tie < 40


@pytest.mark.parametrize("n", [6000, 60000, 360000, 720000])
def test_align_shifted_pairs(handle, golden, gf, n):
    from ffsubsync_b200.aligners import FFTAligner
    ref, sub = cases.shifted_pair(n)
    for c in golden["shifted"]:
        if c["n"] != n:
            continue
        score, off = FFTAligner(c["mos"]).fit_transform(ref, sub, get_score=True)
        assert off == c["offset"] == -1234
        assert score == n - 1234  # binary signals: the exact integer
        assert _score_ok(score, gf(c["score"]))


def test_align_unmasked_two_hours(handle, golden, gf):
    """FFTAligner() with no mask on the 2 h config: every one of the 2^21 offsets is a candidate."""
    from ffsubsync_b200.aligners import FFTAligner
    ref, sub = cases.shifted_pair(720000)
    score, off = FFTAligner().fit_transform(ref, sub, get_score=True)
    want = [c for c in golden["shifted"] if c["n"] == 720000 and c["mos"] is None][0]
    assert off == want["offset"] and score == 720000 - 1234


def test_align_four_hours_unmasked_and_wide_mask(handle, golden, gf):
    """n = 1 440 000 (N = 2^22): FFTAligner() and a 1000 s mask go through the large-FFT path, the
    +-60 s mask through the overlap-save path; all three equal the reference."""
    from ffsubsync_b200.aligners import FFTAligner
    ref, sub = cases.shifted_pair(1440000)
    for c in golden["shifted"]:
        if c["n"] != 1440000:
            continue
        score, off = FFTAligner(c["mos"]).fit_transform(ref, sub, get_score=True)
        assert off == c["offset"] == -1234 and score == 1440000 - 1234, c


def test_wide_window_cases_both_paths(handle, golden, gf, monkeypatch):
    """The wide-window fixtures (unmasked / very wide masks, lopsided lengths, float levels, R + S at
    and above a power of two) through the large-FFT path and through the tiled overlap-save path:
    both equal the reference (offset exact, score <= 1e-5)."""
    from ffsubsync_b200.aligners import FFTAligner
    for path in ("big", "tiled"):
        monkeypatch.setenv("B2_ALIGN_PATH", path)
        for c in golden["wide"]:
            kw = dict(c["case"])
            kw.pop("mos_list")
            ref, sub = cases.wide_pair(**kw)
            score, off = FFTAligner(c["mos"]).fit_transform(ref, sub, get_score=True)
            assert off == c["offset"], (path, c, off)
            assert _score_ok(score, gf(c["score"])), (path, c, score)
    monkeypatch.delenv("B2_ALIGN_PATH")


def test_unmasked_batch_mixed_sizes_vs_oracle(handle):
    """b2_align_batch unmasked with pairs of different padded lengths (2^17, 2^18, 2^19) and K = 3
    subtitle signals per pair whose lengths straddle a power of two (the pair's transform takes the
    largest padded length; every job keeps its own index semantics), an empty and a constant signal."""
    rng = np.random.RandomState(12)
    refs, subs = [], []
    for R, S_list, shift in ((60000, (70000, 71000, 72000), 300), (131000, (131000, 131072, 131200), -2500),
                             (250000, (200000, 262144, 270000), 40000)):
        ref = (rng.rand(R) > 0.5).astype(np.float32)
        refs.append(ref)
        for S in S_list:
            idx = np.arange(S) - shift
            ok = (idx >= 0) & (idx < R)
            subs.append(np.where(ok, ref[np.clip(idx, 0, R - 1)], rng.rand(S) > 0.5).astype(np.float32))
    refs.append(np.ones(70000, np.float32))
    subs += [np.zeros(0, np.float32), np.ones(65000, np.float32), (rng.rand(66000) > 0.5).astype(np.float32)]
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])])
    sub_off = np.concatenate([[0], np.cumsum([len(s) for s in subs])])
    score, off, st = handle.align_batch(np.concatenate(refs), ref_off, np.concatenate(subs), sub_off, 4, 3, None)
    from ffsubsync_b200 import _native
    for b in range(4):
        for k in range(3):
            j = 3 * b + k
            if len(subs[j]) == 0:
                assert st[j] & _native.ALIGN_EMPTY
                continue
            ws, wo = ao.fft_align(refs[b], subs[j], None)
            if b == 3 and k == 1:      # constant x constant: a plateau of exact ties, more than the re-score budget
                assert st[j] & _native.ALIGN_CAND_OVERFLOW or off[j] == wo
                continue
            assert off[j] == wo and _score_ok(score[j], ws), (b, k, off[j], wo, score[j], ws)


def test_sync_batch_unmasked_vs_oracle(handle):
    """b2_sync_batch with max_offset_seconds=None: bit-mask subtitle signals through the large-FFT path."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    bs = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=None)
    pairs = make_pairs([31, 32, 33], 1200.0, BENCH_RATIOS, handle=bs.handle)
    n_win = int(pairs.win_off[-1])
    pcm = vo.synth_pcm(pairs.window_class, 160, seed=21)
    res = bs.sync_host(pcm, pairs.win_off * 160, pairs.cue_start, pairs.cue_end, pairs.cue_off, want_all=True)
    assert (res[1] == pairs.true_offset).all() and (res[2] == pairs.true_k).all()
    for b in range(3):
        ref = vo.energy_zcr_detect(pcm[b * 120000 * 160:(b + 1) * 120000 * 160], 100, 16000, 0.0)
        c0, c1 = int(pairs.cue_off[b]), int(pairs.cue_off[b + 1])
        for k, r in enumerate(BENCH_RATIOS):
            sub = ro.rasterize(pairs.cue_start[c0:c1], pairs.cue_end[c0:c1], None, 100, 0, r)[0]
            ws, wo = ao.fft_align(ref, sub, None)
            assert res[4][b * 5 + k] == wo and _score_ok(res[3][b * 5 + k], ws), (b, k)
    # winner-only run (ratios that provably cannot win keep their fp32 result): same best triples
    win = bs.sync_host(pcm, pairs.win_off * 160, pairs.cue_start, pairs.cue_end, pairs.cue_off)
    assert all(np.array_equal(a, b) for a, b in zip(win[:3], res[:3]))


def test_align_multi_segment_grid(handle, golden, golden_arrays, gf):
    from ffsubsync_b200.aligners import FFTAligner, MaxScoreAligner
    grid = cases.ratio_grid()
    for ci, c in enumerate(golden["multi_segment"]):
        n = int(golden_arrays["ms_sparse_len_%d" % ci])
        sparse = np.unpackbits(golden_arrays["ms_sparse_%d" % ci])[:n].astype(float)
        _, sub = cases.multi_segment_case(c["scale"], c["shift"])
        subs = [cases.scaled_signal(sub, sf) for sf in grid]
        m = MaxScoreAligner(FFTAligner, None, 100, 60).fit(sparse, subs)
        for (got, _), want in zip(m._scores, c["per_ratio"]):
            assert got[1] == want["offset"] and _score_ok(got[0], gf(want["score"]))
        (score, off), pipe = m.transform()
        k = [i for i, s in enumerate(subs) if s is pipe][0]
        assert k == c["best"]["index"] and off == c["best"]["offset"]
        assert grid[k] == pytest.approx(c["scale"], abs=1e-3)
        assert off / 100.0 == pytest.approx(c["shift"], abs=0.05)


def test_maxscore_grid_and_failure(handle, golden, gf):
    from ffsubsync_b200.aligners import FailedToFindAlignmentException, FFTAligner, MaxScoreAligner
    grid = cases.ratio_grid()
    for c in golden["maxscore"]:
        rng = np.random.RandomState(300 + c["seed"])
        true_k = int(rng.randint(0, len(grid)))
        shift = int(rng.randint(-3000, 3001))
        base = (rng.rand(30000) > 0.55).astype(float)
        ref = np.roll(cases.scaled_signal(base, grid[true_k]), shift)
        ref = np.where(rng.rand(len(ref)) < 0.10, 1.0 - ref, ref)
        subs = [cases.scaled_signal(base, r) * min(1.0 / r, 1.0) for r in grid]
        m = MaxScoreAligner(FFTAligner, None, 100, 60).fit(ref, subs)
        for (got, _), want in zip(m._scores, c["per_ratio"]):
            assert got[1] == want["offset"] and _score_ok(got[0], gf(want["score"]))
        (score, off), pipe = m.transform()
        assert [i for i, s in enumerate(subs) if s is pipe][0] == c["best"]["index"]
        assert off == c["best"]["offset"]
    ref, sub = cases.shifted_pair(2000, 300)
    m = MaxScoreAligner(FFTAligner(max_offset_samples=None), None, 100, 0.01).fit(ref, [sub])
    with pytest.raises(FailedToFindAlignmentException, match="max-offset-seconds"):
        m.transform()


def test_reduce_ratios_kernel(handle):
    score = np.array([5.0, 5.0, 4.0, 1.0, 9.0, 2.0, 3.0, 3.0, 3.0])
    offset = np.array([1, 2, 0, 100, 200, 5, -7, 7, 8], dtype=np.int32)
    bs, bo, bk = handle.reduce_ratios(score, offset, None, 3, 3, 10)
    assert bk.tolist() == [0, 2, 0] and bo.tolist() == [1, 5, -7] and bs.tolist() == [5.0, 2.0, 3.0]
    bs, bo, bk = handle.reduce_ratios(score, offset, None, 3, 3, None)
    assert bk.tolist() == [0, 1, 0]
    bs, bo, bk = handle.reduce_ratios(score[:3], np.array([50, 60, 70], np.int32), None, 1, 3, 10)
    assert bk.tolist() == [-1]


def test_gss_fit(handle, golden, gf):
    """--gss: 17 sequential evaluations with the reference's ratios; same winner."""
    from ffsubsync_b200.aligners import FFTAligner, MaxScoreAligner
    want = golden["gss_fit"]
    ref_full, sub = cases.multi_segment_case(25.0 / 24.0, 3.0)
    evals = []

    class Pipe:
        def __init__(self, ratio):
            self.ratio = ratio

        def fit_transform(self, _):
            return cases.scaled_signal(sub, self.ratio)

    def maker(ratio):
        evals.append(float(ratio))
        return Pipe(ratio)

    m = MaxScoreAligner(FFTAligner, None, 100, 60)
    m.fit(ref_full, [maker])
    (score, off), pipe = m.transform()
    assert evals == want["evals"]
    assert off == want["offset"] and pipe.ratio == want["ratio"] and _score_ok(score, gf(want["score"]))


def test_gss_batched_over_pairs(handle):
    """Batched --gss: every pair follows exactly the evaluation sequence the reference's scalar
    search would (oracle: golden_section_trace over rasterise + fft_align), 17 rounds."""
    from oracle import gss_oracle as go
    from ffsubsync_b200.gss_batch import gss_align_batch
    specs = [(41, 200.0, 1.0417, 300), (42, 260.0, 0.96, -450), (43, 180.0, 1.0, 77)]
    refs, cs, ce, cue_off, ref_off = [], [], [], [0], [0]
    for seed, dur, true_ratio, delta in specs:
        st, en = cases.synthetic_cues(seed, dur)
        mask = ro.rasterize(st, en, None, 100, 0, true_ratio)[0] != 0
        n = int(dur * 100 * 1.06) + 700
        ref = np.zeros(n)
        src = np.arange(n) - delta
        ok = (src >= 0) & (src < len(mask))
        ref[ok] = mask[src[ok]]
        ref = np.where(np.random.RandomState(seed).rand(n) < 0.08, 1 - ref, ref)
        refs.append(ref)
        cs.append(st)
        ce.append(en)
        cue_off.append(cue_off[-1] + len(st))
        ref_off.append(ref_off[-1] + n)
    res = gss_align_batch(np.concatenate(refs).astype(np.float32), ref_off, np.concatenate(cs),
                          np.concatenate(ce), cue_off, max_offset_samples=6000, handle=handle)
    assert res.evals.shape == (3, 17)
    for b, (seed, dur, true_ratio, delta) in enumerate(specs):
        rec = {}

        def f(ratio, last, b=b):
            score, off = ao.fft_align(refs[b], ro.rasterize(cs[b], ce[b], None, 100, 0, ratio)[0], 6000)
            if last:
                rec.update(score=score, offset=off, ratio=ratio)
            return -score

        _, calls = go.golden_section_trace(f, 0.9, 1.1)
        assert [c[0] for c in calls] == res.evals[b].tolist()
        assert res.ratio[b] == rec["ratio"] and res.offset[b] == rec["offset"]
        assert _score_ok(res.score[b], rec["score"])


# ========================================================================= whole hot path, batch

def _pair(seed, duration_s, ratio_k, delta, grid, fr=16000):
    """Synthetic (PCM, cues) pair: the reference mask is the subtitle mask at grid[ratio_k] delayed
    by delta frames with 10 % of the frames flipped (SURVEY.md section 8d)."""
    starts, ends = cases.synthetic_cues(seed, duration_s)
    mask, _, _, _ = ro.rasterize(starts, ends, None, 100, 0, grid[ratio_k])
    mask = (mask != 0)
    n = int(duration_s * 100)
    ref = np.zeros(n, dtype=bool)
    src = np.arange(n) - delta
    ok = (src >= 0) & (src < len(mask))
    ref[ok] = mask[src[ok]]
    rng = np.random.RandomState(seed + 1000)
    ref ^= rng.rand(n) < 0.10
    hiss = rng.rand(n) < 0.05
    cls = np.where(ref, 1, np.where(hiss, 2, 0)).astype(np.uint8)
    return cls, starts, ends


def test_sync_batch_small_vs_oracle(handle):
    grid = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
    fpw = 160
    spec = [(31, 240.0, 0, 250), (32, 300.0, 2, -700), (33, 180.0, 4, 0), (34, 200.0, 1, 1234)]
    cls_all, pcm_off, cs, ce, cue_off = [], [0], [], [], [0]
    for seed, dur, k, delta in spec:
        cls, st, en = _pair(seed, dur, k, delta, grid)
        cls_all.append(cls)
        pcm_off.append(pcm_off[-1] + len(cls) * fpw)
        cs.append(st)
        ce.append(en)
        cue_off.append(cue_off[-1] + len(st))
    cls_cat = np.concatenate(cls_all)
    pcm = vo.synth_pcm(cls_cat, fpw, seed=9)
    bs, bo, bk, a_s, a_o = handle.sync_batch(
        pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, np.concatenate(cs), np.concatenate(ce), None,
        cue_off, grid, 0.0, 6000, want_all=True)
    for b, (seed, dur, k, delta) in enumerate(spec):
        ref_sig = vo.energy_zcr_detect(pcm[pcm_off[b]:pcm_off[b + 1]], 100, 16000, 0.0)
        subs = [ro.rasterize(cs[b], ce[b], None, 100, 0, r)[0] for r in grid]
        results = [ao.fft_align(ref_sig, s, 6000) for s in subs]
        for kk, (ws, wo) in enumerate(results):
            assert a_o[b * len(grid) + kk] == wo
            assert _score_ok(a_s[b * len(grid) + kk], ws)
        wk = ao.max_score_select(results, 6000)
        assert (bk[b], bo[b]) == (wk, results[wk][1]) == (k, delta)
        assert _score_ok(bs[b], results[wk][0])
    # winner-only mode (no per-ratio outputs requested): identical best (score, offset, ratio)
    bs2, bo2, bk2, _, _ = handle.sync_batch(
        pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, np.concatenate(cs), np.concatenate(ce), None,
        cue_off, grid, 0.0, 6000, want_all=False)
    assert np.array_equal(bs2, bs) and np.array_equal(bo2, bo) and np.array_equal(bk2, bk)
    # sub-batch pipeline (VAD of sub-batch i+1 overlapping the alignment of sub-batch i on a second
    # stream) forced on this small batch: bit-identical results, per-ratio outputs included
    import os
    for n_sub in ("2", "3", "4"):
        os.environ["B2_SUBBATCHES"] = n_sub
        try:
            r = handle.sync_batch(pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, np.concatenate(cs),
                                  np.concatenate(ce), None, cue_off, grid, 0.0, 6000, want_all=True)
        finally:
            del os.environ["B2_SUBBATCHES"]
        assert np.array_equal(r[0], bs) and np.array_equal(r[1], bo) and np.array_equal(r[2], bk)
        assert np.array_equal(r[3], a_s) and np.array_equal(r[4], a_o)
    # rasterise-to-HBM fallback (float subtitle signals) vs the default in-kernel rasterisation
    for env in ({"B2_FUSED_RASTER": "0"}, {"B2_FUSED_RASTER": "0", "B2_SUBBATCHES": "2"},
                {"B2_ALIGN_SPLIT": "1"}, {"B2_ALIGN_SPLIT": "5"}, {"B2_ALIGN_SPLIT": "2", "B2_FUSED_RASTER": "0"}):
        os.environ.update(env)
        try:
            r = handle.sync_batch(pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, np.concatenate(cs),
                                  np.concatenate(ce), None, cue_off, grid, 0.0, 6000, want_all=True)
        finally:
            for k_ in env:
                del os.environ[k_]
        assert np.array_equal(r[0], bs) and np.array_equal(r[1], bo) and np.array_equal(r[2], bk)
        assert np.array_equal(r[3], a_s) and np.array_equal(r[4], a_o)


@pytest.mark.gpu
def test_sync_batch_fused_raster_edge_cases(handle):
    """In-kernel rasterisation against the oracle where the cue arithmetic is awkward: dropped
    (metadata) cues, cues past the end / before the start (Python slice wrap), overlapping and
    zero-length cues, a pair without cues, and a pair with more cues than the kernel's table
    (falls back to the rasterise-to-HBM path for the whole call)."""
    grid = cases.ratio_grid()
    fpw = 160
    rs = np.random.RandomState(77)

    def build(n_big):
        cls_all, pcm_off, cs, ce, keep, cue_off = [], [0], [], [], [], [0]
        for b, dur in enumerate((90.0, 140.0, 60.0, 75.0)):
            n = int(dur * 100)
            cls = (rs.rand(n) < 0.45).astype(np.uint8)
            cls = np.repeat(cls[::20], 20)[:n]            # 0.2 s runs of speech / silence
            if b == 2:
                st, en, kp = np.zeros(0), np.zeros(0), np.zeros(0, np.uint8)
            else:
                m = n_big if b == 3 else 60
                st = np.sort(rs.uniform(-3.0, dur + 8.0, m))
                en = st + rs.uniform(0.0, 2.5, m)
                en[::7] = st[::7]                            # zero-length
                st[1::11] -= 0.004999                        # microsecond rounding boundary cases
                kp = (rs.rand(m) > 0.15).astype(np.uint8)
            cls_all.append(cls)
            pcm_off.append(pcm_off[-1] + n * fpw)
            cs.append(st); ce.append(en); keep.append(kp)
            cue_off.append(cue_off[-1] + len(st))
        pcm = vo.synth_pcm(np.concatenate(cls_all), fpw, seed=5)
        return pcm, pcm_off, cs, ce, keep, cue_off

    for n_big in (300, 4500):                               # 4500 > 4096: whole call unfused
        pcm, pcm_off, cs, ce, keep, cue_off = build(n_big)
        bs, bo, bk, a_s, a_o = handle.sync_batch(
            pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, np.concatenate(cs), np.concatenate(ce),
            np.concatenate(keep), cue_off, grid, 0.0, 3000, want_all=True)
        for b in range(4):
            ref_sig = vo.energy_zcr_detect(pcm[pcm_off[b]:pcm_off[b + 1]], 100, 16000, 0.0)
            subs = [ro.rasterize(cs[b], ce[b], keep[b].astype(bool), 100, 0, r)[0] for r in grid]
            if len(cs[b]) == 0:
                # all-zero 2-frame signal: thousands of offsets tie exactly and the reference's pick is
                # FFT round-off; the defined answer is the exact argmax (largest offset among equals)
                results = [ao.exact_align(ref_sig, s, 3000) for s in subs]
            else:
                results = [ao.fft_align(ref_sig, s, 3000) for s in subs]
            for kk, (ws, wo) in enumerate(results):
                go = int(a_o[b * len(grid) + kk])
                if go != wo:
                    # random signals, integer-valued scores: only an exact tie (which the reference
                    # breaks by FFT round-off, this path by np.argmax order on exact values) may differ
                    assert ao.exact_score(ref_sig, subs[kk], go) == ao.exact_score(ref_sig, subs[kk], wo)
                    assert go > wo, (n_big, b, kk)
                    results[kk] = (ws, go)
                assert _score_ok(a_s[b * len(grid) + kk], ws)
            wk = ao.max_score_select(results, 3000)
            assert (bk[b], bo[b]) == (wk, results[wk][1])


def test_serialized_speech_replay_batch(handle, tmp_path):
    """make_test_case replay: ref.npz{"speech"} files + cue lists through sync_signals, vs the
    oracle on the same deserialised signals (DeserializeSpeechTransformer semantics included)."""
    from ffsubsync_b200.batch import BatchSynchronizer, load_serialized_speech
    grid = cases.ratio_grid()
    paths, cs, ce, cue_off, truth = [], [], [], [0], []
    for i, (seed, dur, k, delta) in enumerate([(51, 150.0, 3, 120), (52, 210.0, 0, -333), (53, 95.0, 6, 5)]):
        st, en = cases.synthetic_cues(seed, dur)
        mask = ro.rasterize(st, en, None, 100, 0, grid[k])[0]
        n = int(dur * 100)
        ref = np.zeros(n)
        src = np.arange(n) - delta
        ok = (src >= 0) & (src < len(mask))
        ref[ok] = (mask != 0)[src[ok]]
        ref = np.where(np.random.RandomState(seed).rand(n) < 0.05, 0.3, ref)   # "unsure" frames < 1
        p = str(tmp_path / ("ref%d.npz" % i))
        np.savez_compressed(p, speech=ref)
        paths.append(p)
        cs.append(st)
        ce.append(en)
        cue_off.append(cue_off[-1] + len(st))
        truth.append((k, delta))
    sig, off = load_serialized_speech(paths, non_speech_label=0.0)
    bs = BatchSynchronizer(grid, max_offset_seconds=60)
    score, offset, best_k = bs.sync_signals(sig, off, np.concatenate(cs), np.concatenate(ce), cue_off)
    for b in range(3):
        ref = sig[off[b]:off[b + 1]].astype(np.float64)
        assert set(np.unique(ref)) <= {0.0, 1.0}          # values < 1 were relabelled
        subs = [ro.rasterize(cs[b], ce[b], None, 100, 0, r)[0] for r in grid]
        (ws, wo), wk = ao.max_score_align(ref, subs, 100, 60)
        assert (best_k[b], offset[b]) == (wk, wo) == truth[b]
        assert _score_ok(score[b], ws)


def test_sync_two_hour_pair_recovers_offset(handle):
    """BASELINE config 2: synthetic 2 h PCM at 16 kHz + shifted cues, VAD + alignment end to end.
    Full-size check through domain properties: the known offset/ratio are recovered, the score is
    the exact count of agreeing minus disagreeing frames (binary signals)."""
    grid = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
    cls, st, en = _pair(77, 7200.0, 0, -2718, grid)
    pcm = handle.synth_pcm(cls, len(cls), 160, seed=123)
    assert len(pcm) == 115200000
    bs, bo, bk, a_s, a_o = handle.sync_batch(pcm, [0, len(pcm)], 16000, 100, 0.0, 100000, -1, -1, st, en,
                                             None, [0, len(st)], grid, 0.0, 6000, want_all=True)
    assert (bk[0], bo[0]) == (0, -2718)
    # reference-side signal from the numpy restatement of the detector, in 100 s chunks like the
    # reference's loop (a few loud-hiss windows legitimately fall inside the zero-crossing band)
    chunk = 1600000
    ref_sig = np.concatenate([vo.energy_zcr_detect(pcm[i:i + chunk], 100, 16000, 0.0)
                              for i in range(0, len(pcm), chunk)])
    assert len(ref_sig) == 720000 and abs(int(ref_sig.sum()) - int((cls == 1).sum())) < 200
    sub = ro.rasterize(st, en, None, 100, 0, 1.0)[0]
    assert bs[0] == ao.exact_score(ref_sig, sub, -2718)   # binary signals: exact integer
    assert np.all(a_s[1:] < bs[0])
    subs = [ro.rasterize(st, en, None, 100, 0, r)[0] for r in grid]
    for k in range(1, len(grid)):      # every ratio candidate: offset exact, score exact for +-1 x {-1, a}
        ws, wo = ao.fft_align(ref_sig, subs[k], 6000)
        assert a_o[k] == wo and _score_ok(a_s[k], ws)
    # a single pair is split over CTAs by block ranges (8 chunks here by default); any other
    # split, and none, must give bit-identical results (exact re-score, deterministic merge)
    import os
    for split in ("1", "3", "35", "40"):
        os.environ["B2_ALIGN_SPLIT"] = split
        try:
            r = handle.sync_batch(pcm, [0, len(pcm)], 16000, 100, 0.0, 100000, -1, -1, st, en, None,
                                  [0, len(st)], grid, 0.0, 6000, want_all=True)
        finally:
            del os.environ["B2_ALIGN_SPLIT"]
        assert np.array_equal(r[0], bs) and np.array_equal(r[1], bo) and np.array_equal(r[2], bk)
        assert np.array_equal(r[3], a_s) and np.array_equal(r[4], a_o), split


# ============================================================== auditok detector (V3) on the GPU

def _auditok_pcm(rng, frame_rate, n_blocks, cut=0):
    """PCM whose per-block energies straddle the 50 dB edge, in runs that exercise the tokenizer:
    blips shorter than min_length, silences around max_continuous_silence = 25, runs beyond
    max_length = 500."""
    fpw = frame_rate // 100
    runs = []
    while sum(runs) < n_blocks:
        runs.append(int(rng.choice([1, 3, 8, 19, 20, 21, 24, 25, 26, 27, 60, 150, 499, 500, 501, 700])))
    amp = np.concatenate([np.full(r, 1.12 if (i % 2 == 0) else 0.88) for i, r in enumerate(runs)])[:n_blocks]
    amp = amp * rng.uniform(0.9, 1.1, len(amp))     # decisions flip near the edge inside the runs too
    pcm = np.round(rng.randn(n_blocks * fpw) * 316.2 * np.repeat(amp, fpw)).astype(np.int16)
    return pcm[: len(pcm) - cut] if cut else pcm


@pytest.mark.parametrize("frame_rate", [16000, 48000, 44100, 8000])
@pytest.mark.parametrize("label", [0.0, 0.3])
def test_auditok_detector_matches_oracle(handle, frame_rate, label):
    from ffsubsync_b200.speech_transformers import _make_auditok_detector
    from oracle import auditok_oracle as au
    rng = np.random.RandomState(frame_rate % 89 + int(label * 10))
    det = _make_auditok_detector(100, frame_rate, label)
    fpw = frame_rate // 100
    for n_blocks, cut in ((6000, 0), (2500, 13), (700, fpw - 1), (30, 1), (1, 0)):
        pcm = _auditok_pcm(rng, frame_rate, n_blocks, cut)
        want = au.auditok_detect_fast(pcm.tobytes(), 100, frame_rate, label)
        got = det(np.frombuffer(pcm.tobytes(), np.uint8))
        assert got.dtype == np.float64 and len(got) == len(want)
        assert np.array_equal(got, want), (frame_rate, label, n_blocks, cut, int(np.argmax(got != want)))
    assert len(det(b"")) == 0
    with pytest.raises(ValueError):
        det(b"\x01\x02\x03")
    # the literal (per-block numpy validator) restatement on a shorter input
    pcm = _auditok_pcm(rng, frame_rate, 1200, 5)
    assert np.array_equal(det(pcm.tobytes()), au.auditok_detect(pcm.tobytes(), 100, frame_rate, label))


def test_auditok_one_long_call(handle):
    """A whole 30-minute signal in ONE detector call (180 000 blocks through one warp's scan), and the
    same signal through the batch ABI in 100 s calls."""
    from ffsubsync_b200.speech_transformers import _make_auditok_detector
    from oracle import auditok_oracle as au
    rng = np.random.RandomState(180)
    pcm = _auditok_pcm(rng, 16000, 180000, cut=3)
    got = _make_auditok_detector(100, 16000, 0.0)(pcm.tobytes())
    assert np.array_equal(got, au.auditok_detect_fast(pcm.tobytes(), 100, 16000, 0.0))
    out, _ = handle.vad_auditok(pcm, [0, len(pcm)], 16000, 100, 0.0, chunk_samples=160 * 10000)
    want = np.concatenate([au.auditok_detect_fast(pcm[i:i + 1600000].tobytes(), 100, 16000, 0.0)
                           for i in range(0, len(pcm), 1600000)])
    assert np.array_equal(out, want)


def test_energy_rule_equals_the_auditok_validator(handle):
    """The per-window energy decision of this package's detectors (E >= fpw * 10^5) is auditok's
    AudioEnergyValidator(energy_threshold=50) on the same block - the pin for the VAD arithmetic."""
    from ffsubsync_b200.speech_transformers import _make_energy_detector
    from oracle import auditok_oracle as au
    rng = np.random.RandomState(17)
    for frame_rate in (16000, 48000):
        fpw = frame_rate // 100
        pcm = _auditok_pcm(rng, frame_rate, 3000)
        # exact-edge blocks: E == fpw * 10^5 (valid) and one LSB below (invalid)
        edge = np.zeros(fpw, np.int16)
        edge[: fpw * 10 // 16] = 400                    # (10/16) fpw * 160000 = fpw * 10^5
        pcm[:fpw] = edge
        edge[0] = 399
        pcm[fpw:2 * fpw] = edge
        got = _make_energy_detector(100, frame_rate, 0.0)(pcm.tobytes())
        want = np.array([1.0 if au.block_is_valid(b, 50) else 0.0 for b in au.read_blocks(pcm, fpw)])
        assert np.array_equal(got, want) and got[0] == 1.0 and got[1] == 0.0
        assert 0.2 < want.mean() < 0.8


def test_auditok_chunk_loop_250s(handle):
    """VideoSpeechTransformer(vad='auditok') over 250 s: three detector calls (100 + 100 + 50 s), the
    tokenizer restarting in each (speech_transformers.py:142,746)."""
    from ffsubsync_b200.speech_transformers import VideoSpeechTransformer
    from oracle import auditok_oracle as au
    rng = np.random.RandomState(250)
    pcm = _auditok_pcm(rng, 16000, 25000, cut=77)
    for label in (0.0, 0.5):
        vst = VideoSpeechTransformer("auditok", 100, 16000, label).fit(pcm.tobytes())
        chunk = 160 * 10000
        want = np.concatenate([au.auditok_detect_fast(pcm[i:i + chunk].tobytes(), 100, 16000, label)
                               for i in range(0, len(pcm), chunk)])
        assert np.array_equal(vst.transform(), want)
        # restarting matters: one call over the whole buffer gives a different signal
        assert not np.array_equal(want, au.auditok_detect_fast(pcm.tobytes(), 100, 16000, label))


def test_auditok_batch_abi_chunked(handle):
    from oracle import auditok_oracle as au
    rng = np.random.RandomState(99)
    sigs = [_auditok_pcm(rng, 16000, n, cut) for n, cut in ((23000, 0), (10000, 159), (1, 0), (12000, 8))]
    sigs.insert(2, np.zeros(0, np.int16))
    off = np.concatenate([[0], np.cumsum([len(s) for s in sigs])])
    chunk = 160 * 10000
    out, out_off = handle.vad_auditok(np.concatenate(sigs), off, 16000, 100, 0.0, chunk_samples=chunk)
    for b, s in enumerate(sigs):
        want = [au.auditok_detect_fast(s[i:i + chunk].tobytes(), 100, 16000, 0.0) for i in range(0, len(s), chunk)]
        want = np.concatenate(want) if want else np.zeros(0)
        assert np.array_equal(out[out_off[b]:out_off[b + 1]], want), b
    # other tokenizer parameters / threshold through the ABI
    out, _ = handle.vad_auditok(sigs[0], [0, len(sigs[0])], 16000, 100, 0.0, energy_threshold_db=49.0,
                                min_length=3, max_length=40, max_continuous_silence=0)
    fl = (sigs[0].astype(np.int64).reshape(-1, 160) ** 2).sum(axis=1) >= au.energy_floor(160, 49.0)
    m = np.zeros(len(fl) + 1)
    for s, e in au.tokenize(list(fl), 3, 40, 0):
        m[s] = 1.0
        m[e + 1] = -1.0
    assert np.array_equal(out, np.clip(np.cumsum(m)[:-1], 0, 1))


# ============================================================ ABI corner cases (round-1 advice)

def test_mask_width_corner_cases(handle):
    """Any integer mask width goes through the reference's slice arithmetic: negative widths mask
    everything (score -inf, offset N-1-S), huge widths mask nothing."""
    from ffsubsync_b200.aligners import FFTAligner
    rng = np.random.RandomState(4)
    ref = (rng.rand(500) > 0.5).astype(float)
    sub = np.concatenate([np.zeros(17), ref])[:480]
    for mos in (-1, -7, -10 ** 6, 0, 1, 2 ** 31, 2 ** 40, 2 ** 70):
        got = FFTAligner(max_offset_samples=mos).fit_transform(ref, sub, get_score=True)
        want = ao.fft_align(ref, sub, mos)
        assert got[1] == want[1] and _score_ok(got[0], want[0]), (mos, got, want)
    assert FFTAligner(max_offset_samples=-1).fit_transform(ref, sub, get_score=True)[0] == -np.inf


def test_device_calls_reject_host_pointers(handle):
    from ffsubsync_b200 import _native
    pcm = np.zeros(1600, np.int16)
    out = np.zeros(10, np.float32)
    with pytest.raises(_native.NativeError):
        handle.vad_energy_zcr(pcm.ctypes.data, [0, 1600], 16000, 100, 0.0, 100000, out=out.ctypes.data,
                              memspace=_native.B2_DEVICE)


# ======================================================= BASELINE configs[2] at its stated size

def test_sync_batch_config3_256_pairs_vs_oracle(handle):
    """B = 256 two-hour pairs, K = 5 (the benchmarked configuration: n_split = 1, 1280 correlation
    jobs, winner-only pruning): every ratio of a seeded sample of 8 pairs against the oracle (offset
    exact, score <= 1e-5), winner triples of the all-ratio and the winner-only runs identical, and
    the planted (offset, ratio) recovered on all 256 pairs."""
    import torch
    import bench
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    B, ratios = 256, BENCH_RATIOS
    bs = BatchSynchronizer(ratios, 16000, 100, 0.0, max_offset_seconds=60)
    pairs = make_pairs([13 + b for b in range(B)], 7200.0, ratios, handle=bs.handle)
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(pairs.window_class).cuda()
    pcm_d = torch.empty(n_win * 160, dtype=torch.int16, device="cuda")
    bs.handle.synth_pcm(cls_d.data_ptr(), n_win, 160, 1234, out=pcm_d.data_ptr(), memspace=_native.B2_DEVICE)
    bs.handle.synchronize()
    del cls_d
    pcm_off = pairs.win_off * 160
    rep = bench.verify_against_oracle(bs, pairs, pcm_d, pcm_off, ratios, 8, 2024 + B)
    assert rep["ok"], rep
    assert rep["winner_only_equals_all_ratios"] and len(rep["pairs_checked"]) == 8
    out = bs.sync_device(pcm_d, pcm_off, pairs.cue_start, pairs.cue_end, pairs.cue_off)
    torch.cuda.synchronize()
    assert (out["best_offset"].cpu().numpy() == pairs.true_offset).all()
    assert (out["best_k"].cpu().numpy() == pairs.true_k).all()
    del pcm_d
    torch.cuda.empty_cache()


def test_sync_batch_resident_chained_calls_equal_ordered_calls(handle):
    """B2_DEVICE_RESIDENT: back-to-back b2_sync_batch calls over resident corpora overlap (the VAD of call
    m starts behind call m-1's fence and writes the other reference-signal buffer).  Two corpora of
    different sizes, alternated without any synchronisation, must give exactly what ordered B2_DEVICE
    calls give; an entry point in between (b2_synchronize) breaks the chain and the next call falls
    back to stream order."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    bs = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=60)
    corpora = []
    for seed0, B in ((100, 120), (900, 100)):
        pairs = make_pairs([seed0 + b for b in range(B)], 600.0, BENCH_RATIOS, handle=bs.handle)
        n_win = int(pairs.win_off[-1])
        cls_d = torch.from_numpy(pairs.window_class).cuda()
        pcm = torch.empty(n_win * 160, dtype=torch.int16, device="cuda")
        bs.handle.synth_pcm(cls_d.data_ptr(), n_win, 160, seed0, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
        bs.handle.synchronize()
        args = (pcm, pairs.win_off * 160, pairs.cue_start, pairs.cue_end, pairs.cue_off)
        want = bs.sync_device(*args)
        bs.handle.synchronize()
        torch.cuda.synchronize()
        want = {k: v.clone() for k, v in want.items()}
        assert (want["best_offset"].cpu().numpy() == pairs.true_offset).all()
        assert (want["best_k"].cpu().numpy() == pairs.true_k).all()
        corpora.append((args, want))
    order = [0, 1, 0, 0, 1, 1, 0, 1]
    outs = [bs.sync_device(*corpora[c][0], inputs_resident=True) for c in order]   # nothing synchronised in between
    bs.handle.synchronize()                                                         # breaks the chain
    outs.append(bs.sync_device(*corpora[0][0], inputs_resident=True))               # unchained resident call
    outs.append(bs.sync_device(*corpora[1][0], inputs_resident=True))               # chained again
    outs.append(bs.sync_device(*corpora[0][0]))                                     # ordered call after a chained one
    bs.handle.synchronize()
    torch.cuda.synchronize()
    for c, got in zip(order + [0, 1, 0], outs):
        want = corpora[c][1]
        for k in ("best_score", "best_offset", "best_k"):
            assert torch.equal(got[k], want[k]), (c, k)


def test_resident_memspace_is_sync_batch_only(handle):
    """B2_DEVICE_RESIDENT is a promise about b2_sync_batch's inputs; every other entry point rejects it."""
    import torch
    from ffsubsync_b200 import _native
    pcm = torch.zeros(16000, dtype=torch.int16, device="cuda")
    out = torch.zeros(100, dtype=torch.float32, device="cuda")
    with pytest.raises(_native.NativeError) as ei:
        handle.vad_energy_zcr(pcm.data_ptr(), [0, 16000], 16000, 100, 0.0, 100000, out=out.data_ptr(),
                              memspace=_native.B2_DEVICE_RESIDENT)
    assert "memspace" in str(ei.value)


def test_candidate_sharded_mode_single_rank_equals_sync_batch(handle):
    """The B < G mode's compute path (VAD -> own candidates -> reduce) with world = 1 equals
    b2_sync_batch; the multi-rank exchange is covered by the gloo test and tools/candidate_mode_bench.py."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.constants import FRAMERATE_RATIOS
    from ffsubsync_b200.synth import make_pairs
    r = np.array(FRAMERATE_RATIOS)
    ratios = [1.0] + list(np.concatenate([r, 1.0 / r]))
    bs = BatchSynchronizer(ratios, 16000, 100, 0.0, max_offset_seconds=60)
    pairs = make_pairs([5, 6, 7], 600.0, ratios, handle=bs.handle)
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(pairs.window_class).cuda()
    pcm = torch.empty(n_win * 160, dtype=torch.int16, device="cuda")
    bs.handle.synth_pcm(cls_d.data_ptr(), n_win, 160, 9, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    bs.handle.synchronize()
    args = (pcm, pairs.win_off * 160, pairs.cue_start, pairs.cue_end, pairs.cue_off)
    a = bs.sync_device_candidate_sharded(*args)
    b = bs.sync_device(*args)
    bs.handle.synchronize()
    torch.cuda.synchronize()
    assert torch.equal(a[1], b["best_offset"]) and torch.equal(a[2], b["best_k"]) and torch.equal(a[0], b["best_score"])
    assert (a[1].cpu().numpy() == pairs.true_offset).all() and (a[2].cpu().numpy() == pairs.true_k).all()


# ===================================================== decode / probe subprocess branches (fake binaries)

_FAKE_FFMPEG = r'''#!/usr/bin/env python3
# stand-in for ffmpeg in tests: "decodes" $FAKE_PCM (s16le mono at the rate given by -ar), honouring -ss / -t
import os, sys
a = sys.argv[1:]
def hms(v):
    h, m, s = v.split(":")
    return int(h) * 3600 + int(m) * 60 + float(s)
rate = int(a[a.index("-ar") + 1])
ss = hms(a[a.index("-ss") + 1]) if "-ss" in a else 0.0
t = hms(a[a.index("-t") + 1]) if "-t" in a else None
assert a[-1] == "-" and "-i" in a and "s16le" in a
data = open(os.environ["FAKE_PCM"], "rb").read()
lo = 2 * int(round(ss * rate))
hi = len(data) if t is None else lo + 2 * int(round(t * rate))
sys.stdout.buffer.write(data[lo:hi])
'''
_FAKE_FFPROBE = '#!/bin/sh\necho "$FAKE_DURATION"\n'


def test_ffmpeg_and_ffprobe_subprocess_branches(handle, tmp_path, monkeypatch):
    """A media path goes through an ffmpeg subprocess (speech_transformers.py:682-704) and, for the
    multi-segment transformer, an ffprobe duration query (:851-853).  Neither binary exists in this
    image: small stand-ins on ``ffmpeg_path`` exercise the argument list (-ss / -t / -ar / -f s16le),
    the pipe reader and the per-segment thread pool; results equal the raw-PCM path."""
    import os
    import stat
    from ffsubsync_b200.speech_transformers import MultiSegmentVideoSpeechTransformer, VideoSpeechTransformer
    for name, body in (("ffmpeg", _FAKE_FFMPEG), ("ffprobe", _FAKE_FFPROBE)):
        path = tmp_path / name
        path.write_text(body)
        path.chmod(path.stat().st_mode | stat.S_IEXEC)
    rng = np.random.RandomState(8)
    pcm = vo.synth_pcm(rng.randint(0, 2, 30000).astype(np.uint8), 160, seed=2)   # 300 s
    pcm_file = tmp_path / "audio.pcm"
    pcm_file.write_bytes(pcm.tobytes())
    monkeypatch.setenv("FAKE_PCM", str(pcm_file))
    monkeypatch.setenv("FAKE_DURATION", "300.0")
    direct = VideoSpeechTransformer("energy_zcr", 100, 16000, 0.0).fit(pcm.tobytes()).transform()
    via = VideoSpeechTransformer("energy_zcr", 100, 16000, 0.0, ffmpeg_path=str(tmp_path)).fit("movie.mkv").transform()
    assert np.array_equal(via, direct)
    part = VideoSpeechTransformer("energy_zcr", 100, 16000, 0.0, start_seconds=120, max_duration_seconds=60,
                                  ffmpeg_path=str(tmp_path), ref_stream="0:a:1").fit("movie.mkv").transform()
    assert np.array_equal(part, direct[12000:18000])
    ms = MultiSegmentVideoSpeechTransformer("energy_zcr", 100, 16000, 0.0, segment_count=3, segment_duration=60,
                                            ffmpeg_path=str(tmp_path))
    sparse = ms.fit("movie.mkv").transform()
    raw = MultiSegmentVideoSpeechTransformer("energy_zcr", 100, 16000, 0.0, segment_count=3,
                                             segment_duration=60).fit(str(pcm_file)).transform()
    assert np.array_equal(sparse, raw) and sparse.sum() > 0
    with pytest.raises(ValueError, match="no ffmpeg binary"):
        VideoSpeechTransformer("energy_zcr", 100, 16000, 0.0, ffmpeg_path=str(tmp_path / "nowhere")).fit("movie.mkv")


# ================================================= adversarial signal families (round-off bound, ties)

_adv_family = cases.signal_family


@pytest.mark.parametrize("mos", [6000, None])
def test_adversarial_families_offsets_are_exact_maxima(handle, mos):
    """Constant, periodic, sparse and wide-dynamic-range signals (large means, flat or periodic
    correlation landscapes, many exact ties) through both correlation paths: the returned offset must
    attain the maximum of the EXACT scores over the surviving window (the reference breaks exact ties
    by its float64 round-off, so only the score and tie-membership are comparable), unless the kernel
    flagged more tied candidates than its re-score budget."""
    from ffsubsync_b200 import _native
    fams = ["random", "ones", "period2", "period_block", "sparse", "wide"]
    rng = np.random.RandomState(77)
    refs, subs, meta = [], [], []
    for fr in fams:
        for fs in fams:
            refs.append(_adv_family(fr, 70000, rng))
            subs.append(_adv_family(fs, 66000, rng, 0.96))
            meta.append((fr, fs))
    B = len(refs)
    ref_off = np.arange(B + 1, dtype=np.int64) * 70000
    sub_off = np.arange(B + 1, dtype=np.int64) * 66000
    score, off, st = handle.align_batch(np.concatenate(refs), ref_off, np.concatenate(subs), sub_off, B, 1, mos)
    n_flagged, problems = 0, []
    for b in range(B):
        ws, wo = ao.fft_align(refs[b], subs[b], mos)
        mine = ao.exact_score(refs[b], subs[b], int(off[b]))
        tol = 1e-9 * max(abs(ws), 1.0) + 1e-6 * float(np.abs(2 * subs[b] - 1).max() * np.abs(2 * refs[b] - 1).max())
        if abs(score[b] - mine) > 1e-9 * max(abs(mine), 1.0) + 1e-9:
            problems.append(("score is not the exact score of the returned offset", meta[b], float(score[b]), mine))
        if st[b] & _native.ALIGN_CAND_OVERFLOW:
            n_flagged += 1      # a plateau of exact ties wider than the re-score budget: flagged, not checked
            continue
        if not (mine >= ws - tol and _score_ok(score[b], ws)):
            problems.append(("not a maximum", meta[b], mos, int(off[b]), int(wo), mine, ws))
    assert not problems, problems[:6]
    # plateaus of exact ties wider than the re-score budget: a constant reference against ANY subtitle
    # signal that it fully overlaps (the score does not depend on the offset), period-2 signals against
    # each other and, unmasked, every all-negative correlation, whose maximum is the block of structural
    # zeros.  Measured: 16 of 36 (masked), <= 24 (unmasked).
    assert n_flagged <= 24, n_flagged


def test_unmasked_largest_transform_size(handle):
    """N = 2^23 (M1 = 4096, the largest four-step factorisation): R + S = 5.5 M frames (15 h of signal)."""
    from ffsubsync_b200.aligners import FFTAligner
    rng = np.random.RandomState(23)
    ref = (rng.rand(3000000) > 0.5).astype(np.float32)
    sub = np.concatenate([np.zeros(4321, np.float32), ref])[:2500001]
    score, off = FFTAligner().fit_transform(ref, sub, get_score=True)
    ws, wo = ao.fft_align(ref, sub, None)
    assert off == wo == -4321 and _score_ok(score, ws)
