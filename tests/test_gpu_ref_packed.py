"""GPU tests of the packed reference (csrc/sync_plan.h plan_ref_format): on sub-batches whose chain takes the run
path the lane-per-window VAD writes the reference as bits m = (r == 1.0f) instead of floats, a scan builds the run
path's reference table from them and the exact re-score rebuilds r = m ? 1.0f : label.  Every output must equal
the float reference's (B2_REF_PACKED=0) bit for bit: best_* and the per-ratio all_* scores, offsets and statuses,
at 16 and 8 kHz, at labels 0, 0.3, 1.0 and -0.5, for reference lengths off the 32-window grid, shorter than 32
windows and with a trailing partial window, with empty videos, several tracks per video, sub-batches, resident
chained calls, the GSS rounds and B2_ALIGN_PATH=runs under a capture."""
import contextlib
import os

import numpy as np
import pytest

import cases
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
LABELS = [0.0, 0.3, 1.0, -0.5]


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@contextlib.contextmanager
def _env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _corpus(videos, fpw, seed0=0):
    """videos: list of (windows, extra samples, [(k, delta) per track]); the extra samples (a multiple of 8, so the
    next video stays 16-byte aligned) make a trailing partial window.  Track = the video's master cues at GRID[k]
    moved by delta frames, 10 % of the cues dropped, +-10 ms jitter."""
    pcms, tv, cs, ce = [], [], [], []
    for v, (n, extra, tracks) in enumerate(videos):
        seed = seed0 + 31 * v + 7
        starts, ends = cases.synthetic_cues(seed, max(n / 100.0, 60.0))   # short videos' tracks have cues too
        mask = ro.rasterize(starts, ends, None, 100, 0, 1.0)[0] != 0
        ref = np.zeros(n, dtype=bool)
        ref[: min(n, len(mask))] = mask[:n]
        rng = np.random.RandomState(seed + 1000)
        ref ^= rng.rand(n) < 0.10
        cls = np.where(ref, 1, np.where(rng.rand(n) < 0.05, 2, 0)).astype(np.uint8)
        pcm = vo.synth_pcm(cls, fpw, seed=seed) if n else np.zeros(0, np.int16)
        if extra:
            pcm = np.concatenate([pcm, (rng.randint(-9000, 9000, extra)).astype(np.int16)])
        pcms.append(pcm)
        for i, (k, delta) in enumerate(tracks):
            r = np.random.RandomState(seed * 100 + i)
            keep = r.rand(len(starts)) >= 0.1
            jit = r.randint(-1, 2, len(starts)) * 0.01
            st = (starts - delta / 100.0 + jit) / GRID[k]
            en = (ends - delta / 100.0 + jit) / GRID[k]
            keep &= st >= 0
            tv.append(v)
            cs.append(np.round(st[keep], 3))
            ce.append(np.round(en[keep], 3))
    return dict(pcm=np.concatenate(pcms), pcm_off=np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64),
                track_video=np.array(tv, np.int32), cue_start=np.concatenate(cs), cue_end=np.concatenate(ce),
                cue_off=np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64), fpw=fpw)


# windows per video: off the 32-window grid, under 32, a multiple of 32, an empty video with a track and one
# without, and a trailing partial window (40 samples) on several
VIDEOS = [(24000, 0, [(0, 250)]), (30017, 40, [(2, -700), (4, 0), (1, 1234)]), (0, 0, []),
          (20000, 0, [(3, 40), (0, -1500), (2, 9), (4, 600), (1, -321)]), (25, 40, [(0, 3)]), (0, 0, [(1, 0)]),
          (18031, 8, [(1, 5999), (3, -6000)])]


@pytest.fixture(scope="module", params=[160, 80], ids=["16k", "8k"])
def corpus(request):
    return _corpus(VIDEOS, request.param, seed0=11)


def _tracks(handle, c, label, mos=6000, want_all=True):
    fr = 100 * c["fpw"]
    return handle.sync_tracks(c["pcm"], c["pcm_off"], c["track_video"], fr, 100, label, 100000, -1, -1,
                              c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, mos, want_all=want_all)


def _same(a, b):
    for x, y in zip(a, b):
        if x is None and y is None:
            continue
        np.testing.assert_array_equal(np.asarray(x), np.asarray(y))   # NaN == NaN: gss_ratio of an empty reference


def _packed_vs_float(run):
    with _env(B2_REF_PACKED=0):
        want = run()
    got = run()
    _same(got, want)
    return got


@pytest.mark.parametrize("label", LABELS)
@pytest.mark.parametrize("want_all", [True, False])
def test_packed_equals_float(handle, corpus, label, want_all):
    _packed_vs_float(lambda: _tracks(handle, corpus, label, want_all=want_all))


@pytest.mark.parametrize("label", [0.0, 1.0])
def test_packed_sub_batches(handle, corpus, label):
    """Cut into sub-batches (the VADs of the later ones on a partition of the SMs)."""
    with _env(B2_SUBBATCHES=3, B2_VAD_SMS=60):
        _packed_vs_float(lambda: _tracks(handle, corpus, label))


def test_packed_gss(handle, corpus):
    """The GSS rounds read the packed reference through the same scan and re-score."""
    fr = 100 * corpus["fpw"]
    _packed_vs_float(lambda: handle.sync_tracks_gss(
        corpus["pcm"], corpus["pcm_off"], corpus["track_video"], fr, 100, 0.3, 100000, -1, -1, corpus["cue_start"],
        corpus["cue_end"], None, corpus["cue_off"], GRID, 0.0, 6000, want_all=True, want_evals=True))


def test_forced_tiled_keeps_floats(handle, corpus):
    """A packed-eligible call forced onto the tiled path gets the float reference, and the float result."""
    with _env(B2_ALIGN_PATH="tiled"):
        tiled = _packed_vs_float(lambda: _tracks(handle, corpus, 0.3))
    _same(_tracks(handle, corpus, 0.3), tiled)   # and the run path agrees with it


def test_forced_runs_under_capture(handle, corpus):
    """B2_ALIGN_PATH=runs with a capture: the run path's float64 scores are captured, from either reference."""
    T = len(corpus["track_video"])
    J = T * len(GRID)
    caps = []
    for packed in ("0", "1"):
        with _env(B2_ALIGN_PATH="runs", B2_REF_PACKED=packed):
            with handle.capture_nominations(J, 12001) as cap:
                out = _tracks(handle, corpus, 0.0)
        caps.append((out, cap))
    _same(caps[0][0], caps[1][0])
    for k in ("win", "stat", "cand"):
        assert np.array_equal(caps[0][1][k], caps[1][1][k]), k
    for j in range(J):
        n = int(caps[0][1]["win"][j, 1])
        assert np.array_equal(caps[0][1]["scores"][j, :n], caps[1][1]["scores"][j, :n]), j


def _device_corpora(bs, specs):
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    corpora = []
    for seed0, B in specs:
        pairs = make_pairs([seed0 + b for b in range(B)], 600.0, BENCH_RATIOS, handle=bs.handle)
        n_win = int(pairs.win_off[-1])
        cls_d = torch.from_numpy(pairs.window_class).cuda()
        pcm = torch.empty(n_win * 160, dtype=torch.int16, device="cuda")
        bs.handle.synth_pcm(cls_d.data_ptr(), n_win, 160, seed0, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
        bs.handle.synchronize()
        corpora.append((pcm, pairs.win_off * 160, pairs.cue_start, pairs.cue_end, pairs.cue_off))
    return corpora


def test_packed_resident_chained_calls(handle):
    """11 resident b2_sync_batch calls alternating two corpora of >= 96 pairs (sub-batched by default), chained
    without synchronisation, as the packed reference double-buffers in the same slots as the floats."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS
    bs = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=60)
    corpora = _device_corpora(bs, ((300, 120), (700, 100)))
    want = []
    with _env(B2_REF_PACKED=0):
        for args in corpora:
            w = bs.sync_device(*args)
            bs.handle.synchronize()
            torch.cuda.synchronize()
            want.append({k: v.clone() for k, v in w.items()})
    order = [0, 1, 0, 0, 1, 1, 0, 1]
    outs = [bs.sync_device(*corpora[c], inputs_resident=True) for c in order]
    bs.handle.synchronize()
    outs.append(bs.sync_device(*corpora[0], inputs_resident=True))
    outs.append(bs.sync_device(*corpora[1], inputs_resident=True))
    outs.append(bs.sync_device(*corpora[0]))
    bs.handle.synchronize()
    torch.cuda.synchronize()
    for c, got in zip(order + [0, 1, 0], outs):
        for k in ("best_score", "best_offset", "best_k"):
            assert torch.equal(got[k], want[c][k]), (c, k)
