"""GPU tests of the run path of the aligner (csrc/runcorr.cu): cue-mode calls score every offset of the
window from the cue runs and the two-level VAD reference, then nominate within a float64 margin.

The run path must give exactly what the overlap-save FFT path (B2_ALIGN_PATH=tiled) gives - winners and
per-ratio outputs - and match the oracle; the selection must keep the FFT paths under a capture and for
large windows.  Which path ran is read from the handle's launch counter (the paths launch different
kernel sequences)."""
import contextlib
import os

import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
FPW = 160


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


def _corpus(videos, seed0=0, label_noise=0.10):
    """videos: list of (duration_s, [(k, delta) per track]); track = the video's master cues at GRID[k],
    moved by delta frames, 10 % of the cues dropped, +-10 ms jitter."""
    pcms, tv, cs, ce = [], [], [], []
    for v, (dur, tracks) in enumerate(videos):
        seed = seed0 + 31 * v + 7
        starts, ends = cases.synthetic_cues(seed, dur)
        mask = ro.rasterize(starts, ends, None, 100, 0, 1.0)[0] != 0
        n = int(dur * 100)
        ref = np.zeros(n, dtype=bool)
        ref[: min(n, len(mask))] = mask[:n]
        rng = np.random.RandomState(seed + 1000)
        ref ^= rng.rand(n) < label_noise
        cls = np.where(ref, 1, np.where(rng.rand(n) < 0.05, 2, 0)).astype(np.uint8)
        pcms.append(vo.synth_pcm(cls, FPW, seed=seed))
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
    return dict(pcm=np.concatenate(pcms), pcms=pcms,
                pcm_off=np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64),
                track_video=np.array(tv, np.int32), cs=cs, ce=ce,
                cue_start=np.concatenate(cs), cue_end=np.concatenate(ce),
                cue_off=np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64))


def _pairs(c):
    """The corpus as b2_sync_batch pairs: each track with its own copy of its video's PCM."""
    pcm = np.concatenate([c["pcms"][v] for v in c["track_video"]])
    off = np.concatenate([[0], np.cumsum([len(c["pcms"][v]) for v in c["track_video"]])]).astype(np.int64)
    return pcm, off


def _batch(handle, c, mos, label=0.0, want_all=True):
    pcm, off = _pairs(c)
    n0 = handle.launch_count
    out = handle.sync_batch(pcm, off, 16000, 100, label, 100000, -1, -1, c["cue_start"], c["cue_end"], None,
                            c["cue_off"], GRID, 0.0, mos, want_all=want_all)
    return out, handle.launch_count - n0


def _tracks(handle, c, mos, label=0.0, want_all=True):
    n0 = handle.launch_count
    out = handle.sync_tracks(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, label, 100000, -1, -1,
                             c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, mos, want_all=want_all)
    return out, handle.launch_count - n0


def _same(a, b):
    for x, y in zip(a, b):
        if x is None and y is None:
            continue
        assert np.array_equal(np.asarray(x), np.asarray(y)), (x, y)


def _oracle_check(c, out, mos, label=0.0):
    best_score, best_offset, best_k, all_score, all_offset = out
    for t in range(len(c["cs"])):
        ref = vo.energy_zcr_detect(c["pcms"][c["track_video"][t]], 100, 16000, label)
        for k, r in enumerate(GRID):
            sub = ro.rasterize(c["cs"][t], c["ce"][t], None, 100, 0, r)[0]
            ws, wo = ao.fft_align(ref, sub, mos)
            j = t * len(GRID) + k
            assert abs(all_score[j] - ws) <= 1e-5 * max(abs(ws), 1e-3) + 1e-6, (t, k, all_score[j], ws)
            if all_offset[j] != wo:   # a tie, which the oracle's complex128 round-off breaks its own way
                x, y = _exact_at(ref, sub, all_offset[j]), _exact_at(ref, sub, wo)
                assert abs(x - y) <= 1e-12 * max(abs(y), 1.0), (t, k, all_offset[j], wo, x, y)


def _exact_at(ref, sub, o):
    """sum_j (2 sub[j] - 1)(2 ref[j + o] - 1) over the overlap, in float64."""
    lo, hi = max(0, -o), min(len(sub), len(ref) - o)
    if hi <= lo:
        return 0.0
    return float(np.dot(2.0 * sub[lo:hi] - 1.0, 2.0 * ref[lo + o:hi + o] - 1.0))


VIDEOS = [(240.0, [(0, 250)]), (300.0, [(2, -700), (4, 0), (1, 1234)]), (120.0, []),
          (200.0, [(3, 40), (0, -1500), (2, 9), (4, 600), (1, -321)]), (45.0, [(0, 3)]),
          (180.0, [(1, 5999), (3, -6000)])]


@pytest.fixture(scope="module")
def corpus():
    return _corpus(VIDEOS, seed0=5)


@pytest.mark.parametrize("label", [0.0, 0.3])
@pytest.mark.parametrize("mos", [6000, 14000])
def test_runs_equal_tiled_per_ratio_and_winners(handle, corpus, label, mos):
    """Default (run path) == B2_ALIGN_PATH=tiled bit for bit: per-ratio scores / offsets and winners, with
    and without per-ratio outputs (winner-only pruning), for +-1 and two-level signals, and windows of
    12 001 and 28 001 offsets."""
    with _env(B2_ALIGN_PATH="runs"):
        forced, n_runs = _batch(handle, corpus, mos, label)
    with _env(B2_ALIGN_PATH="tiled"):
        tiled, n_tiled = _batch(handle, corpus, mos, label)
        tiled_w, _ = _batch(handle, corpus, mos, label, want_all=False)
    got, n_def = _batch(handle, corpus, mos, label)
    got_w, _ = _batch(handle, corpus, mos, label, want_all=False)
    assert n_def == n_runs != n_tiled, (n_def, n_runs, n_tiled)   # the default took the run path
    _same(got, tiled)
    _same(forced, tiled)
    _same(got_w[:3], tiled_w[:3])
    _same(got_w[:3], got[:3])
    _oracle_check(corpus, got, mos, label)


@pytest.mark.parametrize("n_sub", [1, 2, 3, 4])
def test_runs_vs_oracle_sub_batches(handle, n_sub):
    """The run path inside the sub-batch pipeline, 1-4 sub-batches."""
    c = _corpus([(150.0, [(k % 5, 37 * k - 400)]) for k in range(8)], seed0=40 + n_sub)
    with _env(B2_SUBBATCHES=n_sub, B2_VAD_SMS=60):
        got, _ = _batch(handle, c, 6000)
    _oracle_check(c, got, 6000)
    with _env(B2_SUBBATCHES=n_sub, B2_VAD_SMS=60, B2_ALIGN_PATH="tiled"):
        tiled, _ = _batch(handle, c, 6000)
    _same(got, tiled)


def test_runs_tracks_equal_tiled_and_oracle(handle, corpus):
    got, _ = _tracks(handle, corpus, 6000)
    with _env(B2_ALIGN_PATH="tiled"):
        tiled, _ = _tracks(handle, corpus, 6000)
    _same(got, tiled)
    _oracle_check(corpus, got, 6000)
    with _env(B2_SUBBATCHES=3, B2_VAD_SMS=60):
        piped, _ = _tracks(handle, corpus, 6000, want_all=False)
    _same(piped[:3], got[:3])


def test_runs_resident_chained_calls(handle):
    """B2_DEVICE_RESIDENT chains (the bench's call mode) on the run path equal ordered calls and the tiled path."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    bs = BatchSynchronizer(BENCH_RATIOS, 16000, 100, 0.0, max_offset_seconds=60)
    corpora = []
    for seed0, B in ((300, 110), (700, 97)):
        pairs = make_pairs([seed0 + b for b in range(B)], 600.0, BENCH_RATIOS, handle=bs.handle)
        n_win = int(pairs.win_off[-1])
        cls_d = torch.from_numpy(pairs.window_class).cuda()
        pcm = torch.empty(n_win * 160, dtype=torch.int16, device="cuda")
        bs.handle.synth_pcm(cls_d.data_ptr(), n_win, 160, seed0, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
        bs.handle.synchronize()
        args = (pcm, pairs.win_off * 160, pairs.cue_start, pairs.cue_end, pairs.cue_off)
        with _env(B2_ALIGN_PATH="tiled"):
            want = bs.sync_device(*args)
            bs.handle.synchronize()
            want = {k: v.clone() for k, v in want.items()}
        assert (want["best_offset"].cpu().numpy() == pairs.true_offset).all()
        corpora.append((args, want))
    order = [0, 1, 1, 0, 1, 0]
    outs = [bs.sync_device(*corpora[i][0], inputs_resident=True) for i in order]
    bs.handle.synchronize()
    torch.cuda.synchronize()
    for i, got in zip(order, outs):
        for k in ("best_score", "best_offset", "best_k"):
            assert torch.equal(got[k], corpora[i][1][k]), (i, k)


def test_capture_keeps_the_fft_path(handle, corpus):
    """b2_capture_nominations probes the fp32 FFT nomination: a call under a capture takes the tiled path
    (its window scores are captured) and returns what the run path returns."""
    J = len(corpus["cs"]) * len(GRID)
    with handle.capture_nominations(J, 16384) as cap:
        got, n_cap = _batch(handle, corpus, 6000)
    with _env(B2_ALIGN_PATH="tiled"):
        _, n_tiled = _batch(handle, corpus, 6000)
    plain, n_def = _batch(handle, corpus, 6000)
    assert n_cap > n_tiled  # tiled + the capture kernel
    assert n_cap != n_def
    assert (cap["win"][:, 1] > 9000).all()   # every job's fp32 window scores were captured
    _same(got, plain)


def test_large_windows_keep_the_big_path(handle):
    """Windows beyond the tiled plan (here +-10 min) stay on the large-FFT path."""
    c = _corpus([(900.0, [(0, 600), (2, -9000)])], seed0=77)
    with _env(B2_ALIGN_PATH="big"):
        big, n_big = _batch(handle, c, 60000)
    got, n_def = _batch(handle, c, 60000)
    assert n_def == n_big
    _same(got, big)
    # wider than one CTA's 32 x 1024 offsets: the run path cannot be forced
    with _env(B2_ALIGN_PATH="runs"):
        forced, n_forced = _batch(handle, c, 60000)
    with _env(B2_ALIGN_PATH="tiled"):
        tiled, n_tiled = _batch(handle, c, 60000)
    assert n_forced == n_tiled
    _same(forced, tiled)
