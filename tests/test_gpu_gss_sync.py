"""GPU tests of b2_sync_tracks_gss: the golden-section search over the ratio as candidate K of the batched
sync, its 17 rounds driven on the device (run on an H100).

The yardstick is the composition of existing public entry points - the VAD (b2_vad_energy_zcr), the grid
(b2_sync_tracks with per-ratio outputs), gss_align_batch on the VAD signals (float subtitle signals, the FFT
aligner, one host round trip per round) and the reference's combine - which the new call must reproduce bit
for bit: the 17 points of every track, the candidate's score and offset, best_* and all_*."""
import math

import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import gss_oracle as go
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
FPW = 160
MOS = 6000
EVALS = 17


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _corpus(videos, seed0=0):
    """videos: list of (duration_s, [(ratio, delta) per track]).  Each video's reference is its master cue
    list's mask with 10 % of the frames flipped; a track is the master list at its own ratio and delay with
    dropped and jittered cues.  duration 0: a video without PCM (empty reference)."""
    pcms, tv, cs, ce = [], [], [], []
    for v, (dur, tracks) in enumerate(videos):
        seed = seed0 + 31 * v + 7
        starts, ends = cases.synthetic_cues(seed, max(dur, 60.0))
        n = int(dur * 100)
        mask = ro.rasterize(starts, ends, None, 100, 0, 1.0)[0] != 0
        ref = np.zeros(n, dtype=bool)
        ref[: min(n, len(mask))] = mask[:n]
        rng = np.random.RandomState(seed + 1000)
        ref ^= rng.rand(n) < 0.10
        hiss = rng.rand(n) < 0.05
        cls = np.where(ref, 1, np.where(hiss, 2, 0)).astype(np.uint8)
        pcms.append(vo.synth_pcm(cls, FPW, seed=seed) if n else np.zeros(0, np.int16))
        for i, (ratio, delta) in enumerate(tracks):
            r2 = np.random.RandomState(seed * 100 + i)
            keep = r2.rand(len(starts)) >= 0.1
            jit = r2.randint(-1, 2, len(starts)) * 0.01
            st = (starts - delta / 100.0 + jit) / ratio
            en = (ends - delta / 100.0 + jit) / ratio
            keep &= st >= 0
            tv.append(v)
            cs.append(np.round(st[keep], 3))
            ce.append(np.round(en[keep], 3))
    pcm_off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
    cue_off = np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64)
    return dict(pcm=np.concatenate(pcms), pcm_off=pcm_off, track_video=np.array(tv, np.int32),
                cue_start=np.concatenate(cs), cue_end=np.concatenate(ce), cue_off=cue_off, pcms=pcms, cs=cs, ce=ce)


def _args(c, grid, mos, label=0.0):
    return (c["pcm_off"], c["track_video"], 16000, 100, label, 100000, -1, -1, c["cue_start"], c["cue_end"], None,
            c["cue_off"], grid, 0.0, mos)


def _new(handle, c, grid=GRID, mos=MOS):
    bs, bo, bk, a_s, a_o, r, ev = handle.sync_tracks_gss(c["pcm"], *_args(c, grid, mos), want_all=True,
                                                         want_evals=True)
    return dict(bs=bs, bo=bo, bk=bk, a_s=a_s, a_o=a_o, ratio=r, evals=ev.reshape(-1, EVALS))


def _compose(handle, c, grid=GRID, mos=MOS):
    """VAD -> b2_sync_tracks(all_out) -> gss_align_batch on the VAD signals -> the reference's combine."""
    from ffsubsync_b200 import _native
    from ffsubsync_b200.gss_batch import combine_gss, gss_align_batch
    gbs, gbo, gbk, gas, gao = handle.sync_tracks(c["pcm"], *_args(c, grid, mos), want_all=True)
    ref, ref_off = handle.vad_energy_zcr(c["pcm"], c["pcm_off"], 16000, 100, 0.0, 100000)
    parts = [ref[ref_off[v]: ref_off[v + 1]] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    g = gss_align_batch(np.concatenate(parts).astype(np.float32), t_off, c["cue_start"], c["cue_end"], c["cue_off"],
                        None, mos, 100, 0.0, handle=handle)
    assert not np.any(g.status & _native.ALIGN_CAND_OVERFLOW)
    bs, bo, bk, r, a_s, a_o = combine_gss(gbs, gbo, gbk, g, len(grid), mos, gas, gao)
    return dict(bs=bs, bo=bo, bk=bk, a_s=a_s, a_o=a_o, ratio=r, evals=g.evals, status=g.status, score=g.score,
                offset=g.offset)


def _assert_same(got, want, K):
    T = len(want["bk"])
    live = (want["status"] & 1) == 0
    assert np.array_equal(got["evals"][live], want["evals"][live])
    assert np.all(np.isnan(got["evals"][~live])) and np.all(np.isnan(got["ratio"][~live]))
    assert np.array_equal(got["ratio"][live], want["ratio"][live])
    assert np.array_equal(got["ratio"][live], got["evals"][live, -1])
    a_s, a_o = got["a_s"].reshape(T, K + 1), got["a_o"].reshape(T, K + 1)
    assert np.array_equal(a_s[live, K], want["score"][live]) and np.array_equal(a_o[live, K], want["offset"][live])
    # all-masked windows: -inf in both, with B2_ALIGN_ALL_MASKED in the composition
    assert np.array_equal(np.isinf(a_s[live, K]), (want["status"][live] & 2) != 0)
    for key in ("bs", "bo", "bk", "a_s", "a_o"):
        assert np.array_equal(got[key], want[key]), key


# videos with 1, 3, 0 and 2 tracks, one without PCM (empty reference)
VIDEOS = [(240.0, [(1.0, 250)]),
          (300.0, [(1.037, -700), (24 / 25.0, 0), (0.955, 1234)]),
          (120.0, []),
          (0.0, [(1.0, 0)]),
          (200.0, [(1.0712, 40), (25 / 24.0, -1500)])]


@pytest.fixture(scope="module")
def corpus():
    return _corpus(VIDEOS, seed0=1)


def test_gss_equals_composition(handle, corpus):
    got, want = _new(handle, corpus), _compose(handle, corpus)
    _assert_same(got, want, len(GRID))
    # a track whose video has no windows: the grid's answer (-1), no search
    t_empty = int(np.nonzero(corpus["track_video"] == 3)[0][0])
    assert got["bk"][t_empty] == -1 and np.isnan(got["ratio"][t_empty])


def test_gss_candidate_outcomes(handle, corpus):
    got = _new(handle, corpus)
    K = len(GRID)
    # off-grid true ratios: the search wins and lands near the planted ratio
    for t, planted in ((1, 1.037), (3, 0.955), (5, 1.0712)):
        assert got["bk"][t] == K, (t, got["bk"][t], got["ratio"][t])
        assert abs(got["ratio"][t] - planted) < 3e-3, (t, got["ratio"][t])
    # on-grid true ratios: a grid ratio keeps the win
    for t, k in ((0, 0), (2, 4), (6, 2)):
        assert got["bk"][t] == k, (t, got["bk"][t])


def test_gss_exact_tie_goes_to_the_grid(handle):
    # the search's 17th point of a track put in the grid scores exactly what the search's candidate scores
    c = _corpus([(200.0, [(1.0712, 40)])], seed0=5)
    first = _new(handle, c)
    x17 = float(first["ratio"][0])
    grid = [1.0, x17]
    got, want = _new(handle, c, grid=grid), _compose(handle, c, grid=grid)
    _assert_same(got, want, 2)
    a_s = got["a_s"].reshape(1, 3)
    assert a_s[0, 1] == a_s[0, 2] and got["bk"][0] == 1 and got["ratio"][0] == x17


def test_gss_all_masked_windows(handle, corpus):
    # max_offset_samples = 0 leaves no offset of any window: -inf in every round, IEEE bookkeeping
    from ffsubsync_b200.golden_section_search import gss
    got, want = _new(handle, corpus, mos=0), _compose(handle, corpus, mos=0)
    _assert_same(got, want, len(GRID))
    pts = []
    gss(lambda x, last: pts.append(x) or math.inf, 0.9, 1.1)
    live = corpus["track_video"] != 3
    assert np.all(got["evals"][live] == np.array(pts))


def test_gss_host_device_and_subbatches(handle, monkeypatch):
    import torch
    from ffsubsync_b200 import _native
    # 80 videos, 100 tracks (one, two or none per video): the sub-batch pipeline runs
    rng = np.random.RandomState(2)
    videos = []
    for v in range(80):
        n = [1, 2, 0, 2][v % 4]
        videos.append((60.0 + 5 * (v % 7), [(float(rng.uniform(0.92, 1.08)), int(rng.randint(-800, 800)))
                                            for _ in range(n)]))
    c = _corpus(videos, seed0=11)
    T, K = len(c["track_video"]), len(GRID)
    assert T >= 96
    want = _compose(handle, c)
    for n_sub in ("1", "3"):
        monkeypatch.setenv("B2_SUBBATCHES", n_sub)
        _assert_same(_new(handle, c), want, K)
        dev = torch.device("cuda", handle.device)
        pcm = torch.from_numpy(c["pcm"]).to(dev)
        out = {k: torch.full((T,), -7, dtype=dt, device=dev)
               for k, dt in (("bs", torch.float64), ("bo", torch.int32), ("bk", torch.int32), ("r", torch.float64))}
        a_s = torch.zeros(T * (K + 1), dtype=torch.float64, device=dev)
        a_o = torch.zeros(T * (K + 1), dtype=torch.int32, device=dev)
        ev = torch.zeros(T * EVALS, dtype=torch.float64, device=dev)
        torch.cuda.synchronize(dev)
        handle.sync_tracks_gss(pcm.data_ptr(), *_args(c, GRID, MOS), best_score=out["bs"].data_ptr(),
                               best_offset=out["bo"].data_ptr(), best_k=out["bk"].data_ptr(), all_score=a_s.data_ptr(),
                               all_offset=a_o.data_ptr(), gss_ratio=out["r"].data_ptr(), gss_evals=ev.data_ptr(),
                               memspace=_native.B2_DEVICE)
        handle.synchronize()
        got = dict(bs=out["bs"].cpu().numpy(), bo=out["bo"].cpu().numpy(), bk=out["bk"].cpu().numpy(),
                   a_s=a_s.cpu().numpy(), a_o=a_o.cpu().numpy(), ratio=out["r"].cpu().numpy(),
                   evals=ev.cpu().numpy().reshape(T, EVALS))
        _assert_same(got, want, K)


def test_gss_resident_calls_alternate_with_sync_batch(handle):
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    rng = np.random.RandomState(3)
    ca = _corpus([(70.0, [(float(rng.uniform(0.92, 1.08)), int(rng.randint(-500, 500))) for _ in range(2)])
                  for _ in range(50)], seed0=21)
    cb = _corpus([(80.0, [(GRID[v % 5], int(rng.randint(-500, 500)))]) for v in range(100)], seed0=41)
    want_a = _new(handle, ca)
    want_b = handle.sync_batch(cb["pcm"], cb["pcm_off"], 16000, 100, 0.0, 100000, -1, -1, cb["cue_start"],
                               cb["cue_end"], None, cb["cue_off"], GRID, 0.0, MOS)
    sg = BatchSynchronizer(GRID + [None], max_offset_seconds=MOS / 100)
    sb = BatchSynchronizer(GRID, max_offset_seconds=MOS / 100)
    assert sg.handle is sb.handle is handle
    dev = torch.device("cuda", handle.device)
    pa, pb = torch.from_numpy(ca["pcm"]).to(dev), torch.from_numpy(cb["pcm"]).to(dev)
    torch.cuda.synchronize(dev)
    outs = []
    for i in range(3):   # gss, batch, gss, batch, ... with no synchronisation in between
        oa = sg.sync_device_tracks(pa, ca["pcm_off"], ca["track_video"], ca["cue_start"], ca["cue_end"], ca["cue_off"],
                                   inputs_resident=True)
        ob = sb.sync_device(pb, cb["pcm_off"], cb["cue_start"], cb["cue_end"], cb["cue_off"], inputs_resident=True)
        outs.append((oa, ob))
    handle.synchronize()
    for oa, ob in outs:
        assert np.array_equal(oa["best_score"].cpu().numpy(), want_a["bs"])
        assert np.array_equal(oa["best_offset"].cpu().numpy(), want_a["bo"])
        assert np.array_equal(oa["best_k"].cpu().numpy(), want_a["bk"])
        assert np.array_equal(oa["gss_ratio"].cpu().numpy(), want_a["ratio"])
        for x, y in zip((ob["best_score"], ob["best_offset"], ob["best_k"]), want_b[:3]):
            assert np.array_equal(x.cpu().numpy(), y)
    # the batch form of the front end (identity track map) returns the same as the tracks form
    r = sg.sync_host(cb["pcm"], cb["pcm_off"], cb["cue_start"], cb["cue_end"], cb["cue_off"])
    w = handle.sync_tracks_gss(cb["pcm"], *_args(dict(cb, track_video=np.arange(100, dtype=np.int32)), GRID, MOS))
    for x, y in zip(r, (w[0], w[1], w[2], w[5])):
        assert np.array_equal(x, y)


def test_gss_envelope(handle, corpus):
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    # 1 << 62 is where the binding clamps every larger width (1 << 80 arrives as 1 << 62): twice it overflows int64
    for mos in (None, 16385, 10 ** 9, -1, 1 << 62, 1 << 80, (1 << 62) - 1):
        with pytest.raises(_native.NativeError) as e:
            handle.sync_tracks_gss(c["pcm"], *_args(c, GRID, mos))
        assert e.value.status == -6 and "max_offset_samples" in str(e.value)
    # INT64_MAX and INT64_MIN + 1 straight through the C ABI
    T, K = len(c["track_video"]), len(GRID)
    pcm = np.ascontiguousarray(c["pcm"])
    tv = np.ascontiguousarray(c["track_video"], np.int32)
    grid = np.array(GRID)
    outs = [np.empty(T), np.empty(T, np.int32), np.empty(T, np.int32), np.empty(T)]
    for mos in ((1 << 63) - 1, -(1 << 63) + 1):
        st = handle.lib.b2_sync_tracks_gss(handle.h, pcm.ctypes.data, c["pcm_off"].ctypes.data, len(c["pcm_off"]) - 1,
                                           tv.ctypes.data, T, 16000, 100, 0.0, 100000, -1, -1,
                                           c["cue_start"].ctypes.data, c["cue_end"].ctypes.data, None,
                                           c["cue_off"].ctypes.data, grid.ctypes.data, K, 0.0, mos,
                                           outs[0].ctypes.data, outs[1].ctypes.data, outs[2].ctypes.data, None, None,
                                           outs[3].ctypes.data, None, _native.B2_HOST)
        assert st == -6, (mos, st)
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_gss(c["pcm"], *_args(c, GRID, MOS, label=float("nan")))
    assert e.value.status == -6 and "non_speech_label" in str(e.value)
    many = dict(c)
    n = 16385
    many.update(cue_start=np.arange(n) * 0.02, cue_end=np.arange(n) * 0.02 + 0.01,
                cue_off=np.array([0, n] + [n] * (len(c["track_video"]) - 1), np.int64))
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_gss(c["pcm"], *_args(many, GRID, MOS))
    assert e.value.status == -6 and "16384" in str(e.value)
    handle.sync_tracks_gss(c["pcm"], *_args(c, GRID, 16384))   # the edge of the envelope runs
    # outside the envelope the front end composes the public steps
    for mos in (20000, None, 10 ** 19):
        sync = BatchSynchronizer(GRID + [None], max_offset_seconds=None if mos is None else mos / 100)
        assert sync.max_offset_samples == mos
        got = sync.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                                    c["cue_off"], want_all=True)
        want = _compose(handle, c, mos=mos)
        for x, key in zip(got, ("bs", "bo", "bk", "a_s", "a_o", "ratio")):
            assert np.array_equal(x, want[key], equal_nan=key == "ratio"), key


def test_gss_against_oracle(handle, corpus, record_property):
    """The oracle's search: its VAD and rasteriser and golden_section_trace over fft_align (a float64 FFT).
    Its scores carry FFT round-off, so an exact tie between two of its evaluations (or one within that
    round-off) may order differently from the exact scores; those are counted and reported, not skipped."""
    got = _new(handle, corpus)
    tracks = [0, 1, 3, 5]
    agree, ties = 0, 0
    for t in tracks:
        v = corpus["track_video"][t]
        ref = vo.energy_zcr_detect(corpus["pcms"][v], 100, 16000, 0.0)
        vals = []

        def f(x, last):
            s, o = ao.fft_align(ref, ro.rasterize(corpus["cs"][t], corpus["ce"][t], None, 100, 0, x)[0], MOS)
            vals.append((s, o))
            return -s

        _, calls = go.golden_section_trace(f, 0.9, 1.1)
        xs = np.array([x for x, _ in calls])
        ys = np.array([-s for s, _ in vals])
        n_tie = sum(int(ys[i] == ys[j]) for i in range(len(ys)) for j in range(i))
        ties += n_tie
        if np.array_equal(xs, got["evals"][t]):
            agree += 1
        else:
            # a different path is acceptable only behind a decision the FFT round-off could flip
            k = int(np.argmax(xs != got["evals"][t]))
            assert k >= 3
            near = any(abs(ys[i] - ys[j]) <= 1e-6 * max(1.0, abs(ys[i])) for i in range(k) for j in range(i))
            assert near, (t, k)
            continue
        # the winner: the oracle's grid and its 17th evaluation under MaxScoreAligner.transform
        cands = [ao.fft_align(ref, ro.rasterize(corpus["cs"][t], corpus["ce"][t], None, 100, 0, r)[0], MOS)
                 for r in GRID] + [vals[-1]]
        kept = [i for i, (s, o) in enumerate(cands) if abs(o) <= MOS]
        k_or = max(kept, key=lambda i: cands[i][0]) if kept else -1
        assert got["bk"][t] == k_or, (t, got["bk"][t], k_or)
        assert got["bo"][t] == cands[k_or][1]
        assert abs(got["bs"][t] - cands[k_or][0]) <= 1e-6 * abs(cands[k_or][0])
    record_property("oracle_exact_score_ties", ties)
    print("gss oracle: %d of %d tracks follow the oracle's path; %d exact score ties in its traces"
          % (agree, len(tracks), ties))
    assert agree >= len(tracks) - 1


def test_gss_sync_signals_and_candidate_sharding(handle, corpus):
    """sync_signals (reference signals instead of PCM) runs the search by composition; the candidate-sharded mode
    deals grid ratios over ranks and refuses a ratio list with the search."""
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    ref, ref_off = handle.vad_energy_zcr(c["pcm"], c["pcm_off"], 16000, 100, 0.0, 100000)
    parts = [ref[ref_off[v]: ref_off[v + 1]] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    sync = BatchSynchronizer(GRID + [None], max_offset_seconds=MOS / 100)
    got = sync.sync_signals(np.concatenate(parts), t_off, c["cue_start"], c["cue_end"], c["cue_off"])
    want = _compose(handle, c)
    for x, key in zip(got, ("bs", "bo", "bk", "ratio")):
        assert np.array_equal(x, want[key], equal_nan=key == "ratio"), key
    grid_only = BatchSynchronizer(GRID, max_offset_seconds=MOS / 100).sync_signals(
        np.concatenate(parts), t_off, c["cue_start"], c["cue_end"], c["cue_off"])
    assert len(grid_only) == 3
    import torch
    with pytest.raises(ValueError):
        sync.sync_device_candidate_sharded(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["cue_start"],
                                           c["cue_end"], c["cue_off"])
