"""GPU tests of b2_sync_tracks: several subtitle tracks per video in one call (run on an H100).

Each video is a seeded master cue list whose speech mask, with 10 % of the frames flipped, is the reference
signal of the video's synthetic PCM.  Each track is the master cue list at its own framerate ratio and
delay, with dropped and jittered cues, so the tracks of one video have different true answers."""
import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
FPW = 160
MOS = 6000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _score_ok(got, want):
    if np.isinf(want) or np.isinf(got):
        return got == want
    return abs(got - want) <= 1e-5 * max(abs(want), 1e-3) + 1e-6


def _track(starts, ends, k, delta, seed, keep_until=None):
    """Master cues (seconds) -> a track that rasterised at GRID[k] and moved by delta frames lies on them."""
    rng = np.random.RandomState(seed)
    keep = rng.rand(len(starts)) >= 0.1                         # 10 % of the cues dropped
    if keep_until is not None:
        keep &= ends <= keep_until
    jit = rng.randint(-1, 2, len(starts)) * 0.01                # +-10 ms on every cue
    st = (starts - delta / 100.0 + jit) / GRID[k]
    en = (ends - delta / 100.0 + jit) / GRID[k]
    keep &= st >= 0
    return np.round(st[keep], 3), np.round(en[keep], 3)


def _corpus(videos, seed0=0):
    """videos: list of (duration_s, [(k, delta[, keep_until]) per track]).  Returns the inputs of
    b2_sync_tracks plus the per-video PCM and per-track cue lists."""
    pcms, tv, cs, ce, planted = [], [], [], [], []
    for v, (dur, tracks) in enumerate(videos):
        seed = seed0 + 31 * v + 7
        starts, ends = cases.synthetic_cues(seed, dur)
        mask = ro.rasterize(starts, ends, None, 100, 0, 1.0)[0] != 0
        n = int(dur * 100)
        ref = np.zeros(n, dtype=bool)
        ref[: min(n, len(mask))] = mask[:n]
        rng = np.random.RandomState(seed + 1000)
        ref ^= rng.rand(n) < 0.10
        hiss = rng.rand(n) < 0.05
        cls = np.where(ref, 1, np.where(hiss, 2, 0)).astype(np.uint8)
        pcms.append(vo.synth_pcm(cls, FPW, seed=seed))
        for i, tr in enumerate(tracks):
            k, delta = tr[0], tr[1]
            st, en = _track(starts, ends, k, delta, seed * 100 + i, tr[2] if len(tr) > 2 else None)
            tv.append(v)
            cs.append(st)
            ce.append(en)
            planted.append((k, delta))
    pcm_off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
    cue_off = np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64)
    return dict(pcm=np.concatenate(pcms), pcm_off=pcm_off, track_video=np.array(tv, np.int32),
                cue_start=np.concatenate(cs), cue_end=np.concatenate(ce), cue_off=cue_off,
                pcms=pcms, cs=cs, ce=ce, planted=planted)


def _run_tracks(handle, c, mos=MOS, want_all=True, grid=GRID):
    return handle.sync_tracks(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, 100000, -1, -1,
                              c["cue_start"], c["cue_end"], None, c["cue_off"], grid, 0.0, mos, want_all=want_all)


def _run_pairs(handle, c, mos=MOS, want_all=True, grid=GRID):
    """The same tracks through b2_sync_batch, each video's PCM copied once per track."""
    pcm = np.concatenate([c["pcms"][v] for v in c["track_video"]])
    pcm_off = np.concatenate([[0], np.cumsum([len(c["pcms"][v]) for v in c["track_video"]])]).astype(np.int64)
    return handle.sync_batch(pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, c["cue_start"], c["cue_end"], None,
                             c["cue_off"], grid, 0.0, mos, want_all=want_all)


def _same(a, b, n=5):
    for x, y in zip(a[:n], b[:n]):
        assert np.array_equal(x, y), (x, y)


def _ref_sig(c, v):
    memo = c.setdefault("ref_sigs", {})
    if v not in memo:
        memo[v] = vo.energy_zcr_detect(c["pcms"][v], 100, 16000, 0.0)
    return memo[v]


def _oracle(c, t, mos, grid=GRID):
    ref_sig = _ref_sig(c, c["track_video"][t])
    subs = [ro.rasterize(c["cs"][t], c["ce"][t], None, 100, 0, r)[0] for r in grid]
    return [ao.fft_align(ref_sig, s, mos) for s in subs]


# 4 videos with 1, 3, 0 and 5 tracks
VIDEOS = [(240.0, [(0, 250)]),
          (300.0, [(2, -700), (4, 0), (1, 1234)]),
          (120.0, []),
          (200.0, [(3, 40), (0, -1500), (2, 9), (4, 600), (1, -321)])]


@pytest.fixture(scope="module")
def corpus():
    return _corpus(VIDEOS, seed0=1)


def test_tracks_vs_oracle(handle, corpus):
    c = corpus
    bs, bo, bk, a_s, a_o = _run_tracks(handle, c)
    K = len(GRID)
    assert len(bs) == len(c["planted"]) == 9
    for t, (k, delta) in enumerate(c["planted"]):
        results = _oracle(c, t, MOS)
        for kk, (ws, wo) in enumerate(results):
            assert a_o[t * K + kk] == wo, (t, kk)
            assert _score_ok(a_s[t * K + kk], ws), (t, kk)
        wk = ao.max_score_select(results, MOS)
        assert (bk[t], bo[t]) == (wk, results[wk][1]) == (k, delta), t
        assert _score_ok(bs[t], results[wk][0])


def test_tracks_equal_duplicated_pairs(handle, corpus, monkeypatch):
    c = corpus
    want = _run_pairs(handle, c)
    _same(_run_tracks(handle, c), want)
    _same(_run_tracks(handle, c, want_all=False), want, 3)          # winner-only
    _same(_run_pairs(handle, c, want_all=False), want, 3)
    envs = [{"B2_SUBBATCHES": n} for n in ("1", "2", "3", "4")] + [
        {"B2_FUSED_RASTER": "0"}, {"B2_FUSED_RASTER": "0", "B2_SUBBATCHES": "3"},
        {"B2_ALIGN_SPLIT": "1"}, {"B2_ALIGN_SPLIT": "5"}]
    for env in envs:
        with monkeypatch.context() as m:
            for k_, v_ in env.items():
                m.setenv(k_, v_)
            _same(_run_tracks(handle, c), want)
            _same(_run_tracks(handle, c, want_all=False), want, 3)


def test_tracks_device_memspace(handle, corpus):
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    want = _run_pairs(handle, c)
    bs = BatchSynchronizer(GRID, 16000, 100, 0.0, max_offset_seconds=MOS / 100)
    host = bs.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                               want_all=True)
    _same(host, want)
    pcm = torch.from_numpy(c["pcm"]).cuda()
    T, K = len(c["track_video"]), len(GRID)
    all_out = {"score": torch.empty(T * K, dtype=torch.float64, device="cuda"),
               "offset": torch.empty(T * K, dtype=torch.int32, device="cuda")}
    for kw in ({"all_out": all_out}, {}):
        out = bs.sync_device_tracks(pcm, c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                                    **kw)
        bs.handle.synchronize()
        got = [out[k].cpu().numpy() for k in ("best_score", "best_offset", "best_k")]
        if kw:
            got += [all_out["score"].cpu().numpy(), all_out["offset"].cpu().numpy()]
        _same(got, want, len(got))


def test_tracks_large_window_slices(handle, monkeypatch):
    """Unmasked: one 25-minute video whose five tracks have padded lengths 2^19 and 2^18 (two tracks keep only
    the first half of the cues), and a second video.  With a 64 MB budget the large-window path cuts the first
    video's tracks into slices of three; both paths agree with the oracle."""
    c = _corpus([(1500.0, [(0, 300), (2, -450, 700.0), (4, 0), (1, 77, 700.0), (3, -20)]),
                 (400.0, [(2, 100), (0, -90)])], seed0=500)
    T, K = len(c["track_video"]), len(GRID)
    want = [_oracle(c, t, None) for t in range(T)]
    for path in ("big", "tiled"):
        with monkeypatch.context() as m:
            m.setenv("B2_ALIGN_PATH", path)
            m.setenv("B2_BIG_WS_MB", "64")
            bs, bo, bk, a_s, a_o = _run_tracks(handle, c, mos=None)
            bs2, bo2, bk2, _, _ = _run_tracks(handle, c, mos=None, want_all=False)
        for t in range(T):
            for kk, (ws, wo) in enumerate(want[t]):
                assert a_o[t * K + kk] == wo and _score_ok(a_s[t * K + kk], ws), (path, t, kk)
            wk = ao.max_score_select(want[t], None)
            assert (bk[t], bo[t]) == (wk, want[t][wk][1]) == c["planted"][t], (path, t)
            assert (bk2[t], bo2[t], bs2[t]) == (bk[t], bo[t], bs[t]), (path, t)


def test_tracks_resident_chained_calls_equal_ordered_calls(handle, monkeypatch):
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    monkeypatch.setenv("B2_SUBBATCHES", "3")   # pipelined calls: resident calls chain
    bs = BatchSynchronizer(GRID, 16000, 100, 0.0, max_offset_seconds=MOS / 100)
    rng = np.random.RandomState(8)
    corpora = []
    for seed0, n_tracks in ((100, [2, 1, 4, 0, 3, 1]), (900, [3, 5, 1, 2])):
        vids = [(150.0, [(int(rng.randint(0, 5)), int(rng.randint(-2000, 2001))) for _ in range(n)])
                for n in n_tracks]
        c = _corpus(vids, seed0=seed0)
        args = (torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                c["cue_off"])
        want = bs.sync_device_tracks(*args)
        bs.handle.synchronize()
        want = {k: v.clone() for k, v in want.items()}
        corpora.append((args, want))
    order = [0, 1, 0, 0, 1, 1, 0, 1]
    outs = [bs.sync_device_tracks(*corpora[i][0], inputs_resident=True) for i in order]   # nothing synchronised
    bs.handle.synchronize()
    for i, got in zip(order, outs):
        for k in ("best_score", "best_offset", "best_k"):
            assert torch.equal(got[k], corpora[i][1][k]), (i, k)


def test_identity_map_equals_sync_batch(handle, corpus):
    """One track per video: b2_sync_tracks is b2_sync_batch, launches included."""
    c = dict(corpus)
    c["track_video"] = np.arange(len(c["pcm_off"]) - 1, dtype=np.int32)
    c["cs"] = [c["cs"][t] for t in (0, 1, 4, 3)]   # one cue list for each of the 4 videos
    c["ce"] = [c["ce"][t] for t in (0, 1, 4, 3)]
    c["cue_start"], c["cue_end"] = np.concatenate(c["cs"]), np.concatenate(c["ce"])
    c["cue_off"] = np.concatenate([[0], np.cumsum([len(x) for x in c["cs"]])]).astype(np.int64)
    for want_all in (True, False):
        n0 = handle.launch_count
        a = _run_tracks(handle, c, want_all=want_all)
        n1 = handle.launch_count
        b = handle.sync_batch(c["pcm"], c["pcm_off"], 16000, 100, 0.0, 100000, -1, -1, c["cue_start"],
                              c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, want_all=want_all)
        n2 = handle.launch_count
        _same(a, b, 5 if want_all else 3)
        assert n1 - n0 == n2 - n1 > 0


def test_tracks_nominations_within_tau(handle, corpus):
    from test_gpu_nomination import _Exact, _check_jobs
    c = corpus
    T, K = len(c["track_video"]), len(GRID)
    refs = [_ref_sig(c, v) for v in range(len(c["pcms"]))]
    level = [float(np.float32(min(1.0 / r, 1.0))) for r in GRID]   # the level the kernels use
    sigs = [(refs[c["track_video"][t]], (ro.rasterize(c["cs"][t], c["ce"][t], None, 100, 0, r)[0] != 0) * level[k])
            for t in range(T) for k, r in enumerate(GRID)]
    stride = max(ao.offset_range(len(r), len(s), MOS)[1] - ao.offset_range(len(r), len(s), MOS)[0] + 1
                 for r, s in sigs)
    for want_all in (True, False):
        with handle.capture_nominations(T * K, stride) as cap:
            res = _run_tracks(handle, c, want_all=want_all)
        out = (res[3], res[4], None) if want_all else None
        _check_jobs(cap, sigs, MOS, _Exact(), ("tracks", "bits"), out=out, winner_only=not want_all, K=K)


def test_tracks_bad_arguments(handle, corpus):
    import torch
    from ffsubsync_b200 import _native
    c = corpus

    def call(**kw):
        a = dict(c)
        a.update(kw)
        with pytest.raises(_native.NativeError) as ei:
            handle.sync_tracks(a["pcm"], a["pcm_off"], a["track_video"], 16000, 100, 0.0, 100000, -1, -1,
                               a["cue_start"], a["cue_end"], None, a["cue_off"], GRID, 0.0, MOS,
                               memspace=a.get("memspace", _native.B2_HOST))
        assert ei.value.status == -1, ei.value

    tv = c["track_video"].copy()
    dec = tv.copy()
    dec[[0, 1]] = dec[[1, 0]]                                  # 1, 0, ...: decreasing
    call(track_video=dec)
    big = tv.copy()
    big[-1] = len(c["pcm_off"]) - 1                            # index == V
    call(track_video=big)
    neg = tv.copy()
    neg[0] = -1
    call(track_video=neg)
    call(cue_off=c["cue_off"][:-1])                            # cue_off of the wrong length
    bad_pcm_off = c["pcm_off"].copy()
    bad_pcm_off[1] = bad_pcm_off[2] + 1                        # not monotone
    call(pcm_off=bad_pcm_off)
    bad_cue_off = c["cue_off"].copy()
    bad_cue_off[1] = bad_cue_off[2] + 1
    call(cue_off=bad_cue_off)
    # B2_DEVICE with a host PCM pointer, and with host outputs
    T = len(tv)
    outs = [torch.empty(T, dtype=dt, device="cuda") for dt in (torch.float64, torch.int32, torch.int32)]
    with pytest.raises(_native.NativeError) as ei:
        handle.sync_tracks(c["pcm"].ctypes.data, c["pcm_off"], tv, 16000, 100, 0.0, 100000, -1, -1, c["cue_start"],
                           c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, *(o.data_ptr() for o in outs),
                           memspace=_native.B2_DEVICE)
    assert ei.value.status == -1
    pcm_d = torch.from_numpy(c["pcm"]).cuda()
    host_k = np.empty(T, np.int32)
    with pytest.raises(_native.NativeError) as ei:
        handle.sync_tracks(pcm_d.data_ptr(), c["pcm_off"], tv, 16000, 100, 0.0, 100000, -1, -1, c["cue_start"],
                           c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, outs[0].data_ptr(), outs[1].data_ptr(),
                           host_k.ctypes.data, memspace=_native.B2_DEVICE)
    assert ei.value.status == -1
    # null outputs
    grid = np.array(GRID)
    st = handle.lib.b2_sync_tracks(handle.h, pcm_d.data_ptr(), c["pcm_off"].ctypes.data, len(c["pcm_off"]) - 1,
                                   tv.ctypes.data, T, 16000, 100, 0.0, 100000, -1, -1, c["cue_start"].ctypes.data,
                                   c["cue_end"].ctypes.data, None, c["cue_off"].ctypes.data,
                                   grid.ctypes.data, len(GRID), 0.0, MOS, None, None, None, None, None,
                                   _native.B2_DEVICE)
    assert st == -1
    # nothing to sync: legal
    assert _run_tracks(handle, dict(c, track_video=np.zeros(0, np.int32), cue_off=c["cue_off"][:1]))[0].shape == (0,)


def test_sync_batch_rejects_a_host_output_under_b2_device(handle, corpus):
    """b2_sync_batch checks every device output the way the track calls do, before it launches anything."""
    import torch
    from ffsubsync_b200 import _native
    c = corpus
    B = len(c["pcm_off"]) - 1
    cue_off = c["cue_off"][: B + 1]                  # the first B tracks, track b against video b
    pcm_d = torch.from_numpy(c["pcm"]).cuda()
    dev = dict(best_score=torch.empty(B, dtype=torch.float64, device="cuda"),
               best_offset=torch.empty(B, dtype=torch.int32, device="cuda"),
               best_k=torch.empty(B, dtype=torch.int32, device="cuda"),
               all_score=torch.empty(B * len(GRID), dtype=torch.float64, device="cuda"),
               all_offset=torch.empty(B * len(GRID), dtype=torch.int32, device="cuda"))
    args = (c["pcm_off"], 16000, 100, 0.0, 100000, -1, -1, c["cue_start"], c["cue_end"], None, cue_off, GRID, 0.0, MOS)
    handle.sync_batch(pcm_d.data_ptr(), *args, **{k: v.data_ptr() for k, v in dev.items()},
                      memspace=_native.B2_DEVICE)
    handle.synchronize()
    for host in dev:
        host_buf = np.empty(dev[host].numel(), dtype=dev[host].cpu().numpy().dtype)
        ptrs = {k: (host_buf.ctypes.data if k == host else v.data_ptr()) for k, v in dev.items()}
        n0 = handle.launch_count
        with pytest.raises(_native.NativeError) as ei:
            handle.sync_batch(pcm_d.data_ptr(), *args, **ptrs, memspace=_native.B2_DEVICE)
        assert ei.value.status == -1 and "sync_batch: %s" % host in str(ei.value), host
        assert handle.launch_count == n0, host
