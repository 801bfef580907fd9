"""GPU tests of b2_sync_tracks_auditok: the reference's auditok detector inside the batched sync calls, for the
grid, several tracks per video and the golden-section search (run on an H100).

Two yardsticks:
  * the oracle: oracle.auditok_oracle over the reference's chunk loop, the float64 FFT aligner and
    MaxScoreAligner's rule per ratio;
  * the per-stage composition of public entry points the call replaces - b2_vad_auditok (same detector arguments
    and chunk_samples), one rounding to float32, one copy of the video's signal per track, b2_rasterize,
    b2_align_batch, b2_reduce_ratios (and for the search gss_align_batch + the reference's combine) - which the
    call must reproduce bit for bit under every pipeline, path and memory knob."""
import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import auditok_oracle as au
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
MOS = 6000
EVALS = 17


def _chunk(fr):
    return (2 * fr // 100) * 5000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _corpus(videos, fr=16000, seed0=0):
    """videos: list of (duration_s, [(ratio, delay in frames) per track]).  A video's blocks pass auditok's
    energy test where its master cue list has speech (10 % flipped, 5 % loud hiss); a track is the master list at
    its own ratio and delay with dropped and jittered cues.  duration 0: a video without PCM."""
    fpw = fr // 100
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
        pcms.append(vo.synth_pcm(cls, fpw, seed=seed) if n else np.zeros(0, np.int16))
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
    return _pack(pcms, tv, cs, ce, fr)


def _pack(pcms, tv, cs, ce, fr):
    pcm_off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
    cue_off = np.concatenate([[0], np.cumsum([len(c) for c in cs])]).astype(np.int64)
    return dict(pcm=np.concatenate(pcms) if pcms else np.zeros(0, np.int16), pcm_off=pcm_off,
                track_video=np.array(tv, np.int32), cue_start=np.concatenate(cs), cue_end=np.concatenate(ce),
                cue_off=cue_off, pcms=pcms, cs=cs, ce=ce, fr=fr)


def _new(handle, c, label=0.0, grid=GRID, mos=MOS, chunk=None, gss=False, memspace=None):
    from ffsubsync_b200 import _native
    chunk = _chunk(c["fr"]) if chunk is None else chunk
    r = handle.sync_tracks_auditok(c["pcm"], c["pcm_off"], c["track_video"], c["fr"], 100, label, c["cue_start"],
                                   c["cue_end"], None, c["cue_off"], grid, 0.0, mos, chunk, gss=gss, want_all=True,
                                   want_evals=gss, memspace=_native.B2_HOST if memspace is None else memspace)
    out = dict(bs=r[0], bo=r[1], bk=r[2], a_s=r[3], a_o=r[4])
    if gss:
        out.update(ratio=r[5], evals=r[6].reshape(-1, EVALS))
    return out


def _ref(handle, c, label, chunk):
    """b2_vad_auditok over the chunk loop, rounded once to float32, one copy per track."""
    ref64, ref_off = handle.vad_auditok(c["pcm"], c["pcm_off"], c["fr"], 100, label, chunk_samples=chunk)
    ref = ref64.astype(np.float32)
    parts = [ref[ref_off[v]: ref_off[v + 1]] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    return (np.concatenate(parts) if parts else np.zeros(0, np.float32)), t_off, ref64, ref_off


def _compose(handle, c, label=0.0, grid=GRID, mos=MOS, chunk=None, gss=False):
    chunk = _chunk(c["fr"]) if chunk is None else chunk
    t_ref, t_off, _, _ = _ref(handle, c, label, chunk)
    T, K = len(c["track_video"]), len(grid)
    sub, sub_off = handle.rasterize(c["cue_start"], c["cue_end"], None, c["cue_off"], grid, K, False, 100, 0.0)
    score, offset, status = handle.align_batch(t_ref, t_off, sub, sub_off, T, K, mos)
    bs, bo, bk = handle.reduce_ratios(score, offset, status, T, K, mos)
    out = dict(bs=bs, bo=bo, bk=bk, a_s=score, a_o=offset)
    if gss:
        from ffsubsync_b200.gss_batch import combine_gss, gss_align_batch
        g = gss_align_batch(t_ref, t_off, c["cue_start"], c["cue_end"], c["cue_off"], None, mos, 100, 0.0,
                            handle=handle)
        bs, bo, bk, r, a_s, a_o = combine_gss(bs, bo, bk, g, K, mos, score, offset)
        out = dict(bs=bs, bo=bo, bk=bk, a_s=a_s, a_o=a_o, ratio=r, evals=g.evals, status=g.status)
    return out


def _same(got, want, keys=("bs", "bo", "bk", "a_s", "a_o"), where=""):
    for k in keys:
        assert np.array_equal(got[k], want[k]), (where, k, got[k], want[k])


# videos with 1, 3, 0 and 5 tracks; 240 s and 300 s cross the 100 s chunk boundaries
VIDEOS = [(240.0, [(1.0, 250)]),
          (300.0, [(25 / 24.0, -700), (24 / 25.0, 0), (1.0, 1234)]),
          (120.0, []),
          (210.0, [(1.0, 40), (25 / 24.0, -1500), (23.976 / 24, 300), (1.0, -2500), (24 / 23.976, 900)])]


@pytest.fixture(scope="module")
def corpus():
    return _corpus(VIDEOS, seed0=1)


@pytest.mark.parametrize("label", [0.0, 0.3])
def test_oracle_parity(handle, corpus, label):
    """Per ratio and for the winner.  Offsets: the oracle's, or one the exact float64 score (math.fsum) rates
    equal (a tie).  Scores at label 0: the reference is 0 / 1, so the call's score is the exact score of its offset
    - an integer wherever the subtitle level is 1 (ratio <= 1); at other labels within 1e-5 of the oracle's."""
    c = corpus
    got = _new(handle, c, label)
    chunk = _chunk(16000)
    K = len(GRID)
    for t, v in enumerate(c["track_video"]):
        pcm = c["pcms"][v]
        ref = np.concatenate([au.auditok_detect_fast(pcm[s: s + chunk].tobytes(), 100, 16000, label)
                              for s in range(0, len(pcm), chunk)])
        assert label != 0.0 or set(np.unique(ref).tolist()) <= {0.0, 1.0}
        subs = [ro.rasterize(c["cs"][t], c["ce"][t], None, 100, 0, r)[0] for r in GRID]
        cands = [ao.fft_align(ref, sub, MOS) for sub in subs]
        a_s, a_o = got["a_s"].reshape(-1, K)[t], got["a_o"].reshape(-1, K)[t]
        for k, (s, o) in enumerate(cands):
            if a_o[k] != o:   # only a tie may order differently
                assert ao.exact_score(ref, subs[k], int(a_o[k])) == ao.exact_score(ref, subs[k], int(o)), (t, k)
            if label == 0.0:
                # the subtitle level as the call holds it: float32
                exact = ao.exact_score(ref, subs[k].astype(np.float32), int(a_o[k]))
                if GRID[k] <= 1.0:
                    assert a_s[k] == exact and float(a_s[k]).is_integer(), (t, k, a_s[k], exact)
                else:
                    assert abs(a_s[k] - exact) <= 1e-12 * max(1.0, abs(exact)), (t, k, a_s[k], exact)
            else:
                assert abs(a_s[k] - s) <= 1e-5 * max(1.0, abs(s)), (t, k, a_s[k], s)
        kept = [k for k, (s, o) in enumerate(cands) if abs(o) <= MOS]
        k_or = max(kept, key=lambda k: cands[k][0]) if kept else -1
        kg, og = int(got["bk"][t]), int(got["bo"][t])
        if (kg, og) != (k_or, cands[k_or][1]):   # a tie across ratios or offsets: equal exact scores
            assert kg >= 0 and abs(og) <= MOS, (t, kg, og)
            assert ao.exact_score(ref, subs[kg], og) == ao.exact_score(ref, subs[k_or], cands[k_or][1]), (t, kg, k_or)


def test_grid_equals_composition_on_every_path_and_memspace(handle, monkeypatch):
    import torch
    from ffsubsync_b200 import _native
    # 80 videos of 120 s (two detector calls each), 100 tracks: the partitioned pipeline runs by default
    rng = np.random.RandomState(2)
    videos = [(120.0 + 3 * (v % 5), [(GRID[int(rng.randint(0, 5))], int(rng.randint(-800, 800)))
                                     for _ in range([1, 2, 0, 2][v % 4])]) for v in range(80)]
    c = _corpus(videos, seed0=11)
    T, K = len(c["track_video"]), len(GRID)
    assert T >= 96
    for label in (0.0, 0.3):
        want = _compose(handle, c, label)
        _same(_new(handle, c, label), want, where=("default", label))
        for env in ({"B2_SUBBATCHES": "1"}, {"B2_SUBBATCHES": "2"}, {"B2_SUBBATCHES": "4"},
                    {"B2_SUBBATCHES": "3", "B2_VAD_SMS": "8"}, {"B2_ALIGN_PATH": "tiled"},
                    {"B2_ALIGN_PATH": "runs"}, {"B2_ALIGN_PATH": "big"}, {"B2_FUSED_RASTER": "0"},
                    {"B2_VAD_LAYOUT": "group"}):
            with monkeypatch.context() as m:
                for k, v in env.items():
                    m.setenv(k, v)
                _same(_new(handle, c, label), want, where=(env, label))
        # device and resident memory
        dev = torch.device("cuda", handle.device)
        pcm = torch.from_numpy(c["pcm"]).to(dev)
        for ms in (_native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
            bs = torch.full((T,), -7, dtype=torch.float64, device=dev)
            bo, bk = torch.full((T,), -7, dtype=torch.int32, device=dev), torch.full((T,), -7, dtype=torch.int32,
                                                                                    device=dev)
            a_s = torch.zeros(T * K, dtype=torch.float64, device=dev)
            a_o = torch.zeros(T * K, dtype=torch.int32, device=dev)
            torch.cuda.synchronize(dev)
            handle.sync_tracks_auditok(pcm.data_ptr(), c["pcm_off"], c["track_video"], 16000, 100, label,
                                       c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS,
                                       _chunk(16000), best_score=bs.data_ptr(), best_offset=bo.data_ptr(),
                                       best_k=bk.data_ptr(), all_score=a_s.data_ptr(), all_offset=a_o.data_ptr(),
                                       memspace=ms)
            handle.synchronize()
            got = dict(bs=bs.cpu().numpy(), bo=bo.cpu().numpy(), bk=bk.cpu().numpy(), a_s=a_s.cpu().numpy(),
                       a_o=a_o.cpu().numpy())
            _same(got, want, where=(ms, label))


def test_large_window_path(handle, monkeypatch, corpus):
    # max_offset_seconds=None: FFTAligner's whole window, the large-window path
    for label in (0.0, -0.5):
        want = _compose(handle, corpus, label, mos=None)
        _same(_new(handle, corpus, label, mos=None), want, where=label)
        with monkeypatch.context() as m:
            m.setenv("B2_ALIGN_PATH", "tiled")
            _same(_new(handle, corpus, label, mos=None), want, where=("tiled", label))


def test_chunk_edges(handle):
    fr, chunk = 16000, _chunk(16000)
    rng = np.random.RandomState(5)
    fpw = 160
    pcms, tv, cs, ce = [], [], [], []
    # lengths chunk - 1, chunk, chunk + 1, and two videos whose second call ends on a 37-sample block after a
    # token and exactly max_continuous_silence (25) silent blocks: that block continues the token only if it
    # passes the energy test against its own floor (+-400 does, +-300 does not; a full block's floor is higher)
    edge = chunk + 35 * fpw + 37
    for v, n in enumerate((chunk - 1, chunk, chunk + 1, edge, edge)):
        cls = (rng.rand(n // fpw + 1) < 0.5).astype(np.uint8)
        if v >= 3:
            cls[10000:10010] = 1
            cls[10010:] = 0
        p = vo.synth_pcm(cls, fpw, seed=50 + v)[:n].copy()
        if v >= 3:
            amp = 400 if v == 3 else 300
            p[-37:] = np.where(np.arange(37) % 2, amp, -amp)
        pcms.append(p)
        starts, ends = cases.synthetic_cues(60 + v, 110.0)
        tv += [v, v]
        cs += [starts, starts + 0.5]
        ce += [ends, ends + 0.5]
    c = _pack(pcms, tv, cs, ce, fr)
    for label in (0.0, 0.3):
        _same(_new(handle, c, label), _compose(handle, c, label), where=label)
    assert au.energy_floor(37) <= 37 * 400 * 400 < au.energy_floor(160) and 37 * 300 * 300 < au.energy_floor(37)
    ref64, ref_off = handle.vad_auditok(c["pcm"], c["pcm_off"], fr, 100, 0.0, chunk_samples=chunk)
    for v, last in ((3, 1.0), (4, 0.0)):
        want = au.auditok_detect_fast(pcms[v][chunk:].tobytes(), 100, fr, 0.0)
        assert len(want) == 36 and want[-2] == 1.0 and want[-1] == last
        assert np.array_equal(ref64[ref_off[v + 1] - 36: ref_off[v + 1]], want)


def test_chunk_restart_changes_the_answer(handle):
    """A token across a chunk boundary: chunked and unchunked detector calls give different signals, so different
    scores; each call equals its own composition."""
    fr, fpw = 16000, 160
    chunk = 700 * fpw
    valid = np.zeros(2000, np.uint8)
    valid[700 - 12: 700 + 13] = 1
    valid[1200:1260] = 1
    pcm = vo.synth_pcm(valid, fpw, seed=3)
    starts = np.array([6.88, 12.0])
    ends = np.array([7.13, 12.6])
    c = _pack([pcm], [0], [starts], [ends], fr)
    chunked = _new(handle, c, chunk=chunk, mos=300)
    whole = _new(handle, c, chunk=0, mos=300)
    _same(chunked, _compose(handle, c, chunk=chunk, mos=300))
    _same(whole, _compose(handle, c, chunk=0, mos=300))
    assert not np.array_equal(chunked["a_s"], whole["a_s"])


@pytest.mark.parametrize("fr,layout", [(8000, None), (22050, None), (44100, "group"), (48000, "group")])
def test_rates(handle, monkeypatch, fr, layout):
    rng = np.random.RandomState(fr)
    videos = [(150.0, [(GRID[int(rng.randint(0, 5))], int(rng.randint(-500, 500)))]),
              (130.0, [(1.0, 200), (25 / 24.0, -300)])]
    c = _corpus(videos, fr=fr, seed0=fr % 97)
    if layout:
        monkeypatch.setenv("B2_VAD_LAYOUT", layout)
    for label in (0.0, 0.3):
        _same(_new(handle, c, label), _compose(handle, c, label), where=(fr, label))


def test_unsupported_rate_and_bad_tokenizer_parameters(handle, corpus):
    from ffsubsync_b200 import _native
    c = corpus
    assert handle.lib.b2_auditok_block_size(99, 100) == 0
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_auditok(c["pcm"], c["pcm_off"], c["track_video"], 99, 100, 0.0, c["cue_start"],
                                   c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, 0)
    assert e.value.status == -6
    for kw in (dict(max_length=0), dict(min_length=0.0), dict(min_length=600.0), dict(max_continuous_silence=500.0)):
        with pytest.raises(_native.NativeError) as e:
            handle.sync_tracks_auditok(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, c["cue_start"],
                                       c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, _chunk(16000), **kw)
        assert e.value.status == -1, kw
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_auditok(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, c["cue_start"],
                                   c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, -1)
    assert e.value.status == -1


@pytest.mark.parametrize("label", [0.0, 0.3, -0.5])
def test_label_selects_the_path(handle, corpus, monkeypatch, label):
    """Under B2_ALIGN_PATH=runs a capture records the run path's epsilon (float64 round-off, tiny) at label 0 and
    the FFT path's tau (fp32 round-off) at any other label, where the reference has further levels."""
    c = corpus
    T, K = len(c["track_video"]), len(GRID)
    monkeypatch.setenv("B2_ALIGN_PATH", "runs")
    with handle.capture_nominations(T * K, 2 * MOS + 64) as cap:
        got = _new(handle, c, label)
    live = cap["win"][:, 1] > 0
    assert live.any()
    bound = cap["stat"][live, 1]
    if label == 0.0:
        assert np.all(bound < 1e-6), bound
    else:
        assert np.all(bound > 1e-4), bound
    monkeypatch.delenv("B2_ALIGN_PATH")
    _same(got, _compose(handle, c, label))


def test_search(handle, corpus):
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    got, want = _new(handle, c, gss=True), _compose(handle, c, gss=True)
    live = (want["status"] & 1) == 0
    assert np.array_equal(got["evals"][live], want["evals"][live])
    assert np.array_equal(got["ratio"][live], want["ratio"][live])
    _same(got, want)
    # label 0.3: the search needs the two-level reference
    with pytest.raises(_native.NativeError) as e:
        _new(handle, c, 0.3, gss=True)
    assert e.value.status == -6 and "0.3" in str(e.value)
    sync = BatchSynchronizer(GRID + [None], non_speech_label=0.3, max_offset_seconds=MOS / 100, vad="auditok")
    r = sync.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                              want_all=True)
    w = _compose(handle, c, 0.3, gss=True)
    for x, key in zip(r, ("bs", "bo", "bk", "a_s", "a_o", "ratio")):
        assert np.array_equal(x, w[key], equal_nan=key == "ratio"), key
    # the front end at label 0 runs the call itself
    sync0 = BatchSynchronizer(GRID + [None], max_offset_seconds=MOS / 100, vad="auditok")
    r0 = sync0.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])
    for x, key in zip(r0, ("bs", "bo", "bk", "ratio")):
        assert np.array_equal(x, got[key], equal_nan=key == "ratio"), key


def test_front_end_methods(handle, corpus):
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    want = _compose(handle, c)
    sync = BatchSynchronizer(GRID, max_offset_seconds=MOS / 100, vad="auditok")
    r = sync.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                              want_all=True)
    _same(dict(zip(("bs", "bo", "bk", "a_s", "a_o"), r)), want)
    pcm = torch.from_numpy(c["pcm"]).cuda()
    o = sync.sync_device_tracks(pcm, c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])
    sync.handle.synchronize()
    _same(dict(bs=o["best_score"].cpu().numpy(), bo=o["best_offset"].cpu().numpy(), bk=o["best_k"].cpu().numpy()),
          want, keys=("bs", "bo", "bk"))
    # pair form: one track per video
    pairs = _corpus([(d, tr[:1]) for d, tr in VIDEOS if tr], seed0=1)
    wp = _compose(handle, pairs)
    hp = sync.sync_host(pairs["pcm"], pairs["pcm_off"], pairs["cue_start"], pairs["cue_end"], pairs["cue_off"])
    _same(dict(zip(("bs", "bo", "bk"), hp)), wp, keys=("bs", "bo", "bk"))
    dp = sync.sync_device(torch.from_numpy(pairs["pcm"]).cuda(), pairs["pcm_off"], pairs["cue_start"],
                          pairs["cue_end"], pairs["cue_off"])
    sync.handle.synchronize()
    assert np.array_equal(dp["best_offset"].cpu().numpy(), wp["bo"])
    assert np.array_equal(dp["best_k"].cpu().numpy(), wp["bk"])
    # candidate sharding on one rank: b2_vad_auditok cast to float32, then the grid
    bs, bo, bk = sync.sync_device_candidate_sharded(torch.from_numpy(pairs["pcm"]).cuda(), pairs["pcm_off"],
                                                    pairs["cue_start"], pairs["cue_end"], pairs["cue_off"])
    torch.cuda.synchronize()
    assert np.array_equal(bo.cpu().numpy(), wp["bo"]) and np.array_equal(bk.cpu().numpy(), wp["bk"])
    assert np.array_equal(bs.cpu().numpy(), wp["bs"])


def test_resident_calls_alternate_detectors(handle, monkeypatch):
    """11 unsynchronised resident calls alternating energy / ZCR and auditok calls over two corpora of different
    sizes equal the same calls made one at a time."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    monkeypatch.setenv("B2_SUBBATCHES", "3")   # pipelined calls: resident calls chain
    rng = np.random.RandomState(8)
    corpora = []
    for seed0, n_tracks in ((100, [2, 1, 4, 0, 3, 1]), (900, [3, 5, 1, 2])):
        vids = [(150.0, [(GRID[int(rng.randint(0, 5))], int(rng.randint(-2000, 2001))) for _ in range(n)])
                for n in n_tracks]
        c = _corpus(vids, seed0=seed0)
        corpora.append((torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"], c["cue_start"],
                        c["cue_end"], c["cue_off"]))
    syncs = [BatchSynchronizer(GRID, max_offset_seconds=MOS / 100),
             BatchSynchronizer(GRID, max_offset_seconds=MOS / 100, vad="auditok"),
             BatchSynchronizer(GRID + [None], max_offset_seconds=MOS / 100, vad="auditok")]
    assert all(s.handle is handle for s in syncs)
    order = [(0, 0), (1, 1), (0, 1), (2, 0), (1, 0), (0, 0), (2, 1), (1, 1), (0, 1), (1, 0), (2, 0)]
    want = {}
    for si, ci in set(order):
        o = syncs[si].sync_device_tracks(*corpora[ci])
        handle.synchronize()
        want[si, ci] = {k: v.clone() for k, v in o.items()}
    outs = [syncs[si].sync_device_tracks(*corpora[ci], inputs_resident=True) for si, ci in order]
    handle.synchronize()
    assert len(outs) == 11
    for (si, ci), got in zip(order, outs):
        for k, v in want[si, ci].items():
            assert torch.equal(got[k], v), (si, ci, k)
