"""GPU tests of b2_sync_tracks_subs: videos whose embedded subtitle stream is their reference (the reference's
``--vad subs_then_*``) next to videos that run the detector, in one batched call (run on an H100).

Two yardsticks:
  * the oracle: oracle.raster_oracle at ratio 1.0 for a subtitle reference, oracle.vad_oracle for an audio one,
    the float64 FFT aligner and MaxScoreAligner's rule per ratio;
  * the composition of public entry points the call replaces - per video b2_rasterize (ratio 1.0, level 1.0) or the
    detector (b2_vad_energy_zcr, or b2_vad_auditok rounded to float32), one copy of the video's signal per track,
    b2_rasterize of the tracks, b2_align_batch, b2_reduce_ratios (and for the search gss_align_batch + the
    reference's combine) - which the call must reproduce bit for bit under every pipeline, path and memory knob."""
import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
MOS = 6000
EVALS = 17
THR = 100000   # constants.DEFAULT_ENERGY_THRESHOLD
DETECTORS = ("energy_zcr", "auditok")


def _chunk(fr=16000):
    return (2 * fr // 100) * 5000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _corpus(videos, fr=16000, seed0=0):
    """videos: list of (duration_s, is_subs, [(ratio, delay in frames) per track]).  A video's master cue list is
    where its audio has speech (10 % flipped, 5 % loud hiss) - or, for a subtitle video, its stream (every 9th cue
    a metadata cue, no PCM); a track is the master list at its own ratio and delay with dropped and jittered cues."""
    fpw = fr // 100
    pcms, tv, cs, ce = [], [], [], []
    is_subs, rcs, rce, rck = [], [], [], []
    for v, (dur, subs, tracks) in enumerate(videos):
        seed = seed0 + 31 * v + 7
        starts, ends = cases.synthetic_cues(seed, max(dur, 60.0))
        n = int(dur * 100)
        is_subs.append(int(subs))
        if subs:
            pcms.append(np.zeros(0, np.int16))
            keep = (np.arange(len(starts)) % 9 != 4).astype(np.uint8)
            rcs.append(starts)
            rce.append(ends)
            rck.append(keep)
        else:
            mask = ro.rasterize(starts, ends, None, 100, 0, 1.0)[0] != 0
            ref = np.zeros(n, dtype=bool)
            ref[: min(n, len(mask))] = mask[:n]
            rng = np.random.RandomState(seed + 1000)
            ref ^= rng.rand(n) < 0.10
            hiss = rng.rand(n) < 0.05
            cls = np.where(ref, 1, np.where(hiss, 2, 0)).astype(np.uint8)
            pcms.append(vo.synth_pcm(cls, fpw, seed=seed))
            rcs.append(np.zeros(0))
            rce.append(np.zeros(0))
            rck.append(np.zeros(0, np.uint8))
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
    ref_off = np.concatenate([[0], np.cumsum([len(c) for c in rcs])]).astype(np.int64)
    return dict(pcm=np.concatenate(pcms) if pcms else np.zeros(0, np.int16), pcm_off=pcm_off,
                track_video=np.array(tv, np.int32), cue_start=np.concatenate(cs) if cs else np.zeros(0),
                cue_end=np.concatenate(ce) if ce else np.zeros(0), cue_off=cue_off,
                is_subs=np.array(is_subs, np.uint8), ref_start=np.concatenate(rcs), ref_end=np.concatenate(rce),
                ref_keep=np.concatenate(rck).astype(np.uint8), ref_off=ref_off, pcms=pcms, cs=cs, ce=ce,
                rcs=rcs, rce=rce, rck=rck, fr=fr)


def _det(det):
    from ffsubsync_b200 import _native
    return _native.B2_DETECTOR_AUDITOK if det == "auditok" else _native.B2_DETECTOR_ENERGY_ZCR


_GIVEN = object()   # _new: take the corpus's own array


def _new(handle, c, det="energy_zcr", label=0.0, grid=GRID, mos=MOS, gss=False, memspace=None, want_all=True,
         pcm=_GIVEN, is_subs=_GIVEN):
    from ffsubsync_b200 import _native
    r = handle.sync_tracks_subs(
        c["pcm"] if pcm is _GIVEN else pcm, c["pcm_off"], c["track_video"], c["fr"], 100, label,
        c["is_subs"] if is_subs is _GIVEN else is_subs, c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"],
        c["cue_start"], c["cue_end"], None, c["cue_off"], grid, 0.0, mos, detector=_det(det), energy_threshold=THR,
        chunk_samples=_chunk(c["fr"]), gss=gss, want_all=want_all, want_evals=gss,
        memspace=_native.B2_HOST if memspace is None else memspace)
    out = dict(bs=r[0], bo=r[1], bk=r[2], a_s=r[3], a_o=r[4])
    if gss:
        out.update(ratio=r[5], evals=r[6].reshape(-1, EVALS))
    return out


def _refs(handle, c, det, label):
    """Each video's reference by public calls: b2_rasterize at ratio 1.0 / level 1.0, or the detector."""
    if det == "auditok":
        d64, d_off = handle.vad_auditok(c["pcm"], c["pcm_off"], c["fr"], 100, label, chunk_samples=_chunk(c["fr"]))
        d = d64.astype(np.float32)
    else:
        d, d_off = handle.vad_energy_zcr(c["pcm"], c["pcm_off"], c["fr"], 100, label, THR)
    s, s_off = handle.rasterize(c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"], [1.0], 1, False, 100, 0.0,
                                levels=[1.0])
    return [s[s_off[v]: s_off[v + 1]] if c["is_subs"][v] else d[d_off[v]: d_off[v + 1]]
            for v in range(len(c["pcm_off"]) - 1)]


def _compose(handle, c, det="energy_zcr", label=0.0, grid=GRID, mos=MOS, gss=False):
    refs = _refs(handle, c, det, label)
    parts = [refs[v] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    t_ref = np.concatenate(parts) if parts else np.zeros(0, np.float32)
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


# subtitle and audio videos with 1, 3, 0, 2 and 5 tracks
VIDEOS = [(240.0, True, [(1.0, 250)]),
          (300.0, False, [(25 / 24.0, -700), (24 / 25.0, 0), (1.0, 1234)]),
          (120.0, True, []),
          (180.0, True, [(23.976 / 24, 300), (1.0, -900)]),
          (210.0, False, [(1.0, 40), (25 / 24.0, -1500), (23.976 / 24, 300), (1.0, -2500), (24 / 23.976, 900)])]


@pytest.fixture(scope="module")
def corpus():
    return _corpus(VIDEOS, seed0=1)


def test_oracle_parity(handle, corpus):
    """A mixed batch at label 0 over the 7-ratio grid: offsets are the oracle's (or tie with it on the exact
    float64 score), scores the exact score of their offset - an integer where the subtitle level is 1."""
    c = corpus
    grid = cases.ratio_grid()
    K = len(grid)
    got = _new(handle, c, grid=grid)
    for t, v in enumerate(c["track_video"]):
        if c["is_subs"][v]:
            ref = ro.rasterize(c["rcs"][v], c["rce"][v], c["rck"][v].astype(bool), 100, 0, 1.0)[0]
        else:
            ref = vo.energy_zcr_detect(c["pcms"][v].tobytes(), 100, 16000, 0.0, THR)
        subs = [ro.rasterize(c["cs"][t], c["ce"][t], None, 100, 0, r)[0] for r in grid]
        cands = [ao.fft_align(ref, sub, MOS) for sub in subs]
        a_s, a_o = got["a_s"].reshape(-1, K)[t], got["a_o"].reshape(-1, K)[t]
        for k, (s, o) in enumerate(cands):
            if a_o[k] != o:   # only a tie may order differently
                assert ao.exact_score(ref, subs[k], int(a_o[k])) == ao.exact_score(ref, subs[k], int(o)), (t, k)
            exact = ao.exact_score(ref, subs[k].astype(np.float32), int(a_o[k]))
            if grid[k] <= 1.0:
                assert a_s[k] == exact and float(a_s[k]).is_integer(), (t, k, a_s[k], exact)
            else:
                assert abs(a_s[k] - exact) <= 1e-12 * max(1.0, abs(exact)), (t, k, a_s[k], exact)
        kept = [k for k, (s, o) in enumerate(cands) if abs(o) <= MOS]
        k_or = max(kept, key=lambda k: cands[k][0]) if kept else -1
        kg, og = int(got["bk"][t]), int(got["bo"][t])
        if k_or < 0:
            assert kg == -1, t
        elif (kg, og) != (k_or, cands[k_or][1]):
            assert ao.exact_score(ref, subs[kg], og) == ao.exact_score(ref, subs[k_or], cands[k_or][1]), (t, kg, k_or)


def test_reference_fixture_through_the_call(handle):
    """The reference's own result (tests/golden/subs_ref.json): its 2 h embedded stream as the reference and an
    input track 25/24 slower and 3.5 s late; MaxScoreAligner over the 7-ratio grid."""
    import json
    import os
    from conftest import ROOT
    with open(os.path.join(ROOT, "tests", "golden", "subs_ref.json")) as fh:
        g = json.load(fh)
    ms = g["subs_ref_maxscore"]
    row = [r for r in g["subs_ref"] if r["name"] == ms["video"]][0]
    ch = row["streams"][row["chosen"]]
    grid = cases.ratio_grid()
    n = len(ch["starts"])
    keep = [int(not ro.is_metadata(t, i == 0 or i + 1 == n)) for i, t in enumerate(ch["contents"])]
    r = handle.sync_tracks_subs(None, [0, 0], [0], 16000, 100, 0.0, [1], ch["starts"], ch["ends"], keep,
                                [0, len(ch["starts"])], ms["in_starts"], ms["in_ends"], None, [0, len(ms["in_starts"])],
                                grid, 0.0, ms["max_offset_seconds"] * 100, want_all=True)
    ref = ro.rasterize(ch["starts"], ch["ends"], np.array(keep, bool), 100, 0, 1.0)[0]
    for k, want in enumerate(ms["per_ratio"]):
        if r[4][k] != want["offset"]:   # only a tie may order differently (the reference's FFT rounding picks one)
            sub64 = ro.rasterize(ms["in_starts"], ms["in_ends"], None, 100, 0, grid[k])[0]
            assert ao.exact_score(ref, sub64, int(r[4][k])) == ao.exact_score(ref, sub64, want["offset"]), k
        if grid[k] <= 1.0:   # level 1: the call's score is the exact count, the reference's its FFT rounding
            assert float(r[3][k]).is_integer() and abs(r[3][k] - want["score"]) <= 1e-9 * abs(want["score"]), k
        else:                # the call holds the level min(1/ratio, 1) as float32: its exact score at that level
            sub = ro.rasterize(ms["in_starts"], ms["in_ends"], None, 100, 0, grid[k])[0].astype(np.float32)
            assert abs(r[3][k] - ao.exact_score(ref, sub, int(r[4][k]))) <= 1e-12 * abs(want["score"]), k
            assert abs(r[3][k] - want["score"]) <= 1e-6 * abs(want["score"]), k
    assert int(r[2][0]) == ms["best"]["index"] and r[1][0] == r[4][ms["best"]["index"]]
    assert r[0][0] == r[3][ms["best"]["index"]]


def test_equals_composition_on_every_path_and_memspace(handle, monkeypatch):
    import torch
    from ffsubsync_b200 import _native
    # 80 videos of 90 s, a third of them subtitle references, 100 tracks: the partitioned pipeline runs by default
    rng = np.random.RandomState(2)
    videos = [(90.0 + 3 * (v % 5), v % 3 == 1, [(GRID[int(rng.randint(0, 5))], int(rng.randint(-800, 800)))
                                                for _ in range([1, 2, 0, 2][v % 4])]) for v in range(80)]
    c = _corpus(videos, seed0=11)
    T, K = len(c["track_video"]), len(GRID)
    assert T >= 96 and 0 < c["is_subs"].sum() < 80
    dev = torch.device("cuda", handle.device)
    pcm = torch.from_numpy(c["pcm"]).to(dev)
    for det in DETECTORS:
        for label in (0.0, 0.3):
            want = _compose(handle, c, det, label)
            _same(_new(handle, c, det, label), want, where=("default", det, label))
            _same(_new(handle, c, det, label, want_all=False), want, keys=("bs", "bo", "bk"),
                  where=("winner-only", det, label))
            for env in ({"B2_SUBBATCHES": "1"}, {"B2_SUBBATCHES": "3", "B2_VAD_SMS": "8"},
                        {"B2_ALIGN_PATH": "tiled"}, {"B2_ALIGN_PATH": "runs"}, {"B2_ALIGN_PATH": "big"},
                        {"B2_FUSED_RASTER": "0"}):
                with monkeypatch.context() as m:
                    for k, v in env.items():
                        m.setenv(k, v)
                    _same(_new(handle, c, det, label), want, where=(env, det, label))
                    _same(_new(handle, c, det, label, want_all=False), want, keys=("bs", "bo", "bk"),
                          where=(env, "winner-only", det, label))
            for ms in (_native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
                bs = torch.full((T,), -7, dtype=torch.float64, device=dev)
                bo = torch.full((T,), -7, dtype=torch.int32, device=dev)
                bk = torch.full((T,), -7, dtype=torch.int32, device=dev)
                a_s = torch.zeros(T * K, dtype=torch.float64, device=dev)
                a_o = torch.zeros(T * K, dtype=torch.int32, device=dev)
                torch.cuda.synchronize(dev)
                handle.sync_tracks_subs(pcm.data_ptr(), c["pcm_off"], c["track_video"], 16000, 100, label,
                                        c["is_subs"], c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"],
                                        c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS,
                                        detector=_det(det), energy_threshold=THR, chunk_samples=_chunk(),
                                        best_score=bs.data_ptr(), best_offset=bo.data_ptr(), best_k=bk.data_ptr(),
                                        all_score=a_s.data_ptr(), all_offset=a_o.data_ptr(), memspace=ms)
                handle.synchronize()
                got = dict(bs=bs.cpu().numpy(), bo=bo.cpu().numpy(), bk=bk.cpu().numpy(), a_s=a_s.cpu().numpy(),
                           a_o=a_o.cpu().numpy())
                _same(got, want, where=(ms, det, label))
    # FFTAligner's whole window (max_offset_seconds=None): the large-window path
    for det in DETECTORS:
        _same(_new(handle, c, det, 0.0, mos=None), _compose(handle, c, det, 0.0, mos=None), where=("none", det))


def test_all_audio_calls_equal_the_detector_calls(handle):
    """Without subtitle videos the call is b2_sync_tracks / b2_sync_tracks_gss / b2_sync_tracks_auditok."""
    audio = _corpus([v for v in VIDEOS if not v[1]], seed0=5)
    for is_subs in (None, np.zeros(len(audio["pcm_off"]) - 1, np.uint8)):
        for label in (0.0, 0.3):
            e = handle.sync_tracks(audio["pcm"], audio["pcm_off"], audio["track_video"], 16000, 100, label, THR, -1,
                                   -1, audio["cue_start"], audio["cue_end"], None, audio["cue_off"], GRID, 0.0, MOS,
                                   want_all=True)
            _same(_new(handle, audio, "energy_zcr", label, is_subs=is_subs), dict(zip(("bs", "bo", "bk", "a_s", "a_o"), e)))
            a = handle.sync_tracks_auditok(audio["pcm"], audio["pcm_off"], audio["track_video"], 16000, 100, label,
                                           audio["cue_start"], audio["cue_end"], None, audio["cue_off"], GRID, 0.0,
                                           MOS, _chunk(), want_all=True)
            _same(_new(handle, audio, "auditok", label, is_subs=is_subs), dict(zip(("bs", "bo", "bk", "a_s", "a_o"), a)))
        g = handle.sync_tracks_gss(audio["pcm"], audio["pcm_off"], audio["track_video"], 16000, 100, 0.0, THR, -1, -1,
                                   audio["cue_start"], audio["cue_end"], None, audio["cue_off"], GRID, 0.0, MOS,
                                   want_all=True, want_evals=True)
        got = _new(handle, audio, "energy_zcr", 0.0, gss=True, is_subs=is_subs)
        _same(got, dict(zip(("bs", "bo", "bk", "a_s", "a_o"), g)))
        assert np.array_equal(got["ratio"], g[5], equal_nan=True)
        assert np.array_equal(got["evals"].ravel(), g[6], equal_nan=True)


def test_all_subtitle_calls(handle, monkeypatch):
    """Every video a subtitle reference: no PCM (pcm NULL, all pcm_off equal), with and without the pipeline."""
    import torch
    from ffsubsync_b200 import _native
    rng = np.random.RandomState(4)
    videos = [(300.0, True, [(GRID[int(rng.randint(0, 5))], int(rng.randint(-800, 800)))
                             for _ in range([1, 2, 0, 2][v % 4])]) for v in range(80)]
    c = _corpus(videos, seed0=21)
    assert len(c["track_video"]) >= 96 and c["pcm_off"][-1] == 0
    c["pcm_off"] = np.full_like(c["pcm_off"], 8)   # any equal offsets: no video has samples
    for det in DETECTORS:
        for label in (0.0, 0.3):
            want = _compose(handle, dict(c, pcm_off=np.zeros_like(c["pcm_off"])), det, label)
            _same(_new(handle, c, det, label, pcm=None), want, where=(det, label))
            with monkeypatch.context() as m:
                m.setenv("B2_SUBBATCHES", "1")
                _same(_new(handle, c, det, label, pcm=None), want, where=("one sub-batch", det, label))
            T, K = len(c["track_video"]), len(GRID)
            dev = torch.device("cuda", handle.device)
            o = {k: torch.full((T,), -7, dtype=d, device=dev) for k, d in
                 (("bs", torch.float64), ("bo", torch.int32), ("bk", torch.int32))}
            handle.sync_tracks_subs(None, c["pcm_off"], c["track_video"], 16000, 100, label, c["is_subs"],
                                    c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"], c["cue_start"],
                                    c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, detector=_det(det),
                                    energy_threshold=THR, chunk_samples=_chunk(), best_score=o["bs"].data_ptr(),
                                    best_offset=o["bo"].data_ptr(), best_k=o["bk"].data_ptr(),
                                    memspace=_native.B2_DEVICE_RESIDENT)
            handle.synchronize()
            _same({k: v.cpu().numpy() for k, v in o.items()}, want, keys=("bs", "bo", "bk"), where=("dev", det))
        # the search at a non-zero label: every reference is a subtitle stream, so the run path takes it
        g = _new(handle, c, det, 0.3, gss=True, pcm=None)
        w = _compose(handle, dict(c, pcm_off=np.zeros_like(c["pcm_off"])), det, 0.3, gss=True)
        _same(g, w, where=("search", det))
        assert np.array_equal(g["ratio"], w["ratio"], equal_nan=True)


@pytest.mark.parametrize("det", DETECTORS)
def test_label_selects_the_path(handle, corpus, monkeypatch, det):
    """Under B2_ALIGN_PATH=runs a capture records the run path's epsilon (float64 round-off, tiny) or the FFT path's
    tau (fp32 round-off).  At label 0.5 a mixed call has three levels and takes the FFT path; an all-subtitle call
    has two (1 and 0) and takes the run path, whose every captured score of a job at subtitle level 1 is the exact
    integer count of its offset."""
    c = corpus
    subs_only = _corpus([v for v in VIDEOS if v[1]], seed0=1)
    monkeypatch.setenv("B2_ALIGN_PATH", "runs")
    stride = 2 * MOS + 64
    for cc, run_path in ((c, False), (subs_only, True)):
        T, K = len(cc["track_video"]), len(GRID)
        with handle.capture_nominations(T * K, stride) as cap:
            got = _new(handle, cc, det, 0.5)
        live = cap["win"][:, 1] > 0
        assert live.any()
        bound = cap["stat"][live, 1]
        if run_path:
            assert np.all(bound < 1e-6), bound
        else:
            assert np.all(bound > 1e-4), bound
        with monkeypatch.context() as m:
            m.delenv("B2_ALIGN_PATH")
            _same(got, _compose(handle, cc, det, 0.5))
        if not run_path:
            continue
        refs = _refs(handle, cc, det, 0.5)
        for t, v in enumerate(cc["track_video"]):
            for k, r in enumerate(GRID):
                j = t * K + k
                w0, n = (int(x) for x in cap["win"][j])
                if r > 1.0 or n == 0:
                    continue
                sub = ro.rasterize(cc["cs"][t], cc["ce"][t], None, 100, 0, r)[0]
                exact = ao.exact_scores_window(refs[v], sub, w0, w0 + n - 1)
                f = cap["scores"][j, :n]
                assert np.array_equal(f.astype(np.int64), np.asarray(exact).astype(np.int64)), (t, k)
                assert np.all(np.asarray(exact) == np.round(np.asarray(exact))), (t, k)


@pytest.mark.parametrize("det", DETECTORS)
def test_search(handle, corpus, det):
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    # label 0: one two-level reference for both kinds, the rounds run on the device
    got, want = _new(handle, c, det, gss=True), _compose(handle, c, det, gss=True)
    live = (want["status"] & 1) == 0
    assert np.array_equal(got["evals"][live], want["evals"][live])
    assert np.array_equal(got["ratio"][live], want["ratio"][live])
    _same(got, want)
    # label 0.3 with subtitle and audio videos mixed: three levels, the call declines and names why
    with pytest.raises(_native.NativeError) as e:
        _new(handle, c, det, 0.3, gss=True)
    assert e.value.status == -6 and "0.3" in str(e.value)
    # ... and the front end composes the public steps instead
    sync = BatchSynchronizer(GRID + [None], non_speech_label=0.3, max_offset_seconds=MOS / 100,
                             vad="subs_then_" + det, energy_threshold=THR)
    streams = dict(ref_cue_start=c["ref_start"], ref_cue_end=c["ref_end"], ref_cue_keep=c["ref_keep"],
                   ref_cue_off=np.concatenate([[0], c["ref_off"][1:][c["is_subs"] == 1]]),
                   ref_stream_video=np.flatnonzero(c["is_subs"]))
    r = sync.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                              want_all=True, **streams)
    w = _compose(handle, c, det, 0.3, gss=True)
    for x, key in zip(r, ("bs", "bo", "bk", "a_s", "a_o", "ratio")):
        assert np.array_equal(x, w[key], equal_nan=key == "ratio"), key


def _streams_of(c):
    """The corpus's subtitle references as one stream per subtitle video (front-end keyword arguments)."""
    sel = c["is_subs"] == 1
    return dict(ref_cue_start=c["ref_start"], ref_cue_end=c["ref_end"], ref_cue_keep=c["ref_keep"],
                ref_cue_off=np.concatenate([[0], c["ref_off"][1:][sel]]), ref_stream_video=np.flatnonzero(sel))


@pytest.mark.parametrize("det", DETECTORS)
def test_front_end_methods(handle, corpus, det):
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    want = _compose(handle, c, det)
    sync = BatchSynchronizer(GRID, max_offset_seconds=MOS / 100, vad="subs_then_" + det, energy_threshold=THR)
    st = _streams_of(c)
    r = sync.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                              want_all=True, **st)
    _same(dict(zip(("bs", "bo", "bk", "a_s", "a_o"), r)), want)
    pcm = torch.from_numpy(c["pcm"]).cuda()
    o = sync.sync_device_tracks(pcm, c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"], **st)
    sync.handle.synchronize()
    _same(dict(bs=o["best_score"].cpu().numpy(), bo=o["best_offset"].cpu().numpy(), bk=o["best_k"].cpu().numpy()),
          want, keys=("bs", "bo", "bk"))
    # a second, shorter stream per subtitle video never wins; a stream ending later would
    extra = dict(st)
    sv = st["ref_stream_video"]
    extra["ref_stream_video"] = np.repeat(sv, 2)
    offs, s_all, e_all, k_all = [0], [], [], []
    for i, v in enumerate(sv):
        a, b = c["ref_off"][v], c["ref_off"][v + 1]
        s_all += [c["ref_start"][a:b], c["ref_start"][a:b][:3]]
        e_all += [c["ref_end"][a:b], c["ref_end"][a:b][:3]]
        k_all += [c["ref_keep"][a:b], c["ref_keep"][a:b][:3]]
        offs += [offs[-1] + b - a, offs[-1] + b - a + min(3, b - a)]
    extra.update(ref_cue_start=np.concatenate(s_all), ref_cue_end=np.concatenate(e_all),
                 ref_cue_keep=np.concatenate(k_all), ref_cue_off=np.array(offs))
    r2 = sync.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                               want_all=True, **extra)
    _same(dict(zip(("bs", "bo", "bk", "a_s", "a_o"), r2)), want)
    # pair form: one track per video
    pairs = _corpus([(d, s, tr[:1]) for d, s, tr in VIDEOS if tr], seed0=1)
    wp = _compose(handle, pairs, det)
    hp = sync.sync_host(pairs["pcm"], pairs["pcm_off"], pairs["cue_start"], pairs["cue_end"], pairs["cue_off"],
                        **_streams_of(pairs))
    _same(dict(zip(("bs", "bo", "bk"), hp)), wp, keys=("bs", "bo", "bk"))
    dp = sync.sync_device(torch.from_numpy(pairs["pcm"]).cuda(), pairs["pcm_off"], pairs["cue_start"],
                          pairs["cue_end"], pairs["cue_off"], **_streams_of(pairs))
    sync.handle.synchronize()
    assert np.array_equal(dp["best_offset"].cpu().numpy(), wp["bo"]) and np.array_equal(dp["best_k"].cpu().numpy(),
                                                                                         wp["bk"])
    # without streams: the detector alone
    audio = _corpus([v for v in VIDEOS if not v[1]], seed0=5)
    plain = BatchSynchronizer(GRID, max_offset_seconds=MOS / 100, vad=det, energy_threshold=THR)
    args = (audio["pcm"], audio["pcm_off"], audio["track_video"], audio["cue_start"], audio["cue_end"],
            audio["cue_off"])
    for a, b in zip(sync.sync_host_tracks(*args, want_all=True), plain.sync_host_tracks(*args, want_all=True)):
        assert np.array_equal(a, b)
    with pytest.raises(ValueError):
        sync.sync_device_candidate_sharded(pcm, c["pcm_off"], c["cue_start"], c["cue_end"], c["cue_off"])


def test_resident_calls_alternate_with_the_detector_calls(handle, monkeypatch):
    """12 unsynchronised resident calls alternating b2_sync_tracks, b2_sync_tracks_auditok and b2_sync_tracks_subs
    (both detectors, grid and search) over two corpora equal the same calls made one at a time."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    monkeypatch.setenv("B2_SUBBATCHES", "3")   # pipelined calls: resident calls chain
    rng = np.random.RandomState(8)
    corpora = []
    for seed0, n_tracks in ((100, [2, 1, 4, 0, 3, 1]), (900, [3, 5, 1, 2])):
        vids = [(150.0, i % 2 == 0, [(GRID[int(rng.randint(0, 5))], int(rng.randint(-2000, 2001)))
                                     for _ in range(n)]) for i, n in enumerate(n_tracks)]
        c = _corpus(vids, seed0=seed0)
        corpora.append(((torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"], c["cue_start"],
                         c["cue_end"], c["cue_off"]), _streams_of(c)))
    kw = dict(max_offset_seconds=MOS / 100, energy_threshold=THR)
    syncs = [(BatchSynchronizer(GRID, **kw), False), (BatchSynchronizer(GRID, vad="auditok", max_offset_seconds=MOS / 100), False),
             (BatchSynchronizer(GRID, vad="subs_then_energy_zcr", **kw), True),
             (BatchSynchronizer(GRID, vad="subs_then_auditok", max_offset_seconds=MOS / 100), True),
             (BatchSynchronizer(GRID + [None], vad="subs_then_energy_zcr", **kw), True)]
    assert all(s.handle is handle for s, _ in syncs)
    order = [(0, 0), (2, 1), (1, 1), (3, 0), (4, 1), (0, 1), (2, 0), (3, 1), (1, 0), (4, 0), (2, 1), (0, 0)]

    def call(si, ci, resident):
        s, with_streams = syncs[si]
        args, streams = corpora[ci]
        return s.sync_device_tracks(*args, inputs_resident=resident, **(streams if with_streams else {}))

    want = {}
    for si, ci in set(order):
        o = call(si, ci, False)
        handle.synchronize()
        want[si, ci] = {k: v.clone() for k, v in o.items()}
    outs = [call(si, ci, True) for si, ci in order]
    handle.synchronize()
    for (si, ci), got in zip(order, outs):
        for k, v in want[si, ci].items():
            assert torch.equal(got[k], v), (si, ci, k)


def test_bad_arguments(handle, corpus):
    from ffsubsync_b200 import _native
    c = corpus

    def call(**over):
        a = dict(c)
        a.update(over)
        return handle.sync_tracks_subs(a["pcm"], a["pcm_off"], a["track_video"], 16000, 100, 0.0, a["is_subs"],
                                       a["ref_start"], a["ref_end"], a["ref_keep"], a["ref_off"], a["cue_start"],
                                       a["cue_end"], None, a["cue_off"], GRID, 0.0, MOS, energy_threshold=THR)

    call()
    # a subtitle video with samples
    v = int(np.flatnonzero(c["is_subs"])[0])
    is_subs = c["is_subs"].copy()
    is_subs[1] = 1
    assert c["is_subs"][1] == 0 and c["pcm_off"][2] > c["pcm_off"][1]
    with pytest.raises(_native.NativeError) as e:
        call(is_subs=is_subs)
    assert e.value.status == -1 and "non-empty PCM range" in str(e.value)
    # ref_cue_off not monotone
    bad_off = c["ref_off"].copy()
    bad_off[v + 1] = bad_off[v] - 1
    with pytest.raises(_native.NativeError) as e:
        call(ref_off=bad_off)
    assert e.value.status == -1 and "not monotone" in str(e.value)
    # a non-finite reference cue time: the message names its index
    for bad in (np.nan, np.inf, 1e300):
        rs = c["ref_start"].copy()
        i = int(c["ref_off"][v]) + 5
        rs[i] = bad
        with pytest.raises(_native.NativeError) as e:
            call(ref_start=rs)
        assert e.value.status == -1 and "reference cue start" in str(e.value) and "index %d" % i in str(e.value)
    re_ = c["ref_end"].copy()
    re_[int(c["ref_off"][v])] = np.nan
    with pytest.raises(_native.NativeError) as e:
        call(ref_end=re_)
    assert e.value.status == -1 and "index %d" % int(c["ref_off"][v]) in str(e.value)
    # cues for a video without a subtitle reference
    with pytest.raises(_native.NativeError) as e:
        call(is_subs=np.where(np.arange(len(c["is_subs"])) == v, 0, c["is_subs"]).astype(np.uint8))
    assert e.value.status == -1
    call()   # the handle still works
