"""GPU tests of serialized speech signals as references (b2_sync_tracks_sig; the reference's ``ffs ref.npz -i in.srt``),
alone and next to audio, text-stream and PGS videos in one batched call (run on an H100).

Yardsticks: the fixture recorded from the reference (tests/golden/signal_ref.json), the float64 rule
(oracle/sig_oracle.py), and the composition of public entry points the call replaces - per video the rule applied to
its stored values or what b2_sync_tracks_pgs uses, one copy per track, b2_rasterize of the tracks, b2_align_batch,
b2_reduce_ratios (and for the search gss_align_batch + the reference's combine) - which the call must reproduce bit
for bit, except where the composition's aligner reports B2_ALIGN_CAND_OVERFLOW (the call's score is then at least as
high)."""
import json
import os

import numpy as np
import pytest

import cases
from conftest import ROOT
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import sig_oracle as so
from test_gpu_pgs_ref import _pgs_corpus, _refs as _pgs_refs, _same
from test_gpu_subs_ref import _chunk, _det

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
MOS = 6000
THR = 100000
# stored values below 1.0 that the rule sends to the label, the rounding edge among them
LOW = np.array([0.0, 1.0 - 2.0 ** -53, 1.0 - 2.0 ** -25, -np.inf, 0.3, -0.5, 0.999999])


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "signal_ref.json")) as fh:
        return json.load(fh)


def _sig_corpus(videos, seed0=0):
    """videos: (duration_s, kind in "audio" / "text" / "pgs" / "sig", tracks).  A signal video stores its master cue
    list's frames: 1.0 on the cues, elsewhere runs of LOW's values; it has no PCM and no other reference."""
    c = _pgs_corpus([(d, "text" if k == "sig" else k, t) for d, k, t in videos], seed0=seed0)
    V = len(videos)
    is_sig = np.array([k == "sig" for _, k, _ in videos], np.uint8)
    xs = []
    for v in range(V):
        if not is_sig[v]:
            xs.append(np.zeros(0))
            continue
        a, b = c["ref_off"][v], c["ref_off"][v + 1]
        mask = ro.rasterize(c["ref_start"][a:b], c["ref_end"][a:b], None, 100, 0, 1.0)[0] != 0
        rng = np.random.RandomState(seed0 + 11 * v)
        low = LOW[np.repeat(rng.randint(0, len(LOW), len(mask) // 37 + 1), 37)[: len(mask)]]
        xs.append(np.where(mask, 1.0, low))
    keep_v = (c["is_subs"] != 0) & (is_sig == 0)
    pick = np.concatenate([np.arange(c["ref_off"][v], c["ref_off"][v + 1]) for v in range(V) if keep_v[v]]
                          + [np.zeros(0, np.int64)]).astype(np.int64)
    c["ref_start"], c["ref_end"], c["ref_keep"] = c["ref_start"][pick], c["ref_end"][pick], c["ref_keep"][pick]
    c["ref_off"] = np.concatenate([[0], np.cumsum(np.where(keep_v, np.diff(c["ref_off"]), 0))]).astype(np.int64)
    c["is_subs"] = keep_v.astype(np.uint8)
    c["is_sig"] = is_sig
    c["x"] = np.concatenate(xs) if xs else np.zeros(0)
    c["sig_off"] = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
    return c


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _new(handle, c, det="energy_zcr", label=0.0, grid=GRID, mos=MOS, gss=False, memspace=None, want_all=True,
         outs=None, x=None):
    """b2_sync_tracks_sig on corpus c; x: the values' device pointer for the device memspaces."""
    from ffsubsync_b200 import _native
    other = {}
    if c["is_subs"].any():
        other.update(ref_is_subs=c["is_subs"], ref_cue_start_s=c["ref_start"], ref_cue_end_s=c["ref_end"],
                     ref_cue_keep=c["ref_keep"], ref_cue_off=c["ref_off"])
    if c["is_pgs"].any():
        other.update(ref_is_pgs=c["is_pgs"], pgs_start_s=c["pgs_start"], pgs_end_s=c["pgs_end"], pgs_off=c["pgs_off"])
    host = memspace in (None, _native.B2_HOST)
    r = handle.sync_tracks_sig(
        c["pcm"] if host else c.get("pcm_dev"), c["pcm_off"], c["track_video"], c["fr"], 100, label, c["is_sig"],
        c["x"] if host else x, c["sig_off"], c["cue_start"], c["cue_end"], None, c["cue_off"], grid, 0.0, mos,
        detector=_det(det), energy_threshold=THR, chunk_samples=_chunk(c["fr"]), gss=gss, want_all=want_all,
        want_evals=False, memspace=_native.B2_HOST if memspace is None else memspace, **other, **(outs or {}))
    out = dict(bs=r[0], bo=r[1], bk=r[2], a_s=r[3], a_o=r[4])
    if gss:
        out["ratio"] = r[5]
    return out


def _compose(handle, c, det="energy_zcr", label=0.0, grid=GRID, mos=MOS, gss=False):
    refs = _pgs_refs(handle, c, det, label)
    for v in np.flatnonzero(c["is_sig"]):
        refs[v] = so.frames(c["x"][c["sig_off"][v]: c["sig_off"][v + 1]], label)
    parts = [refs[v] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    t_ref = np.concatenate(parts).astype(np.float32) if parts else np.zeros(0, np.float32)
    T, K = len(c["track_video"]), len(grid)
    sub, sub_off = handle.rasterize(c["cue_start"], c["cue_end"], None, c["cue_off"], grid, K, False, 100, 0.0)
    score, offset, status = handle.align_batch(t_ref, t_off, sub, sub_off, T, K, mos)
    bs, bo, bk = handle.reduce_ratios(score, offset, status, T, K, mos)
    out = dict(bs=bs, bo=bo, bk=bk, a_s=score, a_o=offset, status=status)
    if gss:
        from ffsubsync_b200.gss_batch import combine_gss, gss_align_batch
        g = gss_align_batch(t_ref, t_off, c["cue_start"], c["cue_end"], c["cue_off"], None, mos, 100, 0.0,
                            handle=handle)
        bs, bo, bk, r, a_s, a_o = combine_gss(bs, bo, bk, g, K, mos, score, offset)
        st = np.concatenate([status.reshape(T, K), np.zeros((T, 1), np.int32)], axis=1).ravel()
        out = dict(bs=bs, bo=bo, bk=bk, a_s=a_s, a_o=a_o, ratio=r, status=st)
    return out


def _device_call(handle, c, memspace, det="energy_zcr", label=0.0, gss=False, K=len(GRID)):
    """The call on device memory (outputs pre-filled with -7); returns host copies."""
    import torch
    T = len(c["track_video"])
    dev = torch.device("cuda", handle.device)
    cols = K + 1 if gss else K
    o = dict(best_score=torch.full((T,), -7, dtype=torch.float64, device=dev),
             best_offset=torch.full((T,), -7, dtype=torch.int32, device=dev),
             best_k=torch.full((T,), -7, dtype=torch.int32, device=dev),
             all_score=torch.zeros(T * cols, dtype=torch.float64, device=dev),
             all_offset=torch.zeros(T * cols, dtype=torch.int32, device=dev))
    if gss:
        o["gss_ratio"] = torch.full((T,), -7, dtype=torch.float64, device=dev)
    xd = _dev(c["x"])
    pcm = torch.from_numpy(c["pcm"]).to(dev) if len(c["pcm"]) else None
    c = dict(c, pcm_dev=pcm.data_ptr() if pcm is not None else None)
    torch.cuda.synchronize(dev)
    _new(handle, c, det, label, gss=gss, memspace=memspace, outs={k: v.data_ptr() for k, v in o.items()},
         x=xd.data_ptr() if xd.numel() else None)
    handle.synchronize()
    got = dict(bs=o["best_score"].cpu().numpy(), bo=o["best_offset"].cpu().numpy(), bk=o["best_k"].cpu().numpy(),
               a_s=o["all_score"].cpu().numpy(), a_o=o["all_offset"].cpu().numpy())
    if gss:
        got["ratio"] = o["gss_ratio"].cpu().numpy()
    return got


# ---------------------------------------------------------------- the reference's own results

def test_fixture_frames_through_the_capture(handle, golden):
    """Every fixture signal, at every label, is the reference's DeserializeSpeechTransformer output rounded once to
    float32 - through the oracle and through the call's reference buffer."""
    for label in (0.0, 0.5, -0.5):
        sel = [r for r in golden["signals"] if r["label"] == label]
        xs = [so.stored_signal(golden, r["name"]) for r in sel]
        for r, x in zip(sel, xs):
            want = so.from_runs(r["out_levels"], r["out_starts"], r["length"])
            assert np.array_equal(so.deserialize(x, label), want), (r["name"], label)
        off = np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)
        V = len(xs)
        for packed_env in ("1", "0"):
            with pytest.MonkeyPatch.context() as m:
                m.setenv("B2_REF_PACKED", packed_env)
                with handle.capture_reference(int(off[-1]) + 64, V) as cap:
                    handle.sync_tracks_sig(None, np.zeros(V + 1, np.int64), np.arange(V, dtype=np.int32), 16000, 100,
                                           label, np.ones(V, np.uint8), np.concatenate(xs), off, [1.0] * V,
                                           [2.0] * V, None, np.arange(V + 1), GRID, 0.0, MOS)
            assert np.array_equal(cap["ref_off"], off)
            if packed_env == "0":   # floats everywhere; packed words where the run path runs otherwise
                assert not cap["packed"].any()
            for v, (r, x) in enumerate(zip(sel, xs)):
                f = so.frames(x, label)
                got = cap["ref"][off[v]: off[v + 1]]
                if cap["packed"][v]:
                    W = (len(f) + 31) // 32
                    assert np.array_equal(got[:W].view(np.uint32), so.packed_words(f)), (r["name"], label)
                else:
                    assert np.array_equal(got, f), (r["name"], label)


def test_reference_grid_and_search_through_the_call(handle, golden):
    """The reference's MaxScoreAligner over the 7-ratio grid and with --gss, against its 2 h stored signal."""
    ms, gs = golden["maxscore"], golden["gss"]
    x = so.stored_signal(golden, "two_hours")
    ref = so.deserialize(x, 0.0)
    grid = cases.ratio_grid()
    n_in = len(ms["in_starts"])
    for gss in (False, True):
        r = handle.sync_tracks_sig(None, [0, 0], [0], 16000, 100, 0.0, [1], x, [0, len(x)], ms["in_starts"],
                                   ms["in_ends"], None, [0, n_in], grid, 0.0, ms["max_offset_seconds"] * 100, gss=gss,
                                   want_all=True)
        for k, want in enumerate(ms["per_ratio"]):
            if r[4][k] != want["offset"]:   # only a tie may order differently
                sub64 = ro.rasterize(ms["in_starts"], ms["in_ends"], None, 100, 0, grid[k])[0]
                assert ao.exact_score(ref, sub64, int(r[4][k])) == ao.exact_score(ref, sub64, want["offset"]), k
            tol = 1e-9 if grid[k] <= 1.0 else 1e-6
            assert abs(r[3][k] - want["score"]) <= tol * abs(want["score"]), (k, r[3][k], want["score"])
        best = gs["best"] if gss else ms["best"]
        assert int(r[2][0]) == best["index"] and r[1][0] == best["offset"], (gss, r[2][0], r[1][0])
        if gss:
            want = gs["per_candidate"][-1]
            assert r[4][-1] == want["offset"] and abs(r[3][-1] - want["score"]) <= 1e-6 * abs(want["score"])
            assert abs(r[5][0] - gs["gss_ratio"]) <= 1e-4


# ---------------------------------------------------------------- the call against the composition

@pytest.mark.parametrize("corpus_kind,det", [("all_sig", "energy_zcr"), ("all_sig", "auditok"),
                                             ("sig_audio", "energy_zcr"), ("sig_audio", "auditok"),
                                             ("sig_text_pgs_audio", "energy_zcr"),
                                             ("sig_text_pgs_audio", "auditok")])
def test_equals_composition_on_every_path_and_memspace(handle, monkeypatch, corpus_kind, det):
    from ffsubsync_b200 import _native
    rng = np.random.RandomState(3)
    kinds = {"all_sig": ["sig"], "sig_audio": ["sig", "audio"],
             "sig_text_pgs_audio": ["sig", "text", "pgs", "audio"]}[corpus_kind]
    videos = [(90.0 + 3 * (v % 5) + 0.07 * v, kinds[v % len(kinds)],
               [(GRID[int(rng.randint(0, 5))], int(rng.randint(-800, 800))) for _ in range([1, 2, 0, 3][v % 4])])
              for v in range(80)]
    c = _sig_corpus(videos, seed0=17)
    K = len(GRID)
    # labels at which the call is two-level: all of them for signals alone and with energy audio
    labels = (0.0, 0.3, -0.5)
    for label in labels:
        want = _compose(handle, c, det, label)
        _same(_new(handle, c, det, label), want, K, where=("default", label))
        _same(_new(handle, c, det, label, want_all=False), want, K, keys=("bs", "bo", "bk"), where=("winner", label))
        for env in ({"B2_SUBBATCHES": "1"}, {"B2_SUBBATCHES": "2", "B2_VAD_SMS": "8"},
                    {"B2_SUBBATCHES": "3", "B2_VAD_SMS": "8"}, {"B2_SUBBATCHES": "4", "B2_VAD_SMS": "8"},
                    {"B2_REF_PACKED": "0"}, {"B2_ALIGN_PATH": "tiled"}, {"B2_ALIGN_PATH": "runs"},
                    {"B2_FUSED_RASTER": "0"}):
            with monkeypatch.context() as m:
                for k, v in env.items():
                    m.setenv(k, v)
                _same(_new(handle, c, det, label), want, K, where=(env, label))
        for ms in (_native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
            _same(_device_call(handle, c, ms, det, label), want, K, where=(ms, label))
    # --gss on the device-driven rounds, where the call is two-level: signals alone, or with energy audio, at any
    # label; with text / PGS references or auditok audio only at label 0
    three_levels = corpus_kind != "all_sig" and (det == "auditok" or "text" in kinds)
    for label in ((0.0,) if three_levels else (0.0, 0.3)):
        want = _compose(handle, c, det, label, gss=True)
        for memspace in (None, _native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
            got = (_new(handle, c, det, label, gss=True) if memspace is None
                   else _device_call(handle, c, memspace, det, label, gss=True))
            _same(got, want, K + 1, where=("gss", label, memspace))
            assert np.array_equal(got["ratio"], want["ratio"], equal_nan=True)
    if three_levels:
        with pytest.raises(_native.NativeError) as e:   # three levels with the search
            _new(handle, c, det, 0.3, gss=True)
        assert e.value.status == -6


def test_packed_where_the_run_path_runs(handle):
    """The premise of the packed comparisons: an all-signal call on the run path is packed with either detector,
    a sub-batch with a text reference keeps floats."""
    c = _sig_corpus([(60.0, "sig", [(1.0, 30)]), (61.0, "sig", [(1.0, -30)]), (62.0, "text", [(1.0, 10)])], seed0=3)
    for det in ("energy_zcr", "auditok"):
        with handle.capture_reference(int(c["sig_off"][-1]) + 10000, 3) as cap:
            _new(handle, c, det, 0.0)
        assert cap["packed"].tolist() == [0, 0, 0], det   # one sub-batch, holding the text video
        c2 = _sig_corpus([(60.0, "sig", [(1.0, 30)]), (61.0, "sig", [(1.0, -30)])], seed0=3)
        with handle.capture_reference(int(c2["sig_off"][-1]) + 64, 2) as cap:
            _new(handle, c2, det, 0.3)
        assert cap["packed"].tolist() == [1, 1], det


def test_round_trip_of_an_energy_call(handle, monkeypatch):
    """The float reference an energy-VAD PCM call builds, fed back as stored signals, gives every output of that
    call bit for bit, at labels 0, 0.3 and -0.5."""
    c = _sig_corpus([(100.0 + 7 * v, "audio", [(GRID[v % 5], 100 * v - 300)] * (1 + v % 3)) for v in range(12)],
                    seed0=29)
    V = len(c["pcm_off"]) - 1
    for label in (0.0, 0.3, -0.5):
        with monkeypatch.context() as m:
            m.setenv("B2_REF_PACKED", "0")
            with handle.capture_reference(4_000_000, V) as cap:
                handle.sync_tracks(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, label, THR, -1, -1,
                                   c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS)
        ref_off = cap["ref_off"]
        x = cap["ref"][: ref_off[-1]].astype(np.float64)
        want = handle.sync_tracks(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, label, THR, -1, -1,
                                  c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, want_all=True)
        got = handle.sync_tracks_sig(None, np.zeros(V + 1, np.int64), c["track_video"], 16000, 100, label,
                                     np.ones(V, np.uint8), x, ref_off, c["cue_start"], c["cue_end"], None, c["cue_off"],
                                     GRID, 0.0, MOS, energy_threshold=THR, want_all=True)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), label


def test_capture_equals_the_oracle_at_the_edges(handle, monkeypatch):
    """Every signal video's captured reference equals the oracle frame for frame, packed and as floats, at lengths
    R mod 32 in {0, 1, 31}, R < 32, R = 0 and a 20-minute signal, next to audio videos."""
    rng = np.random.RandomState(5)
    lengths = [32, 33, 63, 7, 0, 64, 95, 1, 120000]
    xs = [LOW[rng.randint(0, len(LOW), n)] for n in lengths]
    for x in xs:
        x[rng.rand(len(x)) < 0.4] = 1.0
    V = len(xs)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    tv = np.repeat(np.arange(V, dtype=np.int32), 2)
    cs = np.tile([1.0, 3.0], len(tv))
    cue_off = np.arange(0, 2 * len(tv) + 1, 2)
    for label in (0.0, 0.3, -0.5):
        for env in ("1", "0"):
            with monkeypatch.context() as m:
                m.setenv("B2_REF_PACKED", env)
                m.setenv("B2_SUBBATCHES", "3")
                with handle.capture_reference(int(off[-1]) + 64, V) as cap:
                    handle.sync_tracks_sig(None, np.zeros(V + 1, np.int64), tv, 16000, 100, label,
                                           np.ones(V, np.uint8), np.concatenate(xs), off, cs, cs + 1.0, None, cue_off,
                                           GRID, 0.0, MOS)
            assert np.array_equal(cap["ref_off"], off)
            if env == "0":
                assert not cap["packed"].any()
            for v, x in enumerate(xs):
                f = so.frames(x, label)
                got = cap["ref"][off[v]: off[v + 1]]
                if cap["packed"][v]:
                    W = (len(f) + 31) // 32
                    assert np.array_equal(got[:W].view(np.uint32), so.packed_words(f)), (v, label)
                else:
                    assert np.array_equal(got, f), (v, label)


def test_out_of_domain_values(handle):
    """A 2.0 in one video and a NaN in another: the sentinel on all their tracks and outputs, in every memspace and
    with the search; every other track equals the same call without those videos; the next call is unaffected."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    videos = [(80.0 + v, ["sig", "audio"][v % 2] if v not in (2, 4) else "sig", [(1.0, 40 * v - 200)] * (1 + v % 2))
              for v in range(10)]
    c = _sig_corpus(videos, seed0=41)
    x = c["x"].copy()
    x[c["sig_off"][2] + 777] = 2.0
    x[c["sig_off"][4] + 5] = np.nan
    x[c["sig_off"][5] - 3] = 3.0   # a later one in the same video
    bad_c = dict(c, x=x)
    K = len(GRID)
    keep_v = [v for v in range(10) if v not in (2, 4)]
    keep_t = np.flatnonzero(np.isin(c["track_video"], keep_v))
    bad_t = np.flatnonzero(~np.isin(c["track_video"], keep_v))
    # the same corpus without the two videos
    remap = {v: i for i, v in enumerate(keep_v)}
    small = dict(c)
    small["track_video"] = np.array([remap[v] for v in c["track_video"][keep_t]], np.int32)
    small["cue_off"] = np.concatenate([[0], np.cumsum(np.diff(c["cue_off"])[keep_t])]).astype(np.int64)
    pick = np.concatenate([np.arange(c["cue_off"][t], c["cue_off"][t + 1]) for t in keep_t]).astype(np.int64)
    small["cue_start"], small["cue_end"] = c["cue_start"][pick], c["cue_end"][pick]
    small["pcm"] = np.concatenate([c["pcm"][c["pcm_off"][v]: c["pcm_off"][v + 1]] for v in keep_v])
    small["pcm_off"] = np.concatenate([[0], np.cumsum([c["pcm_off"][v + 1] - c["pcm_off"][v] for v in keep_v])])
    small["is_sig"] = c["is_sig"][keep_v]
    small["x"] = np.concatenate([c["x"][c["sig_off"][v]: c["sig_off"][v + 1]] for v in keep_v])
    small["sig_off"] = np.concatenate([[0], np.cumsum([c["sig_off"][v + 1] - c["sig_off"][v] for v in keep_v])])
    for k in ("is_subs", "is_pgs"):
        small[k] = np.zeros(len(keep_v), np.uint8)
    for gss in (False, True):
        cols = K + 1 if gss else K
        want = _new(handle, small, gss=gss)
        for memspace in (None, _native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
            got = (_new(handle, bad_c, gss=gss) if memspace is None
                   else _device_call(handle, bad_c, memspace, gss=gss))
            assert np.all(got["bk"][bad_t] == _native.B2_BEST_K_BAD_SIGNAL), (gss, memspace)
            assert np.all(np.isnan(got["bs"][bad_t])) and np.all(got["bo"][bad_t] == 0)
            rows = np.repeat(np.isin(np.arange(len(got["bs"])), bad_t), cols)
            assert np.all(np.isnan(got["a_s"][rows])) and np.all(got["a_o"][rows] == 0)
            if gss:
                assert np.all(np.isnan(got["ratio"][bad_t]))
            for k in want:
                g = got[k] if len(got[k]) == len(got["bs"]) else got[k].reshape(-1, cols)
                w = want[k] if len(want[k]) == len(want["bs"]) else want[k].reshape(-1, cols)
                assert np.array_equal(g[keep_t], w, equal_nan=True), (k, gss, memspace)
        # the next call on the handle is unaffected
        for a, b in zip(_new(handle, c, gss=gss).values(), _new(handle, c, gss=gss).values()):
            assert np.array_equal(a, b, equal_nan=True)
        assert np.all(_new(handle, c, gss=gss)["bk"] >= 0)
    # the host methods name the video and its first offending frame
    s = BatchSynchronizer(GRID, energy_threshold=THR)
    sv = np.flatnonzero(c["is_sig"])
    kw = dict(sig=np.concatenate([x[c["sig_off"][v]: c["sig_off"][v + 1]] for v in sv]),
              sig_off=np.concatenate([[0], np.cumsum(np.diff(c["sig_off"])[sv])]), sig_video=sv)
    with pytest.raises(ValueError, match="video 2: .* 2.0 at frame 777"):
        s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"], **kw)
    out = s.sync_device_tracks(_dev(c["pcm"]), c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                               c["cue_off"], **dict(kw, sig=_dev(kw["sig"])))
    torch.cuda.synchronize()
    assert np.all(out["best_k"].cpu().numpy()[bad_t] == _native.B2_BEST_K_BAD_SIGNAL)


def test_front_end_equals_the_call(handle):
    """BatchSynchronizer's four methods with sig / sig_off / sig_video give the native call's results; mixed with
    PGS and text videos; both kinds on one video and the sharded mode are refused; the search outside the device
    envelope is composed."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    videos = [(70.0 + v, ["sig", "audio", "sig", "pgs"][v % 4], [(GRID[v % 5], 30 * v - 100)]) for v in range(8)]
    c = _sig_corpus(videos, seed0=53)
    sv, pv = np.flatnonzero(c["is_sig"]), np.flatnonzero(c["is_pgs"])
    kw = dict(sig=np.concatenate([c["x"][c["sig_off"][v]: c["sig_off"][v + 1]] for v in sv]).astype(np.float32),
              sig_off=np.concatenate([[0], np.cumsum(np.diff(c["sig_off"])[sv])]), sig_video=sv,
              pgs_start=c["pgs_start"], pgs_end=c["pgs_end"],
              pgs_off=np.concatenate([[0], np.cumsum(np.diff(c["pgs_off"])[pv])]), pgs_video=pv)
    c32 = dict(c, x=c["x"].astype(np.float32).astype(np.float64))   # float32 inputs convert exactly
    for label in (0.0, 0.3):
        s = BatchSynchronizer(GRID, non_speech_label=label, energy_threshold=THR)
        want = _compose(handle, c32, "energy_zcr", label)
        got = s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                                 want_all=True, **kw)
        _same(dict(bs=got[0], bo=got[1], bk=got[2], a_s=got[3], a_o=got[4]), want, len(GRID), where=label)
        T = len(c["track_video"])
        if T == len(c["pcm_off"]) - 1:
            got = s.sync_host(c["pcm"], c["pcm_off"], c["cue_start"], c["cue_end"], c["cue_off"], **kw)
            assert np.array_equal(got[2], want["bk"])
        dkw = dict(kw, sig=torch.from_numpy(kw["sig"]).cuda())
        out = s.sync_device_tracks(_dev(c["pcm"]), c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                                   c["cue_off"], inputs_resident=True, **dkw)
        torch.cuda.synchronize()
        assert np.array_equal(out["best_k"].cpu().numpy(), want["bk"]) and np.array_equal(
            out["best_offset"].cpu().numpy(), want["bo"])
        out = s.sync_device(_dev(c["pcm"]), c["pcm_off"], c["cue_start"], c["cue_end"], c["cue_off"], **dkw)
        torch.cuda.synchronize()
        assert len(out["best_k"]) == len(c["pcm_off"]) - 1
    # --gss at a non-zero label with a PGS video: three levels, composed by the front end
    s = BatchSynchronizer(GRID + [None], non_speech_label=0.3, energy_threshold=THR)
    res = s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                             **kw)
    want = _compose(handle, c32, "energy_zcr", 0.3, gss=True)
    assert np.array_equal(res[2], want["bk"]) and np.array_equal(res[1], want["bo"])
    # refusals
    with pytest.raises(ValueError, match="one reference"):
        s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                           **dict(kw, pgs_video=sv[:1], pgs_off=[0, 1]))
    with pytest.raises(ValueError, match="serialized signal"):
        BatchSynchronizer(GRID).sync_device_candidate_sharded(_dev(c["pcm"]), c["pcm_off"], c["cue_start"],
                                                              c["cue_end"], c["cue_off"], sig=kw["sig"],
                                                              sig_off=kw["sig_off"], sig_video=sv)
    with pytest.raises(ValueError, match="increasing"):
        s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                           **dict(kw, sig_video=sv[::-1].copy()))


def test_resident_chains_interleave_signal_and_pcm_calls(handle, monkeypatch):
    """Unsynchronised resident calls alternating b2_sync_tracks_sig (with signals, text and PGS videos) with
    b2_sync_tracks and b2_sync_tracks_auditok over two corpora equal the same calls unchained."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    monkeypatch.setenv("B2_SUBBATCHES", "3")
    rng = np.random.RandomState(13)
    corpora = []
    for seed in (61, 67):
        videos = [(60.0 + 4 * (v % 3), ["sig", "audio", "sig", "pgs"][v % 4] if v % 3 else "audio",
                   [(GRID[int(rng.randint(0, 5))], int(rng.randint(-500, 500)))]) for v in range(24)]
        corpora.append(_sig_corpus(videos, seed0=seed))
    arms = [("energy_zcr", False, "sync_tracks"), ("energy_zcr", True, "sync_tracks_sig"),
            ("auditok", False, "sync_tracks_auditok"), ("auditok", True, "sync_tracks_sig")]
    syncs = [BatchSynchronizer(GRID, vad=a[0]) for a in arms]
    for s in syncs:
        s.use_torch_stream()
    used = []
    for name in ("sync_tracks", "sync_tracks_auditok", "sync_tracks_sig"):
        orig = getattr(_native.Handle, name)
        monkeypatch.setattr(_native.Handle, name,
                            (lambda o, n: lambda self, *a, **k: used.append(n) or o(self, *a, **k))(orig, name))
    dev = torch.device("cuda", handle.device)
    pcms = [torch.from_numpy(c["pcm"]).to(dev) for c in corpora]
    sigs = []
    for c in corpora:
        sv, pv = np.flatnonzero(c["is_sig"]), np.flatnonzero(c["is_pgs"])
        sigs.append(dict(sig=_dev(np.concatenate([c["x"][c["sig_off"][v]: c["sig_off"][v + 1]] for v in sv])),
                         sig_off=np.concatenate([[0], np.cumsum(np.diff(c["sig_off"])[sv])]), sig_video=sv,
                         pgs_start=c["pgs_start"], pgs_end=c["pgs_end"],
                         pgs_off=np.concatenate([[0], np.cumsum(np.diff(c["pgs_off"])[pv])]), pgs_video=pv))
    seq = [(i % len(arms), (i // 2) % 2) for i in range(4 * len(arms))]

    def call(si, ci, resident):
        c = corpora[ci]
        return syncs[si].sync_device_tracks(pcms[ci], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                                            c["cue_off"], inputs_resident=resident,
                                            **(sigs[ci] if arms[si][1] else {}))

    want = []
    for si, ci in seq:
        o = call(si, ci, False)
        torch.cuda.synchronize(dev)
        want.append({k: v.cpu().numpy() for k, v in o.items()})
    used.clear()
    outs = [call(si, ci, True) for si, ci in seq]
    torch.cuda.synchronize(dev)
    assert used == [arms[si][2] for si, _ in seq]
    for i, (o, w) in enumerate(zip(outs, want)):
        for k in w:
            assert np.array_equal(o[k].cpu().numpy(), w[k]), (i, seq[i], k)


def test_bad_arguments(handle):
    from ffsubsync_b200 import _native
    c = _sig_corpus([(60.0, "sig", [(1.0, 30)]), (61.0, "audio", [(1.0, -30)]), (62.0, "pgs", [(1.0, 10)])],
                    seed0=71)
    n0 = handle.launch_count

    def err(**kw):
        with pytest.raises(_native.NativeError) as e:
            _new(handle, dict(c, **kw))
        assert e.value.status == -1, str(e.value)
        return str(e.value)

    assert "sig_off not monotone" in err(sig_off=c["sig_off"][::-1].copy())
    assert "no signal reference" in err(is_sig=np.zeros(3, np.uint8))
    pcm_off = c["pcm_off"].copy()
    pcm_off[1:] += 160
    assert "non-empty PCM range" in err(pcm_off=pcm_off, pcm=np.zeros(int(pcm_off[-1]), np.int16))
    assert "signal and as a PGS" in err(is_pgs=np.array([1, 0, 1], np.uint8),
                                        pgs_off=np.concatenate([[0], c["pgs_off"][1:] + 1]),
                                        pgs_start=np.concatenate([[1.0], c["pgs_start"]]),
                                        pgs_end=np.concatenate([[2.0], c["pgs_end"]]))
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_sig(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, c["is_sig"], c["x"],
                               c["sig_off"], c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS,
                               ref_is_subs=np.array([1, 0, 0], np.uint8), ref_cue_start_s=[1.0], ref_cue_end_s=[2.0],
                               ref_cue_off=[0, 1, 1, 1])
    assert "signal and as a text" in str(e.value)
    # a host x under B2_DEVICE, and a null x with values
    import torch
    a = _sig_corpus([(60.0, "sig", [(1.0, 30)]), (61.0, "sig", [(1.0, -30)])], seed0=73)
    o = [torch.zeros(2, dtype=t, device="cuda") for t in (torch.float64, torch.int32, torch.int32)]
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_sig(None, a["pcm_off"], a["track_video"], 16000, 100, 0.0, a["is_sig"], a["x"].ctypes.data,
                               a["sig_off"], a["cue_start"], a["cue_end"], None, a["cue_off"], GRID, 0.0, MOS,
                               best_score=o[0].data_ptr(), best_offset=o[1].data_ptr(), best_k=o[2].data_ptr(),
                               memspace=_native.B2_DEVICE)
    assert e.value.status == -1 and "x: B2_DEVICE call with a host pointer" in str(e.value), str(e.value)
    assert "null signal values" in err(x=None)
    assert handle.launch_count == n0
