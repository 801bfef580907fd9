"""GPU tests of PGS display intervals as references (b2_rasterize_pgs, b2_sync_tracks_pgs; the reference's
``--pgs-ref-stream``), next to audio videos and text-stream references in one batched call (run on an H100).

Yardsticks: the fixture recorded from the reference (tests/golden/pgs.json), and the composition of public entry
points the call replaces - per video b2_rasterize_pgs, b2_rasterize (ratio 1.0, level 1.0) or the detector, one
copy per track, b2_rasterize of the tracks, b2_align_batch, b2_reduce_ratios (and for the search gss_align_batch +
the reference's combine) - which the call must reproduce bit for bit, except where the composition's aligner
reports B2_ALIGN_CAND_OVERFLOW: there the call's score is at least as high."""
import json
import os

import numpy as np
import pytest

import cases
from conftest import ROOT
from oracle import aligner_oracle as ao
from oracle import pgs_oracle as po
from oracle import raster_oracle as ro
from test_gpu_subs_ref import _chunk, _corpus, _det

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
MOS = 6000
THR = 100000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(ROOT, "tests", "golden", "pgs.json")) as fh:
        return json.load(fh)


def _runs(x):
    nz = np.asarray(x) != 0
    d = np.diff(np.concatenate([[0], nz.astype(np.int8), [0]]))
    return [int(v) for v in np.flatnonzero(d == 1)], [int(v) for v in np.flatnonzero(d == -1)]


def _pgs_corpus(videos, seed0=0):
    """videos: (duration_s, kind in "audio" / "text" / "pgs", tracks).  A PGS video's intervals are its master cue
    list with one overlapping, one unsorted and one negative-duration interval added; it has no PCM."""
    c = _corpus([(d, k != "audio", t) for d, k, t in videos], seed0=seed0)
    V = len(videos)
    is_pgs = np.array([k == "pgs" for _, k, _ in videos], np.uint8)
    ps, pe, lens = [], [], []
    for v in range(V):
        if is_pgs[v]:
            s, e = list(c["rcs"][v]), list(c["rce"][v])
            s += [s[3] + 0.5, 2.0, 30.0]
            e += [e[3] + 2.0, 3.5, 29.0]
            ps += s
            pe += e
            lens.append(len(s))
        else:
            lens.append(0)
    c["is_pgs"] = is_pgs
    c["pgs_start"], c["pgs_end"] = np.array(ps), np.array(pe)
    c["pgs_off"] = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    # text references only for the text videos
    keep_v = (c["is_subs"] != 0) & (is_pgs == 0)
    pick = np.concatenate([np.arange(c["ref_off"][v], c["ref_off"][v + 1]) for v in range(V) if keep_v[v]]
                          + [np.zeros(0, np.int64)]).astype(np.int64)
    c["ref_start"], c["ref_end"], c["ref_keep"] = c["ref_start"][pick], c["ref_end"][pick], c["ref_keep"][pick]
    c["ref_off"] = np.concatenate([[0], np.cumsum(np.where(keep_v, np.diff(c["ref_off"]), 0))]).astype(np.int64)
    c["is_subs"] = keep_v.astype(np.uint8)
    return c


def _new(handle, c, det="energy_zcr", label=0.0, grid=GRID, mos=MOS, gss=False, memspace=None, want_all=True,
         outs=None):
    from ffsubsync_b200 import _native
    text = {} if not c["is_subs"].any() else dict(ref_is_subs=c["is_subs"], ref_cue_start_s=c["ref_start"],
                                                   ref_cue_end_s=c["ref_end"], ref_cue_keep=c["ref_keep"],
                                                   ref_cue_off=c["ref_off"])
    pcm = c["pcm"] if memspace in (None, _native.B2_HOST) else c["pcm_dev"]
    r = handle.sync_tracks_pgs(
        pcm, c["pcm_off"], c["track_video"], c["fr"], 100, label, c["is_pgs"], c["pgs_start"], c["pgs_end"],
        c["pgs_off"], c["cue_start"], c["cue_end"], None, c["cue_off"], grid, 0.0, mos, detector=_det(det),
        energy_threshold=THR, chunk_samples=_chunk(c["fr"]), gss=gss, want_all=want_all, want_evals=False,
        memspace=_native.B2_HOST if memspace is None else memspace, **text, **(outs or {}))
    out = dict(bs=r[0], bo=r[1], bk=r[2], a_s=r[3], a_o=r[4])
    if gss:
        out["ratio"] = r[5]
    return out


def _refs(handle, c, det, label):
    """Each video's reference by public calls."""
    if c["pcm_off"][-1] == 0:
        d, d_off = np.zeros(0, np.float32), np.zeros(len(c["pcm_off"]), np.int64)
    elif det == "auditok":
        d64, d_off = handle.vad_auditok(c["pcm"], c["pcm_off"], c["fr"], 100, label, chunk_samples=_chunk(c["fr"]))
        d = d64.astype(np.float32)
    else:
        d, d_off = handle.vad_energy_zcr(c["pcm"], c["pcm_off"], c["fr"], 100, label, THR)
    s, s_off = handle.rasterize(c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"], [1.0], 1, False, 100, 0.0,
                                levels=[1.0])
    vids = np.flatnonzero(c["is_pgs"])
    p, p_off = handle.rasterize_pgs(c["pgs_start"], c["pgs_end"],
                                    np.concatenate([[0], np.cumsum(np.diff(c["pgs_off"])[vids])]), 100, 0.0)
    out = []
    for v in range(len(c["pcm_off"]) - 1):
        if c["is_pgs"][v]:
            i = int(np.searchsorted(vids, v))
            out.append(p[p_off[i]: p_off[i + 1]])
        elif c["is_subs"][v]:
            out.append(s[s_off[v]: s_off[v + 1]])
        else:
            out.append(d[d_off[v]: d_off[v + 1]])
    return out


def _compose(handle, c, det="energy_zcr", label=0.0, grid=GRID, mos=MOS, gss=False):
    refs = _refs(handle, c, det, label)
    parts = [refs[v] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    t_ref = np.concatenate(parts) if parts else np.zeros(0, np.float32)
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


def _same(got, want, K, keys=("bs", "bo", "bk", "a_s", "a_o"), where=""):
    """Bit for bit, except a track where a job of the composition overflowed its candidate list
    (B2_ALIGN_CAND_OVERFLOW): there the call's scores are at least the composition's."""
    from ffsubsync_b200._native import ALIGN_CAND_OVERFLOW
    T = len(want["bs"])
    over = (np.asarray(want["status"]).reshape(T, -1) & ALIGN_CAND_OVERFLOW).any(axis=1)
    for k in keys:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        rows = np.repeat(~over, len(g) // max(T, 1)) if len(g) != T else ~over
        assert np.array_equal(g[rows], w[rows]), (where, k)
    if over.any():
        assert np.all(np.asarray(got["bs"])[over] >= np.asarray(want["bs"])[over]), where


# ---------------------------------------------------------------- the rasteriser against the reference

def test_rasterize_pgs_matches_the_reference(handle, golden):
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.speech_transformers import PGSSpeechTransformer
    rows = [r for r in golden["pgs_signals"] if not r["error"]]
    for row in golden["pgs_signals"]:
        iv = list(zip(row["starts"], row["ends"]))
        if row["error"]:
            with pytest.raises(_native.NativeError) as e:
                handle.rasterize_pgs(row["starts"], row["ends"], [0, len(iv)], 100, row["start_seconds"])
            assert e.value.status == -1
            with pytest.raises(ValueError):
                PGSSpeechTransformer(100, row["start_seconds"]).fit(iv)
            continue
        x, off = handle.rasterize_pgs(row["starts"], row["ends"], [0, len(iv)], 100, row["start_seconds"])
        assert len(x) == row["length"] and _runs(x) == (row["run_starts"], row["run_stops"]), row["name"]
        assert set(np.unique(x)) <= {0.0, 1.0}
        t = PGSSpeechTransformer(100, row["start_seconds"]).fit(iv)
        assert np.array_equal(t.transform(), po.pgs_signal(iv, 100, row["start_seconds"])), row["name"]
        assert t.num_frames is None
    # every row in one call, host and device memory, at a non-zero base
    starts = np.concatenate([r["starts"] for r in rows])
    ends = np.concatenate([r["ends"] for r in rows])
    off = np.concatenate([[0], np.cumsum([len(r["starts"]) for r in rows])]).astype(np.int64)
    for ss in (0, 3, -2):
        sel = [r for r in rows if r["start_seconds"] == ss]
        st = np.concatenate([r["starts"] for r in sel])
        en = np.concatenate([r["ends"] for r in sel])
        of = np.concatenate([[0], np.cumsum([len(r["starts"]) for r in sel])]).astype(np.int64)
        x, xo = handle.rasterize_pgs(st, en, of, 100, ss)
        for i, r in enumerate(sel):
            assert _runs(x[xo[i]: xo[i + 1]]) == (r["run_starts"], r["run_stops"]), (r["name"], ss)
        dev = torch.full((int(xo[-1]) + 10,), 7.0, dtype=torch.float32, device="cuda")
        handle.rasterize_pgs(st, en, of, 100, ss, out=dev.data_ptr(), out_off=xo + 5, memspace=_native.B2_DEVICE)
        handle.synchronize()
        y = dev.cpu().numpy()
        assert np.array_equal(y[5:-5], x) and np.all(y[:5] == 7.0) and np.all(y[-5:] == 7.0)
    assert len(starts) == off[-1]


def test_reference_grid_and_search_through_the_call(handle, golden):
    """The reference's own results: its 2 h PGS reference and an input track 25/24 slower and 3.5 s late;
    MaxScoreAligner over the 7-ratio grid, and with the golden-section search."""
    ms, gs = golden["pgs_maxscore"], golden["pgs_gss"]
    row = [r for r in golden["pgs_signals"] if r["name"] == "two_hours" and r["start_seconds"] == 0][0]
    grid = cases.ratio_grid()
    ref = po.pgs_signal(list(zip(row["starts"], row["ends"])), 100, 0)
    n_in = len(ms["in_starts"])
    for gss in (False, True):
        r = handle.sync_tracks_pgs(None, [0, 0], [0], 16000, 100, 0.0, [1], row["starts"], row["ends"],
                                   [0, len(row["starts"])], ms["in_starts"], ms["in_ends"], None, [0, n_in], grid,
                                   0.0, ms["max_offset_seconds"] * 100, gss=gss, want_all=True)
        K1 = len(grid) + int(gss)
        for k, want in enumerate(ms["per_ratio"]):
            if r[4][k] != want["offset"]:   # only a tie may order differently
                sub64 = ro.rasterize(ms["in_starts"], ms["in_ends"], None, 100, 0, grid[k])[0]
                assert ao.exact_score(ref, sub64, int(r[4][k])) == ao.exact_score(ref, sub64, want["offset"]), k
            tol = 1e-9 if grid[k] <= 1.0 else 1e-6
            assert abs(r[3][k] - want["score"]) <= tol * abs(want["score"]), (k, r[3][k], want["score"])
        assert len(r[3]) == K1
        best = gs["best"] if gss else ms["best"]
        assert int(r[2][0]) == best["index"] and r[1][0] == best["offset"], (gss, r[2][0], r[1][0])
        if gss:
            want = gs["per_candidate"][-1]
            assert r[4][-1] == want["offset"] and abs(r[3][-1] - want["score"]) <= 1e-6 * abs(want["score"])
            assert abs(r[5][0] - gs["gss_ratio"]) <= 1e-4


# ---------------------------------------------------------------- the call against the composition

MIXED = [(200.0, "pgs", [(1.0, 250), (25 / 24.0, -600)]),
         (240.0, "audio", [(25 / 24.0, -700), (1.0, 1234)]),
         (150.0, "text", [(23.976 / 24, 300)]),
         (120.0, "pgs", []),
         (180.0, "pgs", [(24 / 25.0, 900), (1.0, -900), (1.0, 40)]),
         (210.0, "audio", [(1.0, 40)])]


@pytest.fixture(scope="module")
def mixed():
    return _pgs_corpus(MIXED, seed0=5)


def test_planted_ratio_and_delay_are_recovered(handle, mixed):
    c = mixed
    got = _new(handle, c)
    t = 0
    for v, (_, kind, tracks) in enumerate(MIXED):
        for ratio, delta in tracks:
            if kind == "pgs":
                assert GRID[int(got["bk"][t])] == pytest.approx(ratio), (v, t)
                assert abs(int(got["bo"][t]) - delta) <= 2, (v, t, got["bo"][t], delta)
            t += 1


# an all-PGS call runs no detector: one detector suffices there
@pytest.mark.parametrize("corpus_kind,det", [("all_pgs", "energy_zcr"), ("pgs_audio", "energy_zcr"),
                                             ("pgs_audio", "auditok"), ("pgs_text_audio", "energy_zcr"),
                                             ("pgs_text_audio", "auditok")])
def test_equals_composition_on_every_path_and_memspace(handle, monkeypatch, corpus_kind, det):
    import torch
    from ffsubsync_b200 import _native
    rng = np.random.RandomState(3)
    kinds = {"all_pgs": ["pgs"], "pgs_audio": ["pgs", "audio"], "pgs_text_audio": ["pgs", "text", "audio"]}[corpus_kind]
    videos = [(90.0 + 3 * (v % 5), kinds[v % len(kinds)],
               [(GRID[int(rng.randint(0, 5))], int(rng.randint(-800, 800))) for _ in range([1, 2, 0, 2][v % 4])])
              for v in range(80)]
    c = _pgs_corpus(videos, seed0=17)
    T, K = len(c["track_video"]), len(GRID)
    dev = torch.device("cuda", handle.device)
    c["pcm_dev"] = torch.from_numpy(c["pcm"]).to(dev).data_ptr() if len(c["pcm"]) else None
    keep = torch.from_numpy(c["pcm"]).to(dev) if len(c["pcm"]) else None   # noqa: F841 (keeps pcm_dev alive)
    labels = (0.0, 0.3) if "audio" in kinds else (0.0,)
    for label in labels:
        want = _compose(handle, c, det, label)
        if keep is not None:
            c["pcm_dev"] = keep.data_ptr()
        _same(_new(handle, c, det, label), want, K, where=("default", label))
        _same(_new(handle, c, det, label, want_all=False), want, K, keys=("bs", "bo", "bk"), where=("winner", label))
        for env in ({"B2_SUBBATCHES": "1"}, {"B2_SUBBATCHES": "3", "B2_VAD_SMS": "8"}, {"B2_ALIGN_PATH": "tiled"},
                    {"B2_ALIGN_PATH": "runs"}, {"B2_ALIGN_PATH": "big"}, {"B2_FUSED_RASTER": "0"}):
            with monkeypatch.context() as m:
                for k, v in env.items():
                    m.setenv(k, v)
                _same(_new(handle, c, det, label), want, K, where=(env, label))
        for ms in (_native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
            o = dict(best_score=torch.full((T,), -7, dtype=torch.float64, device=dev),
                     best_offset=torch.full((T,), -7, dtype=torch.int32, device=dev),
                     best_k=torch.full((T,), -7, dtype=torch.int32, device=dev),
                     all_score=torch.zeros(T * K, dtype=torch.float64, device=dev),
                     all_offset=torch.zeros(T * K, dtype=torch.int32, device=dev))
            torch.cuda.synchronize(dev)
            _new(handle, c, det, label, memspace=ms, outs={k: v.data_ptr() for k, v in o.items()})
            handle.synchronize()
            got = dict(bs=o["best_score"].cpu().numpy(), bo=o["best_offset"].cpu().numpy(),
                       bk=o["best_k"].cpu().numpy(), a_s=o["all_score"].cpu().numpy(),
                       a_o=o["all_offset"].cpu().numpy())
            _same(got, want, K, where=(ms, label))
    # --gss at label 0, on the device-driven rounds
    want = _compose(handle, c, det, 0.0, gss=True)
    got = _new(handle, c, det, 0.0, gss=True)
    _same(got, want, K + 1, where="gss")
    assert np.array_equal(got["ratio"], want["ratio"], equal_nan=True)


def test_calls_without_pgs_equal_the_existing_calls(handle):
    c = _corpus([(120.0, False, [(1.0, 100), (25 / 24.0, -300)]), (90.0, True, [(1.0, 50)]),
                 (100.0, False, [(24 / 25.0, 0)])], seed0=23)
    V = len(c["pcm_off"]) - 1
    for det in ("energy_zcr", "auditok"):
        want = handle.sync_tracks_subs(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, c["is_subs"],
                                       c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"], c["cue_start"],
                                       c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS, detector=_det(det),
                                       energy_threshold=THR, chunk_samples=_chunk(), want_all=True)
        got = handle.sync_tracks_pgs(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, None, [], [],
                                     np.zeros(V + 1, np.int64), c["cue_start"], c["cue_end"], None, c["cue_off"], GRID,
                                     0.0, MOS, ref_is_subs=c["is_subs"], ref_cue_start_s=c["ref_start"],
                                     ref_cue_end_s=c["ref_end"], ref_cue_keep=c["ref_keep"], ref_cue_off=c["ref_off"],
                                     detector=_det(det), energy_threshold=THR, chunk_samples=_chunk(), want_all=True)
        for a, b in zip(got, want):
            assert np.array_equal(a, b), det
    from ffsubsync_b200.batch import BatchSynchronizer
    s = BatchSynchronizer(GRID)
    pcm_off = c["pcm_off"]
    audio = [0, 2]
    pcm = np.concatenate([c["pcm"][pcm_off[v]:pcm_off[v + 1]] for v in audio])
    off = np.array([0, pcm_off[1] - pcm_off[0], pcm_off[1] - pcm_off[0] + pcm_off[3] - pcm_off[2]])
    t_sel = [t for t, v in enumerate(c["track_video"]) if v in audio]
    cs = [c["cue_start"][c["cue_off"][t]:c["cue_off"][t + 1]] for t in t_sel]
    ce = [c["cue_end"][c["cue_off"][t]:c["cue_off"][t + 1]] for t in t_sel]
    tv = np.array([audio.index(c["track_video"][t]) for t in t_sel], np.int32)
    co = np.concatenate([[0], np.cumsum([len(x) for x in cs])])
    a = s.sync_host_tracks(pcm, off, tv, np.concatenate(cs), np.concatenate(ce), co)
    b = s.sync_host_tracks(pcm, off, tv, np.concatenate(cs), np.concatenate(ce), co, pgs_start=None, pgs_end=None,
                           pgs_off=None, pgs_video=None)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_resident_calls_alternate_with_the_other_sync_calls(handle, monkeypatch):
    """Unsynchronised resident calls alternating b2_sync_tracks, b2_sync_tracks_auditok, b2_sync_tracks_subs and
    b2_sync_tracks_pgs (with the energy detector, with auditok, and with text streams as well) over two corpora
    equal the same calls unchained."""
    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    monkeypatch.setenv("B2_SUBBATCHES", "3")
    rng = np.random.RandomState(9)
    corpora = []
    for seed in (31, 37):
        videos = [(60.0 + 4 * (v % 3), ["pgs", "audio", "text"][v % 3] if v % 2 else "audio",
                   [(GRID[int(rng.randint(0, 5))], int(rng.randint(-500, 500)))]) for v in range(24)]
        corpora.append(_pgs_corpus(videos, seed0=seed))
    # (vad, text streams given, PGS intervals given) -> the entry point the call takes
    arms = [("energy_zcr", False, False, "sync_tracks"), ("auditok", False, False, "sync_tracks_auditok"),
            ("subs_then_energy_zcr", True, False, "sync_tracks_subs"), ("energy_zcr", False, True, "sync_tracks_pgs"),
            ("subs_then_auditok", True, True, "sync_tracks_pgs"), ("auditok", False, True, "sync_tracks_pgs")]
    syncs = [BatchSynchronizer(GRID, vad=a[0]) for a in arms]
    for s in syncs:
        s.use_torch_stream()
    used = []
    for name in ("sync_tracks", "sync_tracks_auditok", "sync_tracks_subs", "sync_tracks_pgs"):
        orig = getattr(_native.Handle, name)
        monkeypatch.setattr(_native.Handle, name,
                            (lambda o, n: lambda self, *a, **k: used.append(n) or o(self, *a, **k))(orig, name))

    def args(c, si):
        _, text, pgs, _ = arms[si]
        streams = {}
        if text:
            tv = np.flatnonzero(c["is_subs"])
            streams = dict(ref_cue_start=c["ref_start"], ref_cue_end=c["ref_end"],
                           ref_cue_off=np.concatenate([[0], np.cumsum(np.diff(c["ref_off"])[tv])]),
                           ref_stream_video=tv, ref_cue_keep=c["ref_keep"])
        if pgs:
            pv = np.flatnonzero(c["is_pgs"])
            streams.update(pgs_start=c["pgs_start"], pgs_end=c["pgs_end"],
                           pgs_off=np.concatenate([[0], np.cumsum(np.diff(c["pgs_off"])[pv])]), pgs_video=pv)
        return streams

    dev = torch.device("cuda", handle.device)
    pcms = [torch.from_numpy(c["pcm"]).to(dev) for c in corpora]
    # calls without a kind of reference treat those videos as audio: they have no PCM, so a detector output of 0
    # windows, which both the chained and the unchained calls see
    seq = [(i % len(arms), (i // 3) % 2) for i in range(2 * len(arms))]

    def call(si, ci, resident):
        c = corpora[ci]
        return syncs[si].sync_device_tracks(pcms[ci], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                                            c["cue_off"], inputs_resident=resident, **args(c, si))

    want = []
    for si, ci in seq:
        o = call(si, ci, False)
        torch.cuda.synchronize(dev)
        want.append({k: v.cpu().numpy() for k, v in o.items()})
    used.clear()
    outs = [call(si, ci, True) for si, ci in seq]
    torch.cuda.synchronize(dev)
    assert used == [arms[si][3] for si, _ in seq]
    for i, (o, w) in enumerate(zip(outs, want)):
        for k in w:
            assert np.array_equal(o[k].cpu().numpy(), w[k]), (i, seq[i], k)


def test_bad_arguments(handle, mixed):
    from ffsubsync_b200 import _native
    c = mixed
    V = len(c["pcm_off"]) - 1
    n0 = handle.launch_count

    def call(**kw):
        d = dict(c)
        d.update(kw)
        with pytest.raises(_native.NativeError) as e:
            _new(handle, d, **{k: v for k, v in kw.items() if k in ("det", "label", "gss", "mos")})
        return e.value

    bad_end = c["pgs_end"].copy()
    bad_end[1] = np.nan
    big = c["pgs_end"].copy()
    big[2] = 1e10
    neg = c["pgs_end"].copy()
    v0 = int(np.flatnonzero(c["is_pgs"])[0])
    neg[c["pgs_off"][v0]: c["pgs_off"][v0 + 1]] = -0.05
    pcm_bad = c["pcm_off"].copy()
    pcm_bad[1:] += 160   # video 0 (PGS) gets samples
    empty_off = c["pgs_off"].copy()
    empty_off[v0 + 1:] -= empty_off[v0 + 1] - empty_off[v0]
    both = c["is_subs"].copy()
    both[v0] = 1
    errs = [call(pgs_end=bad_end), call(pgs_end=big), call(pgs_end=neg), call(pcm_off=pcm_bad),
            call(is_pgs=np.zeros(V, np.uint8)), call(pgs_off=c["pgs_off"][::-1].copy()),
            call(pgs_off=empty_off, pgs_start=c["pgs_start"][: empty_off[-1]], pgs_end=c["pgs_end"][: empty_off[-1]])]
    assert all(e.status == -1 for e in errs), [str(e) for e in errs]
    assert "not finite" in str(errs[0]) and "negative signal length" in str(errs[2])
    assert "non-empty PCM range" in str(errs[3]) and "no PGS reference" in str(errs[4])
    assert "empty interval list" in str(errs[6])
    # both kinds on one video: rejected by the ABI
    with pytest.raises(_native.NativeError) as e:
        handle.sync_tracks_pgs(c["pcm"], c["pcm_off"], c["track_video"], 16000, 100, 0.0, c["is_pgs"], c["pgs_start"],
                               c["pgs_end"], c["pgs_off"], c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0,
                               MOS, ref_is_subs=both, ref_cue_start_s=c["ref_start"], ref_cue_end_s=c["ref_end"],
                               ref_cue_off=c["ref_off"])
    assert e.value.status == -1 and "both" in str(e.value)
    # three levels with the search
    with pytest.raises(_native.NativeError) as e:
        _new(handle, c, label=0.3, gss=True)
    assert e.value.status == -6
    with pytest.raises(_native.NativeError) as e:
        handle.rasterize_pgs([], [], [0, 0], 100, 0.0)
    assert e.value.status == -1
    assert handle.launch_count == n0
    # the front end composes the search for the three-level call instead
    from ffsubsync_b200.batch import BatchSynchronizer
    s = BatchSynchronizer(GRID + [None], non_speech_label=0.3)
    pv = np.flatnonzero(c["is_pgs"])
    res = s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                             pgs_start=c["pgs_start"], pgs_end=c["pgs_end"],
                             pgs_off=np.concatenate([[0], np.cumsum(np.diff(c["pgs_off"])[pv])]), pgs_video=pv)
    want = _compose(handle, dict(c, is_subs=np.zeros(V, np.uint8), ref_start=np.zeros(0), ref_end=np.zeros(0),
                                 ref_keep=np.zeros(0, np.uint8), ref_off=np.zeros(V + 1, np.int64)),
                    label=0.3, gss=True)
    assert np.array_equal(res[2], want["bk"]) and np.array_equal(res[1], want["bo"])
