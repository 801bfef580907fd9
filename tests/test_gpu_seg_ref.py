"""GPU tests of sampled segments as references (b2_sync_tracks_seg; the reference's ``--multi-segment-sync``), alone
and next to full-audio, text-stream, PGS and signal videos in one batched call (run on an H100).

Yardsticks: the float64 assembly over the detector oracles (oracle/segment_oracle.py), this package's single-pair
MultiSegmentVideoSpeechTransformer, and the composition of public entry points the call replaces - per video the
detector over its segments placed into the sparse signal (BatchSynchronizer._reference_signals), one copy per track,
b2_rasterize, b2_align_batch, b2_reduce_ratios (and for the search gss_align_batch + the reference's combine) - which
the call must reproduce bit for bit, except where the composition's aligner reports B2_ALIGN_CAND_OVERFLOW."""
import numpy as np
import pytest

from oracle import segment_oracle as so
from oracle import sig_oracle
from oracle import vad_oracle as vo
from test_gpu_pgs_ref import _same

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
MOS = 6000


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _pcm(seconds, fr, seed, silent=False):
    """Synthetic speech-like PCM: 10 ms windows of silence / speech / noise in runs."""
    fpw = fr // 100
    rng = np.random.RandomState(seed)
    n_win = int(seconds * 100) + 1
    cls = np.repeat(rng.choice([0, 1, 2], n_win // 40 + 1, p=[0.4, 0.45, 0.15]), 40)[:n_win].astype(np.uint8)
    if silent:
        cls[:] = 0
    return vo.synth_pcm(cls, fpw, seed=seed)[: int(round(seconds * fr))]


def _cues(seconds, seed, n_tracks):
    from ffsubsync_b200.synth import synthetic_cues
    out = [synthetic_cues(seed + 7 * t, max(seconds, 30.0)) for t in range(n_tracks)]
    return [(s + 0.37 * (t + 1), e + 0.37 * (t + 1)) for t, (s, e) in enumerate(out)]


def _corpus(videos, fr=16000, seed=0, count=8, dur=60, skip=False, tracks=2, decoded=False, gap_noise=False):
    """videos: (seconds, kind) with kind "seg" (segments), "silent" (segments of silence) or "audio".  Segment videos
    hold their full decode (or only the decoded windows with ``decoded``).  Returns the call's inputs."""
    from ffsubsync_b200.batch import segment_table
    from ffsubsync_b200.speech_transformers import MultiSegmentVideoSpeechTransformer
    pcms, full, seg_v, totals, pieces = [], [], [], [], []
    t = MultiSegmentVideoSpeechTransformer(vad="energy", sample_rate=100, frame_rate=fr, non_speech_label=0.0,
                                           segment_count=count, segment_duration=dur, skip_intro_outro=skip)
    for v, (sec, kind) in enumerate(videos):
        x = _pcm(sec, fr, seed + 31 * v, silent=kind == "silent")
        full.append(x)
        if kind == "audio":
            pcms.append(x)
            continue
        seg_v.append(v)
        totals.append(len(x) / fr)
        if decoded:
            ps = []
            for s in t._segment_starts(len(x) / fr):
                a = min(len(x), int(round(s * fr)))
                ps.append(x[a: min(len(x), a + dur * fr)])
            pieces.append([len(q) for q in ps])
            pcms.append(np.concatenate(ps))
        else:
            pcms.append(x)
    pcm_off = np.concatenate([[0], np.cumsum([len(x) for x in pcms])]).astype(np.int64)
    tab = segment_table(pcm_off, fr, videos=seg_v, totals=totals if decoded else None, segment_count=count,
                        segment_duration=dur, skip_intro_outro=skip, piece_samples=pieces if decoded else None)
    pcm = np.concatenate(pcms).astype(np.int16)
    if gap_noise:   # every sample outside the segments of a segment video: loud noise
        used = np.zeros(len(pcm), bool)
        for v in range(len(videos)):
            if v not in seg_v:
                used[pcm_off[v]:pcm_off[v + 1]] = True
        for i, v in enumerate(seg_v):
            for j in range(tab["seg_off"][i], tab["seg_off"][i + 1]):
                used[pcm_off[v] + tab["seg_lo"][j]: pcm_off[v] + tab["seg_hi"][j]] = True
        rng = np.random.RandomState(99)
        pcm[~used] = rng.randint(-30000, 30000, int((~used).sum())).astype(np.int16)
    track_video, cs, ce_, offs = [], [], [], [0]
    for v, (sec, _) in enumerate(videos):
        for s, e in _cues(sec, seed + v, tracks):
            track_video.append(v)
            cs.append(s)
            ce_.append(e)
            offs.append(offs[-1] + len(s))
    return dict(pcm=pcm, pcm_off=pcm_off, fr=fr, full=full, tab=tab, seg_v=seg_v,
                track_video=np.asarray(track_video, np.int32), cue_start=np.concatenate(cs), cue_end=np.concatenate(ce_),
                cue_off=np.asarray(offs, np.int64))


def _sync(c, det="energy_zcr", label=0.0, gss=False, ratios=GRID, **extra):
    from ffsubsync_b200.batch import BatchSynchronizer
    return BatchSynchronizer(list(ratios) + ([None] if gss else []), frame_rate=c["fr"], non_speech_label=label,
                             vad=det, max_offset_seconds=MOS / 100.0, **extra)


def _host(c, **kw):
    bs = _sync(c, **{k: v for k, v in kw.items() if k in ("det", "label", "gss", "ratios")})
    r = bs.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                            want_all=True, **c["tab"], **kw.get("streams", {}))
    out = dict(bs=r[0], bo=r[1], bk=r[2], a_s=r[3], a_o=r[4])
    if kw.get("gss"):
        out["ratio"] = r[5]
    return out


def _device(c, resident=False, **kw):
    import torch
    bs = _sync(c, **{k: v for k, v in kw.items() if k in ("det", "label", "gss", "ratios")})
    T, K = len(c["track_video"]), len(bs.ratios) + (1 if bs.gss else 0)
    dev = torch.device("cuda", bs.handle.device)
    all_out = {"score": torch.zeros(T * K, dtype=torch.float64, device=dev),
               "offset": torch.zeros(T * K, dtype=torch.int32, device=dev)}
    out = bs.sync_device_tracks(torch.from_numpy(c["pcm"]).to(dev), c["pcm_off"], c["track_video"], c["cue_start"],
                                c["cue_end"], c["cue_off"], all_out=all_out, inputs_resident=resident,
                                **c["tab"], **kw.get("streams", {}))
    bs.handle.synchronize()
    r = dict(bs=out["best_score"].cpu().numpy(), bo=out["best_offset"].cpu().numpy(), bk=out["best_k"].cpu().numpy(),
             a_s=all_out["score"].cpu().numpy(), a_o=all_out["offset"].cpu().numpy())
    if bs.gss:
        r["ratio"] = out["gss_ratio"].cpu().numpy()
    return r


def _oracle_ref(c, v, det, label):
    i = c["seg_v"].index(v)
    t = c["tab"]
    js = range(t["seg_off"][i], t["seg_off"][i + 1])
    a, b = c["pcm_off"][v], c["pcm_off"][v + 1]
    from ffsubsync_b200.constants import DEFAULT_ENERGY_THRESHOLD, detector_chunk_bytes
    kw = dict(energy_threshold=DEFAULT_ENERGY_THRESHOLD) if det == "energy_zcr" else dict(
        chunk_samples=detector_chunk_bytes(c["fr"], 100) // 2)
    return so.segment_reference(c["pcm"][a:b], t["seg_total"][i], [t["seg_start"][j] for j in js],
                                [t["seg_lo"][j] for j in js], [t["seg_hi"][j] for j in js], 100, detector=det,
                                frame_rate=c["fr"], non_speech_label=label, **kw)


def _capture(handle, c, det, label, env=None, monkeypatch=None):
    V = len(c["pcm_off"]) - 1
    with handle.capture_reference(60_000_000 // 4, V) as cap:
        _host(c, det=det, label=label)
    return cap


def _check_capture(c, cap, det, label):
    for v in c["seg_v"]:
        a, b = cap["ref_off"][v], cap["ref_off"][v + 1]
        want = _oracle_ref(c, v, det, label).astype(np.float32)
        assert b - a == len(want), v
        if cap["packed"][v]:
            got = cap["ref"][a: a + (len(want) + 31) // 32].view(np.uint32)
            assert np.array_equal(got, sig_oracle.packed_words(want)), v
        else:
            assert np.array_equal(cap["ref"][a:b], want), v
    return cap


# ---------------------------------------------------------------- the reference, frame for frame

@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
@pytest.mark.parametrize("label", [0.0, 0.3])
@pytest.mark.parametrize("count,skip,fr", [(1, False, 16000), (3, True, 16000), (8, False, 16000), (8, True, 48000)])
def test_reference_frame_for_frame(handle, det, label, count, skip, fr):
    # 100 s and 300 s videos overlap their segments; 1500 s ones do not; a 45 s one is shorter than a segment
    c = _corpus([(100, "seg"), (300.5, "seg"), (30, "audio"), (1500, "seg"), (45.3, "seg")], fr=fr, count=count,
                skip=skip, tracks=1)
    _check_capture(c, _capture(handle, c, det, label), det, label)
    if det == "energy_zcr":   # the single-pair transformer on each full decode
        from ffsubsync_b200.speech_transformers import MultiSegmentVideoSpeechTransformer
        cap = _capture(handle, c, det, label)
        for v in c["seg_v"]:
            x = MultiSegmentVideoSpeechTransformer("energy", 100, fr, label, segment_count=count,
                                                   skip_intro_outro=skip).fit(c["full"][v]).transform()
            a, b = cap["ref_off"][v], cap["ref_off"][v + 1]
            if not cap["packed"][v]:
                assert np.array_equal(cap["ref"][a:b], x.astype(np.float32)), v


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
def test_reference_totals_layouts_and_misalignment(handle, monkeypatch, det):
    c = _corpus([(300, "seg"), (100, "seg")], tracks=1)
    # seg_total shorter and longer than the PCM
    c["tab"]["seg_total"] = np.array([250.25, 130.0])
    _check_capture(c, _capture(handle, c, det, 0.0), det, 0.0)
    # a misaligned layout (segments starting off a multiple of 8 samples): the lane-group kernel
    c2 = _corpus([(300, "seg"), (100, "seg")], tracks=1)
    c2["tab"]["seg_lo"] = c2["tab"]["seg_lo"] + 3
    c2["tab"]["seg_hi"] = np.minimum(c2["tab"]["seg_hi"] + 3, [300 * 16000] * 8 + [100 * 16000] * 8)
    _check_capture(c2, _capture(handle, c2, det, 0.0), det, 0.0)


# ---------------------------------------------------------------- results = the composition

def _compose(c, det="energy_zcr", label=0.0, gss=False, streams=None):
    from ffsubsync_b200 import _native
    bs = _sync(c, det=det, label=label, gss=gss)
    h = bs.handle
    refs, pgs, sig, seg = bs._all_refs(len(c["pcm_off"]) - 1, dict(c["tab"], **(streams or {})), on_device=False)
    ref, ref_off = bs._reference_signals(c["pcm"], c["pcm_off"], refs, pgs, sig, seg)
    parts = [ref[ref_off[v]: ref_off[v + 1]] for v in c["track_video"]]
    t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    t_ref = np.concatenate(parts).astype(np.float32)
    T, K = len(c["track_video"]), len(GRID)
    sub, sub_off = h.rasterize(c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, K, False, 100, 0.0)
    score, offset, status = h.align_batch(t_ref, t_off, sub, sub_off, T, K, MOS)
    b, o, k = h.reduce_ratios(score, offset, status, T, K, MOS)
    out = dict(bs=b, bo=o, bk=k, a_s=score, a_o=offset, status=status)
    if gss:
        from ffsubsync_b200.gss_batch import combine_gss, gss_align_batch
        g = gss_align_batch(t_ref, t_off, c["cue_start"], c["cue_end"], c["cue_off"], None, MOS, 100, 0.0, handle=h)
        b, o, k, r, a_s, a_o = combine_gss(b, o, k, g, K, MOS, score, offset)
        st = np.concatenate([status.reshape(T, K), np.zeros((T, 1), np.int32)], axis=1).ravel()
        out = dict(bs=b, bo=o, bk=k, a_s=a_s, a_o=a_o, ratio=r, status=st)
    for v in set(c["seg_v"]):
        if not so.has_speech(ref[ref_off[v]: ref_off[v + 1]]):
            for t in np.flatnonzero(c["track_video"] == v):
                out["bk"][t] = _native.B2_BEST_K_NO_SPEECH
    return out


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
@pytest.mark.parametrize("gss", [False, True])
def test_equals_composition(handle, det, gss):
    c = _corpus([(600, "seg"), (40, "audio"), (300, "seg"), (1200, "seg")], tracks=3)
    want = _compose(c, det, 0.0, gss)
    keys = ("bs", "bo", "bk", "a_s", "a_o") + (("ratio",) if gss else ())
    _same(_host(c, det=det, gss=gss), want, len(GRID), keys, "host")
    _same(_device(c, det=det, gss=gss), want, len(GRID), keys, "device")


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
def test_equals_composition_at_a_non_zero_label(handle, det):
    c = _corpus([(600, "seg"), (40, "audio"), (300, "seg")], tracks=2)
    _same(_host(c, det=det, label=0.3), _compose(c, det, 0.3), len(GRID), where="label 0.3")


def test_mixed_call(handle):
    """Segment, full-audio, text, PGS and signal videos in one call."""
    c = _corpus([(300, "seg"), (60, "audio"), (0.001, "audio"), (0.001, "audio"), (0.001, "audio"), (200, "seg")],
                tracks=2)
    V = 6
    # videos 2, 3, 4: text, PGS and signal references (no PCM)
    c["pcm_off"] = np.array([0, 300 * 16000, 360 * 16000, 360 * 16000, 360 * 16000, 360 * 16000, 560 * 16000],
                            np.int64)
    c["pcm"] = np.concatenate([c["full"][0], c["full"][1], c["full"][5]]).astype(np.int16)
    from ffsubsync_b200.batch import segment_table
    c["tab"] = segment_table(c["pcm_off"], 16000, videos=[0, 5])
    c["seg_v"] = [0, 5]
    sig_vals = np.where(np.arange(5000) % 97 < 40, 1.0, 0.25)
    streams = dict(ref_cue_start=[1.0, 30.0], ref_cue_end=[5.0, 44.0], ref_cue_off=[0, 1, 2],
                   ref_stream_video=[0, 2],   # video 0's text stream is dropped: sampling is audio-only
                   pgs_start=[2.0, 50.0], pgs_end=[9.0, 70.0], pgs_off=[0, 2], pgs_video=[3],
                   sig=sig_vals, sig_off=[0, 5000], sig_video=[4])
    for det in ("energy_zcr", "auditok"):
        for vad in (det, "subs_then_" + det):
            if vad == det:
                s = {k: v for k, v in streams.items() if not k.startswith("ref_")}
            else:
                s = streams
            from ffsubsync_b200.batch import BatchSynchronizer
            bs = BatchSynchronizer(GRID, non_speech_label=0.0, vad=vad, max_offset_seconds=MOS / 100.0)
            r = bs.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                                    c["cue_off"], want_all=True, **c["tab"], **s)
            want = _compose(c, det, 0.0, streams=s) if vad == det else None
            if want is not None:
                _same(dict(bs=r[0], bo=r[1], bk=r[2], a_s=r[3], a_o=r[4]), want, len(GRID), where=vad)
            # every track aligns, but video 2's without its text stream (then an empty audio reference: -1)
            ok = c["track_video"] != 2 if vad == det else np.ones(len(r[2]), bool)
            assert np.all(r[2][ok] >= 0) and (vad != det or np.all(r[2][~ok] == -1)), (vad, r[2])
    # a video with segments and a PGS / signal reference is refused
    from ffsubsync_b200.batch import BatchSynchronizer
    bs = BatchSynchronizer(GRID, max_offset_seconds=MOS / 100.0)
    with pytest.raises(ValueError, match="sampled segments and a PGS reference"):
        bs.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                            **c["tab"], pgs_start=[2.0], pgs_end=[9.0], pgs_off=[0, 1], pgs_video=[0])
    with pytest.raises(ValueError, match="does not take sampled segment"):
        bs.sync_device_candidate_sharded(None, c["pcm_off"], c["cue_start"], c["cue_end"], c["cue_off"], **c["tab"])


# ---------------------------------------------------------------- gaps are never read

def test_gaps_are_not_read(handle):
    base = _corpus([(600, "seg"), (40, "audio"), (100, "seg")], tracks=2)
    noisy = _corpus([(600, "seg"), (40, "audio"), (100, "seg")], tracks=2, gap_noise=True)
    dec = _corpus([(600, "seg"), (40, "audio"), (100, "seg")], tracks=2, decoded=True)
    assert not np.array_equal(base["pcm"], noisy["pcm"])
    for det in ("energy_zcr", "auditok"):
        want = _host(base, det=det)
        for c, where in ((noisy, "noise host"), (dec, "decoded host")):
            got = _host(c, det=det)
            for k in want:
                assert np.array_equal(got[k], want[k], equal_nan=True), (det, where, k)
        for c, where in ((base, "device"), (noisy, "noise device"), (dec, "decoded device")):
            got = _device(c, det=det)
            for k in want:
                assert np.array_equal(got[k], want[k], equal_nan=True), (det, where, k)


# ---------------------------------------------------------------- no speech

def test_no_speech_sentinel(handle):
    from ffsubsync_b200 import _native
    c = _corpus([(600, "seg"), (300, "silent"), (40, "audio")], tracks=2)
    dev = _device(c)
    K = len(GRID)
    bad = c["track_video"] == 1
    assert np.all(dev["bk"][bad] == _native.B2_BEST_K_NO_SPEECH) and np.all(np.isnan(dev["bs"][bad]))
    assert np.all(dev["bo"][bad] == 0) and np.all(np.isnan(dev["a_s"].reshape(-1, K)[bad]))
    assert np.all(dev["a_o"].reshape(-1, K)[bad] == 0)
    # the other tracks are those of the same call without the silent video's tracks... of the composition
    want = _compose(c)
    _same({k: v[~bad] if len(v) == len(bad) else v.reshape(len(bad), -1)[~bad].ravel() for k, v in dev.items()},
          {k: (v[~bad] if len(v) == len(bad) else v.reshape(len(bad), -1)[~bad].ravel()) for k, v in want.items()},
          K, where="other tracks")
    with pytest.raises(ValueError, match="video 1: Unable to detect speech in any sampled segment"):
        _host(c)
    # the search: device-driven and the composed fallback both give the sentinel
    g = _device(c, gss=True)
    assert np.all(g["bk"][bad] == _native.B2_BEST_K_NO_SPEECH) and np.all(np.isnan(g["ratio"][bad]))
    # apply_sync treats it as a failed track
    import torch
    bs = _sync(c)
    out = {"best_score": torch.from_numpy(dev["bs"]).cuda(), "best_offset": torch.from_numpy(dev["bo"]).cuda(),
           "best_k": torch.from_numpy(dev["bk"]).cuda()}
    res = bs.apply_sync(out, c["cue_start"], c["cue_end"], c["cue_off"])
    st = res["status"].cpu().numpy()
    from ffsubsync_b200.sync_output import FAILED
    assert np.all(st[bad] & FAILED) and not np.any(st[~bad] & FAILED)
    assert np.all(np.isnan(res["scale"].cpu().numpy()[bad]))


# ---------------------------------------------------------------- invariance

@pytest.mark.parametrize("env", [{"B2_SUBBATCHES": "1"}, {"B2_SUBBATCHES": "3"}, {"B2_REF_PACKED": "0"},
                                 {"B2_ALIGN_PATH": "tiled"}, {"B2_ALIGN_PATH": "runs"}, {"B2_VAD_LAYOUT": "group"}])
def test_invariant_under_knobs(handle, monkeypatch, env):
    c = _corpus([(600, "seg"), (40, "audio"), (120, "seg")] * 33, tracks=1)   # 99 tracks: three sub-batches
    want = _device(c)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    got = _device(c)
    for k in want:
        assert np.array_equal(got[k], want[k], equal_nan=True), (env, k)


def test_resident_chaining(handle, monkeypatch):
    """Resident calls chain with the other sync calls in any order and give the results of separate calls."""
    import torch
    monkeypatch.setenv("B2_SUBBATCHES", "3")
    c = _corpus([(600, "seg"), (40, "audio"), (120, "seg")] * 33, tracks=1)
    plain = _corpus([(200, "audio"), (100, "audio")] * 50, tracks=1)
    want_seg = _device(c)
    bs = _sync(plain)
    dev = torch.device("cuda", bs.handle.device)
    pp = torch.from_numpy(plain["pcm"]).to(dev)

    def plain_call():
        o = bs.sync_device_tracks(pp, plain["pcm_off"], plain["track_video"], plain["cue_start"], plain["cue_end"],
                                  plain["cue_off"], inputs_resident=True)
        return o

    first = plain_call()
    bs.handle.synchronize()
    want_plain = first["best_k"].cpu().numpy().copy(), first["best_score"].cpu().numpy().copy()
    for order in range(2):
        a = plain_call() if order == 0 else None
        got = _device(c, resident=True)
        b = plain_call()
        bs.handle.synchronize()
        for k in want_seg:
            assert np.array_equal(got[k], want_seg[k], equal_nan=True), (order, k)
        for o in (a, b):
            if o is not None:
                assert np.array_equal(o["best_k"].cpu().numpy(), want_plain[0])
                assert np.array_equal(o["best_score"].cpu().numpy(), want_plain[1])
