"""GPU suite of the speech output of the batched sync calls (b2_speech_output, ``--serialize-speech``).

Every written frame is checked against the oracles the reference-signal suites use (energy / ZCR, auditok, raster,
PGS, segment, the signal rule), rounded to float32 and widened, and against the same call's b2_capture_reference
buffer, unpacked and widened.  The output is prefilled with NaN, so a frame the call did not write fails, and nothing
past speech_off[n] may be written.  Further: the results and launch counts with the output cleared, the round trip
through ``save_serialized_speech`` and signal references, the serialize-only call (no tracks), resident chains and
the refusals."""
import contextlib
import os
import tempfile

import numpy as np
import pytest

import test_gpu_reference_exact as rx
import test_gpu_seg_ref as sr

pytestmark = pytest.mark.gpu

LABELS = rx.LABELS


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@contextlib.contextmanager
def _output(handle, videos, capacity, memspace):
    """The handle's speech output over `videos`, NaN-prefilled: yields dict(buf, off) (numpy once the block exits)."""
    import torch
    from ffsubsync_b200 import _native as N
    off = np.full(len(videos) + 1, -1, np.int64)
    if memspace == N.B2_HOST:
        buf = np.full(capacity + 64, np.nan)
        ptr = buf
    else:
        buf = torch.full((capacity + 64,), float("nan"), dtype=torch.float64, device="cuda")
        torch.cuda.synchronize()
        ptr = buf.data_ptr()
    handle.speech_output(ptr, capacity, videos, off, N.B2_HOST if memspace == N.B2_HOST else N.B2_DEVICE)
    out = {}
    try:
        yield out
    finally:
        handle.speech_output(None, 0, None, None)
        handle.synchronize()
        out.update(buf=buf if isinstance(buf, np.ndarray) else buf.cpu().numpy(), off=off)


def _unpack(cap, v, R, low):
    """Video v of a capture_reference dict, widened: floats, or its packed bits as 1.0 / low."""
    a = int(cap["ref_off"][v])
    if cap["packed"][v]:
        words = cap["ref"].view(np.uint32)[a: a + -(-R // 32)]
        bits = (words[:, None] >> np.arange(32, dtype=np.uint32)) & 1
        return np.where(bits.ravel()[:R] == 1, 1.0, np.float64(np.float32(low)))
    return cap["ref"][a: a + R].astype(np.float64)


def _check(out, want, videos, cap=None, lows=None, where=""):
    """want: per-video float32 oracle of every video of the call; videos: the listed ones."""
    buf, off = out["buf"], out["off"]
    lens = [len(want[v]) for v in videos]
    assert off.tolist() == np.concatenate([[0], np.cumsum(lens)]).astype(int).tolist(), (where, off, lens)
    for i, v in enumerate(videos):
        got = buf[off[i]: off[i + 1]]
        exp = np.asarray(want[v], np.float32).astype(np.float64)
        bad = np.flatnonzero(got != exp)
        assert len(bad) == 0, (where, "video", v, bad[:8].tolist(), got[bad[:8]].tolist(), exp[bad[:8]].tolist())
        if cap is not None:
            assert np.array_equal(got, _unpack(cap, v, lens[i], lows[v])), (where, "capture", v)
    assert np.isnan(buf[off[-1]:]).all(), (where, "written past speech_off[n]")


def _lows(c, label):
    return [0.0 if d["kind"] in ("subs", "pgs") else label for d in c["videos"]]


def _run(handle, c, entry, label, memspace, videos, detector="energy"):
    """One rx._call with the output and the reference capture set: (output, capture, results)."""
    want = rx._oracle(c, "auditok" if entry == "auditok" or detector == "auditok" else "energy", label)
    cap_n = rx._capacity(want)
    res = None
    with handle.capture_reference(cap_n, len(want) + 3) as cap:
        with _output(handle, videos, cap_n, memspace) as out:
            keep = []
            res = rx._call(handle, c, entry, label, memspace, keep=keep, detector=detector)
            handle.synchronize()
    return want, out, cap, res


@pytest.mark.parametrize("memspace", ["host", "device", "resident"])
@pytest.mark.parametrize("entry", rx.ENTRIES)
def test_entry_points_and_memory(handle, entry, memspace):
    from ffsubsync_b200 import _native as N
    ms = {"host": N.B2_HOST, "device": N.B2_DEVICE, "resident": N.B2_DEVICE_RESIDENT}[memspace]
    c = rx._mixed_corpus(entry == "pgs") if entry in ("subs", "pgs") else rx._corpus(rx._win_videos(160, rx.LENGTHS), 16000, 1)
    V = len(c["videos"])
    for label in (0.0, 0.3):
        for videos in (list(range(V)), [1, 3, 4, V - 1]):
            want, out, cap, _ = _run(handle, c, entry, label, ms, videos)
            _check(out, want, videos, cap, _lows(c, label), (entry, memspace, label, videos))


@pytest.mark.parametrize("env", [{}, {"B2_ALIGN_PATH": "runs"}, {"B2_REF_PACKED": "0"}, {"B2_VAD_LAYOUT": "group"},
                                 {"B2_SUBBATCHES": "1"}, {"B2_SUBBATCHES": "3"}])
@pytest.mark.parametrize("label", LABELS)
def test_labels_and_knobs(handle, label, env):
    from ffsubsync_b200 import _native as N
    energy = rx._corpus(rx._win_videos(160, rx.LENGTHS, tracks=1), 16000, 1)
    mixed = rx._mixed_corpus(True)
    with rx._env(**env):
        for entry, c in (("tracks", energy), ("auditok", energy), ("pgs", mixed)):
            for ms in (N.B2_HOST, N.B2_DEVICE):
                videos = list(range(len(c["videos"])))
                want, out, cap, _ = _run(handle, c, entry, label, ms, videos)
                _check(out, want, videos, cap, _lows(c, label), (entry, ms, label, env))


def _sig_call(handle, x, sig_off, label, memspace, packed_env):
    """Two signal videos around an audio video through b2_sync_tracks_sig."""
    from ffsubsync_b200 import _native as N
    c = rx._corpus(rx._win_videos(160, [(0, 0), (32 * 30 + 7, 0), (0, 0)]), 16000, 3)
    is_sig = np.array([1, 0, 1], np.uint8)
    want = [np.where(x[sig_off[0]:sig_off[1]] < 1.0, np.float64(label), x[sig_off[0]:sig_off[1]]).astype(np.float32),
            rx._oracle(c, "energy", label)[1],
            np.where(x[sig_off[1]:sig_off[2]] < 1.0, np.float64(label), x[sig_off[1]:sig_off[2]]).astype(np.float32)]
    voff = np.array([sig_off[0], sig_off[1], sig_off[1], sig_off[2]], np.int64)
    import torch
    with rx._env(**packed_env):
        with handle.capture_reference(rx._capacity(want), 6) as cap:
            with _output(handle, [0, 1, 2], rx._capacity(want), memspace) as out:
                xt = x if memspace == N.B2_HOST else torch.from_numpy(x).cuda()
                pcm = c["pcm"] if memspace == N.B2_HOST else torch.from_numpy(c["pcm"]).cuda()
                outs = {}
                if memspace != N.B2_HOST:
                    t = {k: torch.empty(len(c["tv"]), dtype=dt, device="cuda") for k, dt in
                         (("best_score", torch.float64), ("best_offset", torch.int32), ("best_k", torch.int32))}
                    outs = {k: v.data_ptr() for k, v in t.items()}
                torch.cuda.synchronize()
                handle.sync_tracks_sig(pcm if memspace == N.B2_HOST else pcm.data_ptr(), c["pcm_off"], c["tv"], 16000,
                                       100, label, is_sig, xt if memspace == N.B2_HOST else xt.data_ptr(), voff,
                                       c["cs"], c["ce"], None, c["cue_off"], rx.GRID, 0.0, rx.MOS,
                                       energy_threshold=rx.THR, memspace=memspace, **outs)
                handle.synchronize()
    return want, out, cap


@pytest.mark.parametrize("packed_env", [{"B2_ALIGN_PATH": "runs"}, {"B2_REF_PACKED": "0"}])
@pytest.mark.parametrize("label", LABELS)
def test_signal_videos(handle, label, packed_env):
    from ffsubsync_b200 import _native as N
    rng = np.random.RandomState(4)
    a = np.where(rng.rand(2000) < 0.4, 1.0, rng.rand(2000) * 0.999)
    b = np.where(rng.rand(777) < 0.5, 1.0, -rng.rand(777))
    x = np.concatenate([a, b])
    for ms in (N.B2_HOST, N.B2_DEVICE):
        want, out, cap = _sig_call(handle, x, [0, 2000, 2777], label, ms, packed_env)
        _check(out, want, [0, 1, 2], cap, [label] * 3, ("sig", label, ms, packed_env))


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
def test_segment_videos(handle, det):
    c = sr._corpus([(200.0, "seg"), (30.0, "audio"), (150.0, "seg")], count=3, dur=20, tracks=1)
    bs = sr._sync(c, det=det)
    r = bs.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                            speech_video=[0, 1, 2], **c["tab"])
    speech, off = r[-2], r[-1]
    ref, ref_off = bs._reference_signals(c["pcm"], c["pcm_off"], seg=bs._seg_refs(3, dict(c["tab"])))
    for i, v in enumerate([0, 1, 2]):
        exp = ref[ref_off[v]: ref_off[v + 1]].astype(np.float64)
        if v != 1:
            exp2 = np.asarray(sr._oracle_ref(c, v, det, 0.0), np.float64).astype(np.float32).astype(np.float64)
            assert np.array_equal(exp, exp2), v
        assert np.array_equal(speech[off[i]: off[i + 1]], exp), (det, v)
    d = bs.sync_device_tracks(__import__("torch").from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"],
                              c["cue_start"], c["cue_end"], c["cue_off"], speech_video=[0, 2], **c["tab"])
    bs.handle.synchronize()
    got = d["speech"].cpu().numpy()
    assert np.array_equal(got, np.concatenate([speech[off[0]:off[1]], speech[off[2]:off[3]]]))


def test_results_and_launches_unchanged(handle):
    """best_* / all_* / gss_* bit-identical with and without the output; with it cleared, the launch count deltas of
    a handle that never set it."""
    import torch
    from ffsubsync_b200 import _native as N
    c = rx._mixed_corpus(True)
    fresh = N.Handle(torch.cuda.current_device())
    try:
        for entry in ("tracks", "gss", "auditok", "pgs"):
            base = rx._call(handle, c, entry, 0.0, N.B2_HOST)
            with _output(handle, list(range(len(c["videos"]))), 10_000_000, N.B2_HOST):
                got = rx._call(handle, c, entry, 0.0, N.B2_HOST)
            for a, b in zip(base, got):
                if a is not None:
                    assert np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True), entry
            n0 = handle.launch_count
            rx._call(handle, c, entry, 0.0, N.B2_HOST)
            n1 = fresh.launch_count
            rx._call(fresh, c, entry, 0.0, N.B2_HOST)
            assert handle.launch_count - n0 == fresh.launch_count - n1, entry
    finally:
        fresh.close()


def test_round_trip(handle):
    """Sync audio, text, PGS and segment videos with speech_video, save, load with stored=True, sync the same tracks
    against the signals: the same results (detector videos at every label, the others at label 0)."""
    from ffsubsync_b200.batch import BatchSynchronizer, load_serialized_speech, save_serialized_speech
    c = sr._corpus([(120.0, "audio"), (150.0, "seg"), (90.0, "audio")], count=3, dur=20, tracks=2)
    # video 0 takes a text stream, video 2 a PGS list; their PCM is dropped
    st, en = rx.cases.synthetic_cues(11, 90.0)
    pcm_off = c["pcm_off"].copy()
    keep = np.ones(len(c["pcm"]), bool)
    keep[pcm_off[0]:pcm_off[1]] = False
    keep[pcm_off[2]:pcm_off[3]] = False
    lens = np.diff(pcm_off) * np.array([0, 1, 0])
    new_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    tab = dict(c["tab"])   # segment ranges are relative to the video's range: unchanged
    pcm = c["pcm"][keep]
    streams = dict(ref_cue_start=st, ref_cue_end=en, ref_cue_off=[0, len(st)], ref_stream_video=[0],
                   pgs_start=st[::2] + 0.004, pgs_end=en[::2] + 0.006, pgs_off=[0, len(st[::2])], pgs_video=[2])
    args = (c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])
    for label in (0.0,):
        bs = BatchSynchronizer([1.0, 25 / 24.0], non_speech_label=label, vad="subs_then_energy_zcr",
                               max_offset_seconds=30.0)
        r = bs.sync_host_tracks(pcm, new_off, *args, want_all=True, speech_video=[0, 1, 2], **tab, **streams)
        speech, off = r[-2], r[-1]
        with tempfile.TemporaryDirectory() as d:
            paths = [os.path.join(d, "v%d.npz" % v) for v in range(3)]
            save_serialized_speech(paths, speech, off)
            x, x_off = load_serialized_speech(paths, stored=True)
        assert np.array_equal(x, speech[: off[-1]])
        plain = BatchSynchronizer([1.0, 25 / 24.0], non_speech_label=label, max_offset_seconds=30.0)
        r2 = plain.sync_host_tracks(None, np.zeros(4, np.int64), *args, want_all=True, sig=x, sig_off=x_off,
                                    sig_video=[0, 1, 2])
        for a, b in zip(r[:5], r2[:5]):
            assert np.array_equal(a, b), label
    # detector videos at every label: an audio-only corpus
    a = sr._corpus([(100.0, "audio"), (70.0, "audio")], tracks=2)
    for label in LABELS:
        bs = BatchSynchronizer([1.0, 25 / 24.0], non_speech_label=label, max_offset_seconds=30.0)
        r = bs.sync_host_tracks(a["pcm"], a["pcm_off"], a["track_video"], a["cue_start"], a["cue_end"], a["cue_off"],
                                want_all=True, speech_video=[0, 1])
        with tempfile.TemporaryDirectory() as d:
            paths = [os.path.join(d, "v%d.npz" % v) for v in range(2)]
            save_serialized_speech(paths, r[-2], r[-1])
            x, x_off = load_serialized_speech(paths, stored=True)
        r2 = bs.sync_host_tracks(None, np.zeros(3, np.int64), a["track_video"], a["cue_start"], a["cue_end"],
                                 a["cue_off"], want_all=True, sig=x, sig_off=x_off, sig_video=[0, 1])
        for p, q in zip(r[:5], r2[:5]):
            assert np.array_equal(p, q), label


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
def test_serialize_only(handle, det):
    """No tracks: the listed videos' detector output (b2_vad_energy_zcr / b2_vad_auditok rounded to float32) and
    nothing else."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    c = rx._corpus(rx._win_videos(160, rx.LENGTHS), 16000, 2)
    bs = BatchSynchronizer([1.0], vad=det)
    videos = [0, 2, 3, 6, 9]
    empty = dict(track_video=np.zeros(0, np.int32), cue_start=np.zeros(0), cue_end=np.zeros(0),
                 cue_off=np.zeros(1, np.int64))
    r = bs.sync_host_tracks(c["pcm"], c["pcm_off"], *empty.values(), speech_video=videos)
    if det == "auditok":
        d, d_off = bs._vad_auditok_device(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"])
        d = d.cpu().numpy()
    else:
        d, d_off = bs.handle.vad_energy_zcr(c["pcm"], c["pcm_off"], 16000, 100, 0.0, bs.energy_threshold)
    exp = np.concatenate([d[d_off[v]: d_off[v + 1]] for v in videos]).astype(np.float32).astype(np.float64)
    assert len(r[0]) == 0 and np.array_equal(r[-2], exp) and r[-1][-1] == len(exp)
    n0 = bs.handle.launch_count
    out = bs.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], *empty.values(), speech_video=videos)
    bs.handle.synchronize()
    assert np.array_equal(out["speech"].cpu().numpy(), exp)
    assert bs.handle.launch_count - n0 >= 1
    n0 = bs.handle.launch_count   # without the output a call without tracks launches nothing
    bs.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], *empty.values())
    assert bs.handle.launch_count == n0


def test_resident_chain(capfd):
    """Resident calls alternating with and without the output give the unchained results; setting or clearing the
    output between two resident calls leaves the chain in place (B2_PIPE_TRACE reports chained=1)."""
    import torch
    from ffsubsync_b200 import _native as N
    a, b, c, d = _chain_corpora()
    seq = list(zip((a, b, c, d), ["tracks", "batch", "tracks", "batch"]))
    handle = N.Handle(torch.cuda.current_device())
    try:
        plain = [rx._call(handle, x, e, 0.0, N.B2_HOST, want_all=False) for x, e in seq]
        wants = [rx._oracle(x, "energy", 0.0) for x, _ in seq]
        devs = [rx._device_args(x, e) for x, e in seq]
        bufs = [torch.full((rx._capacity(w),), float("nan"), dtype=torch.float64, device="cuda") for w in wants]
        offs = [np.zeros(len(w) + 1, np.int64) for w in wants]
        torch.cuda.synchronize()
        with rx._env(B2_SUBBATCHES=2, B2_ALIGN_PATH="runs"):
            for (x, e), dev in zip(seq, devs):   # grow every workspace
                rx._call(handle, x, e, 0.0, N.B2_DEVICE_RESIDENT, dev=dev)
            handle.synchronize()
            capfd.readouterr()
            with rx._env(B2_PIPE_TRACE=1):
                for i, ((x, e), dev) in enumerate(zip(seq, devs)):
                    if i % 2 == 0:
                        handle.speech_output(bufs[i].data_ptr(), rx._capacity(wants[i]),
                                             list(range(len(wants[i]))), offs[i], N.B2_DEVICE)
                    else:
                        handle.speech_output(None, 0, None, None)
                    rx._call(handle, x, e, 0.0, N.B2_DEVICE_RESIDENT, dev=dev)
            handle.speech_output(None, 0, None, None)
            handle.synchronize()
        err = capfd.readouterr().err
        lines = [ln for ln in err.splitlines() if ln.startswith("[b2 pipe] V=")]
        assert len(lines) == 4 and all("chained=1" in ln for ln in lines), err
        for i, ((x, e), dev) in enumerate(zip(seq, devs)):
            t = dev[2][1]
            got = (t["best_score"].cpu().numpy(), t["best_offset"].cpu().numpy(), t["best_k"].cpu().numpy())
            for p, q in zip(plain[i][:3], got):
                assert np.array_equal(p, q), (i, e)
            if i % 2 == 0:
                _check(dict(buf=bufs[i].cpu().numpy(), off=offs[i]), wants[i], list(range(len(wants[i]))),
                       where=("chain", i))
    finally:
        handle.close()
        torch.cuda.synchronize()


def _chain_corpora():
    return (rx._corpus(rx._win_videos(160, [(30000, 0), (12345, 40), (32 * 500 + 1, 0), (31, 0)], tracks=2), 16000, 71),
            rx._corpus(rx._win_videos(160, [(20000 + 32, 0), (0, 0), (32 * 300 + 31, 8), (25000, 0), (7, 0)]), 16000,
                       72),
            rx._corpus(rx._win_videos(160, [(28001, 8), (32 * 400, 0), (5, 0)], tracks=3), 16000, 73),
            rx._corpus(rx._win_videos(160, [(32 * 700 + 31, 0), (31000, 40), (0, 0), (19, 0)]), 16000, 74))


def test_refusals_then_a_good_call(handle):
    import torch
    from ffsubsync_b200 import _native as N
    c = rx._corpus(rx._win_videos(160, rx.LENGTHS[:4]), 16000, 6)
    want = rx._oracle(c, "energy", 0.0)
    total = sum(len(w) for w in want)
    dev_buf = torch.empty(total + 8, dtype=torch.float64, device="cuda")
    off = np.zeros(5, np.int64)
    for cap, videos, memspace, msg in ((total - 1, [0, 1, 2, 3], N.B2_HOST, "need %d" % total),
                                       (total, [0, 1, 2, 7], N.B2_HOST, "lists video 7")):
        buf = np.full(total + 8, np.nan)
        handle.speech_output(buf, cap, videos, off, memspace)
        n0 = handle.launch_count
        with pytest.raises(N.NativeError, match=msg):
            rx._call(handle, c, "tracks", 0.0, N.B2_HOST)
        assert handle.launch_count == n0 and np.isnan(buf).all()
        handle.speech_output(None, 0, None, None)
    with pytest.raises(N.NativeError, match="not increasing"):
        handle.speech_output(dev_buf.data_ptr(), total, [2, 1], off, N.B2_DEVICE)
    with pytest.raises(N.NativeError, match="host pointer"):
        handle.speech_output(np.zeros(total), total, [0, 1], off, N.B2_DEVICE)
    with _output(handle, [0, 1, 2, 3], total, N.B2_HOST) as out:
        rx._call(handle, c, "tracks", 0.0, N.B2_HOST)
    _check(out, want, [0, 1, 2, 3])


def test_flagged_videos_are_written(handle):
    """A signal video with a value > 1 (best_k -2) and a segment video without speech (-3) still get their frames;
    save_serialized_speech refuses the -3 video."""
    import torch
    from ffsubsync_b200 import _native as N
    from ffsubsync_b200.batch import save_serialized_speech
    x = np.array([0.5, 1.0, 2.0, 0.1] * 50)
    for env, packed in (({"B2_REF_PACKED": "0"}, 0), ({"B2_ALIGN_PATH": "runs"}, 1)):
        want, out, cap = _sig_call(handle, x, [0, 100, 200], 0.3, N.B2_DEVICE, env)
        assert cap["packed"][0] == packed
        # the frames the call built: sig_ref_kernel writes an out-of-domain value as the label
        want = [np.where(x[:100] == 1.0, np.float32(1.0), np.float32(0.3)), want[1],
                np.where(x[100:200] == 1.0, np.float32(1.0), np.float32(0.3))]
        _check(out, want, [0, 1, 2], cap, [0.3] * 3, ("bad signal", env))
    c = sr._corpus([(100.0, "silent"), (40.0, "audio")], count=2, dur=20, tracks=1)
    bs = sr._sync(c)
    o = bs.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"], c["cue_start"],
                              c["cue_end"], c["cue_off"], speech_video=[0, 1], **c["tab"])
    bs.handle.synchronize()
    bk = o["best_k"].cpu().numpy()
    assert bk[0] == N.B2_BEST_K_NO_SPEECH
    sp = o["speech"].cpu().numpy()
    assert o["speech_off"][1] == int(100.0 * 100) + 2 and not np.isnan(sp).any()
    with tempfile.TemporaryDirectory() as d:
        with pytest.raises(ValueError, match="Unable to detect speech"):
            save_serialized_speech([os.path.join(d, "a.npz"), os.path.join(d, "b.npz")], o["speech"], o["speech_off"],
                                   speech_video=[0, 1], seg_video=c["seg_v"])
        assert not os.listdir(d)


def test_refused_methods(handle):
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    bs = BatchSynchronizer([1.0])
    with pytest.raises(ValueError, match="speech_video"):
        bs.sync_signals(np.zeros(10, np.float32), [0, 10], [1.0], [2.0], [0, 1], speech_video=[0])
    with pytest.raises(ValueError, match="speech_video"):
        bs.sync_device_candidate_sharded(torch.zeros(1600, dtype=torch.int16, device="cuda"), [0, 1600], [1.0], [2.0],
                                         [0, 1], speech_video=[0])


def test_save_orders_itself_after_a_device_call(handle):
    """save_serialized_speech right after a device call that returned without synchronising: the handle runs on a
    stream of its own held back by a sleep, and the files still hold the complete signals."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer, load_serialized_speech, save_serialized_speech
    c = rx._corpus(rx._win_videos(160, rx.LENGTHS), 16000, 8)
    bs = BatchSynchronizer([1.0])
    empty = (np.zeros(0, np.int32), np.zeros(0), np.zeros(0), np.zeros(1, np.int64))
    videos = np.arange(len(rx.LENGTHS))
    want = bs.sync_host_tracks(c["pcm"], c["pcm_off"], *empty, speech_video=videos)
    pcm = torch.from_numpy(c["pcm"]).cuda()
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    bs.handle.set_stream(stream.cuda_stream)
    try:
        with torch.cuda.stream(stream):
            torch.cuda._sleep(200_000_000)   # about 0.1 s ahead of the call on the handle's stream
        out = bs.sync_device_tracks(pcm, c["pcm_off"], *empty, speech_video=videos)
        with tempfile.TemporaryDirectory() as d:
            paths = [os.path.join(d, "v%d.npz" % v) for v in videos]
            save_serialized_speech(paths, out["speech"], out["speech_off"])
            x, x_off = load_serialized_speech(paths, stored=True)
    finally:
        torch.cuda.synchronize()
        bs.handle.set_stream(None)
    assert np.array_equal(x_off, want[-1]) and np.array_equal(x, want[-2][: want[-1][-1]])


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
def test_serialize_only_segments_on_the_host(handle, det):
    """No tracks, B2_HOST, a subset of audio and segment videos: only their samples are staged, and their signals
    equal the composition of public steps; a segment video without speech is refused by save_serialized_speech."""
    from ffsubsync_b200.batch import save_serialized_speech
    c = sr._corpus([(200.0, "seg"), (30.0, "audio"), (150.0, "silent"), (45.0, "audio"), (120.0, "seg")], count=3,
                   dur=20, tracks=1)
    bs = sr._sync(c, det=det)
    empty = (np.zeros(0, np.int32), np.zeros(0), np.zeros(0), np.zeros(1, np.int64))
    ref, ref_off = bs._reference_signals(c["pcm"], c["pcm_off"], seg=bs._seg_refs(5, dict(c["tab"])))
    for videos in ([0, 1, 2, 3, 4], [1, 2], [4], []):
        r = bs.sync_host_tracks(c["pcm"], c["pcm_off"], *empty, speech_video=videos, **c["tab"])
        assert len(r[0]) == 0
        speech, off = r[-2], r[-1]
        exp = [ref[ref_off[v]: ref_off[v + 1]].astype(np.float64) for v in videos]
        assert off.tolist() == np.concatenate([[0], np.cumsum([len(e) for e in exp])]).astype(int).tolist()
        for i, e in enumerate(exp):
            assert np.array_equal(speech[off[i]: off[i + 1]], e), (det, videos, i)
        with tempfile.TemporaryDirectory() as d:
            paths = [os.path.join(d, "v%d.npz" % v) for v in videos]
            if 2 in videos:
                with pytest.raises(ValueError, match="video 2: Unable to detect speech"):
                    save_serialized_speech(paths, speech, off, speech_video=videos, seg_video=c["seg_v"])
                assert not os.listdir(d)
            else:
                save_serialized_speech(paths, speech, off, speech_video=videos, seg_video=c["seg_v"])
