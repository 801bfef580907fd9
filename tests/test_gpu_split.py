"""GPU tests of the per-segment offsets (b2_split_tracks, b2_apply_split; run on an H100).

Yardstick: oracle/split_oracle.py.  Every cue offset, segment count and split score must equal the oracle's bit for
bit on seeded two-level references, in both memspaces; with an infinite penalty every cue takes the sync call's own
offset and apply_split writes what apply_sync writes; planted cuts are found exactly; and the envelope is refused."""
import math

import numpy as np
import pytest

from oracle import raster_oracle as ro
from oracle import split_oracle as sp
from test_gpu_sig_ref import _sig_corpus
from test_gpu_sync_output import _streams

pytestmark = pytest.mark.gpu

GRID = [1.0, 25 / 24.0, 24 / 25.0]


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _cues(rng, n, dur):
    t = np.sort(rng.uniform(0, dur, n))
    cs = np.round(t, 3)
    ce = np.round(cs + rng.uniform(0.01, 3.0, n), 3)
    return cs, ce


def _request(seed, V=3, T=6, R=3000, label=0.0, f64=True):
    """Two-level references (1.0 and label) built from cue lists with random shifts, and T tracks of cues."""
    rng = np.random.RandomState(seed)
    refs = []
    for v in range(V):
        L = R + 97 * v
        cs, ce = _cues(rng, 40, L / 100.0)
        m = ro.rasterize(cs, ce, None, 100, 0, 1.0)[0][:L] > 0
        refs.append(np.where(m, 1.0, label))
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.int64)
    ref = np.concatenate(refs).astype(np.float64 if f64 else np.float32)
    tv = np.sort(rng.randint(0, V, T)).astype(np.int32)
    cs, ce, off = [], [], [0]
    for t in range(T):
        n = int(rng.randint(0, 30))
        a, b = _cues(rng, n, R / 100.0)
        cs.append(a)
        ce.append(b)
        off.append(off[-1] + n)
    cs, ce = np.concatenate(cs), np.concatenate(ce)
    keep = (rng.rand(len(cs)) > 0.15).astype(np.uint8)
    ratio = np.array([GRID[int(rng.randint(0, 3))] for _ in range(T)])
    ratio[rng.rand(T) < 0.2] = np.nan
    return ref, ref_off, tv, cs, ce, keep, np.array(off, np.int64), ratio


@pytest.mark.parametrize("seed", range(6))
def test_split_equals_oracle(handle, seed):
    import torch
    from ffsubsync_b200 import _native
    label = [0.0, 0.3, -0.5][seed % 3]
    mos = [None, 300, 40, 0][seed % 4] if seed % 3 == 0 else [500, 40, 3][seed % 3]
    f64 = seed % 2 == 0
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed, R=1200 + 400 * (seed % 3), label=label, f64=f64)
    for pen in (0.0, 3.0, 25.5, math.inf):
        want = sp.split_tracks(ref.astype(np.float64), ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen)
        got = handle.split_tracks(ref, f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen)
        for w, g, name in zip(want, got, ("cue_offset", "n_segments", "split_score")):
            assert np.array_equal(w, g, equal_nan=True), (seed, pen, name, w, g)
        d_ref = torch.from_numpy(ref).cuda()
        outs = [torch.full((max(len(cs), 1),), 7, dtype=torch.int32, device="cuda"),
                torch.full((len(tv),), 7, dtype=torch.int32, device="cuda"),
                torch.zeros(len(tv), dtype=torch.float64, device="cuda")]
        handle.split_tracks(d_ref.data_ptr(), f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen,
                            outs=[o.data_ptr() for o in outs], memspace=_native.B2_DEVICE)
        handle.synchronize()
        for w, g in zip(want, outs):
            assert np.array_equal(w, g.cpu().numpy()[: len(w)], equal_nan=True), (seed, pen)


@pytest.mark.parametrize("vad,gss", [("energy_zcr", False), ("energy_zcr", True), ("auditok", False)])
def test_no_splits_is_the_sync_call(vad, gss):
    """split_penalty = inf: one segment per track; on +-1 tracks (label 0, ratio <= 1) every cue gets the call's
    best_offset and split_score == best_score bit for bit, elsewhere the score is within the run path's margin; and
    apply_split writes what apply_sync writes wherever the offsets agree."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    rng = np.random.RandomState(11)
    c = _sig_corpus([(60.0 + 3 * v, "audio", [(GRID[int(rng.randint(0, 3))], int(rng.randint(-700, 700)))
                                              for _ in range(1 + v % 2)]) for v in range(5)], seed0=7)
    s = BatchSynchronizer(GRID + ([None] if gss else []), vad=vad, non_speech_label=0.0)
    V = len(c["pcm_off"]) - 1
    sv = np.arange(V)
    host = s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                              speech_video=sv)
    spl = s.split_tracks_host(host, c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"], split_penalty=math.inf)
    want = s.apply_sync_host(host[:-2], c["cue_start"], c["cue_end"], c["cue_off"])   # without (speech, speech_off)
    got = s.apply_split_host(spl, c["cue_start"], c["cue_end"], c["cue_off"])
    _check_no_splits(spl, want, got, *host[:3], c["cue_off"])
    # the same from the device call, without a synchronisation between the steps
    out = s.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"], c["cue_start"],
                               c["cue_end"], c["cue_off"], speech_video=sv)
    d = s.split_tracks(out, c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"], split_penalty=math.inf)
    a = s.apply_split(d, c["cue_start"], c["cue_end"], c["cue_off"])
    w = s.apply_sync(out, c["cue_start"], c["cue_end"], c["cue_off"])
    torch.cuda.synchronize()
    d = {k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in d.items()}
    _check_no_splits(d, {k: v.cpu().numpy() for k, v in w.items()}, {k: v.cpu().numpy() for k, v in a.items()},
                     *[out[k].cpu().numpy() for k in ("best_score", "best_offset", "best_k")], c["cue_off"])


def _check_no_splits(spl, want, got, bs, bo, bk, off):
    pm1 = spl["ratio"] <= 1.0   # level 1 against 1.0 / 0.0: every count is an exact integer
    same = np.zeros(len(bk), bool)
    for t in range(len(bk)):
        if bk[t] < 0:
            assert spl["n_segments"][t] == 0 and np.isnan(spl["split_score"][t])
            continue
        assert spl["n_segments"][t] == 1
        same[t] = np.all(spl["cue_offset"][off[t]: off[t + 1]] == bo[t])
        if pm1[t]:
            assert same[t], t
            assert spl["split_score"][t] == bs[t], (t, spl["split_score"][t], bs[t])
        else:   # exact ties are decided on the re-score's float64 sums there: the score within the run path's margin
            assert abs(spl["split_score"][t] - bs[t]) <= 1e-9 * max(1.0, abs(bs[t])), (t, spl["split_score"][t], bs[t])
    assert same.any()
    cues = np.repeat(same, np.diff(off))
    for k in ("synced_start_us", "synced_end_us"):
        assert np.array_equal(want[k][cues], got[k][cues])


# (d1, d2, penalties): 90 s and 30 s the subtitles do not have (the video's ad break: d2 > d1) over 2 .. 3000, and 90 s
# of subtitles the video does not have (a removal: d2 < d1) over 1000 .. 3000; below that range the removal splits on
# the cues that lose their counterpart, above it the penalty outweighs the second half
CUTS = [(300, 9300, (2.0, 10.0, 50.0, 3000.0)), (300, 3300, (2.0, 10.0, 50.0, 3000.0)),
        (9300, 300, (1000.0, 2000.0, 3000.0))]


@pytest.mark.parametrize("d1,d2,penalties", CUTS)
def test_planted_cut(handle, d1, d2, penalties):
    """A break before cue 40: the reference is the track's own cues shifted by d1 before that cue and by d2 from it
    on.  Over the stated penalties the split finds both offsets exactly, with the break at the planted cue, and equals
    the oracle."""
    rng = np.random.RandomState(4)
    n, cut = 80, 40
    gaps = rng.uniform(1.0, 6.0, n)
    cs = np.round(30 + np.cumsum(gaps), 2)
    ce = np.round(cs + rng.uniform(0.5, 3.0, n), 2)
    m = ro.rasterize(cs, ce, None, 100, 0, 1.0)[0] > 0
    R = len(m) + 9400
    ref = np.zeros(R)
    f = np.arange(len(m))
    for lo, hi, d in ((0, int(round(cs[cut] * 100)), d1), (int(round(cs[cut] * 100)), len(m), d2)):
        g = f[lo:hi][m[lo:hi]] + d
        g = g[(g >= 0) & (g < R)]
        ref[g] = 1.0
    off = np.array([0, n], np.int64)
    for pen in penalties:
        co, ns, sc = handle.split_tracks(ref, True, np.array([0, R]), [0], cs, ce, None, off, [1.0], 100, 0.0, 9500,
                                         pen)
        assert ns[0] == 2, (pen, ns)
        assert np.all(co[:cut] == d1) and np.all(co[cut:] == d2), (pen, co)
    want = sp.split_tracks(ref, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 9500, penalties[-1])
    for w, g in zip(want, (co, ns, sc)):
        assert np.array_equal(w, g, equal_nan=True)


def test_refusals(handle):
    from ffsubsync_b200._native import NativeError
    cs, ce = np.array([1.0, 5.0]), np.array([2.0, 6.0])
    off = np.array([0, 2], np.int64)
    ref = np.zeros(1000)
    ref[10:20] = 1.0
    bad = ref.copy()
    bad[123] = 0.5
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*video 0: frame 123"):
        handle.split_tracks(bad, True, [0, 1000], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0)
    assert handle.launch_count == n0 + 1   # the level scan that found the third level, nothing after it
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*32770 offsets is wider than 32768"):
        handle.split_tracks(np.zeros(40000), True, [0, 40000], [0], [1.0, 200.0], [2.0, 201.0], None, off, [1.0], 100,
                            0.0, 16385, 1.0)
    n = 16385
    many_s = np.arange(n) * 0.03
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*16385 kept cues.*16384 runs"):
        handle.split_tracks(ref, True, [0, 1000], [0], many_s, many_s + 0.01, None, [0, n], [1.0], 100, 0.0, 100, 1.0)
    with pytest.raises(NativeError, match=r"B2_ERR_BAD_ARG.*split_penalty nan"):
        handle.split_tracks(ref, True, [0, 1000], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, math.nan)
    with pytest.raises(NativeError, match=r"B2_ERR_BAD_ARG.*ratio inf"):
        handle.split_tracks(ref, True, [0, 1000], [0], cs, ce, None, off, [math.inf], 100, 0.0, 100, 1.0)
    with pytest.raises(NativeError, match=r"B2_ERR_BAD_ARG.*video 3 is outside"):
        handle.split_tracks(ref, True, [0, 1000], [3], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0)
    assert handle.launch_count == n0   # the other refusals come before any launch


def test_window_and_run_limits(handle):
    """16384 one-frame runs at frame 0 .. S-1 in a 32768-offset window (the 1024-thread CTA) run, and in a narrow
    window equal the oracle."""
    rng = np.random.RandomState(2)
    n = 16384
    cs = np.arange(n) * 0.02
    ce = cs + 0.01
    R = 40000
    ref = (rng.rand(R) < 0.5).astype(np.float64)
    off = np.array([0, n], np.int64)
    for mos in (16384, 40):
        for pen in (0.0, 2.0):
            got = handle.split_tracks(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen)
            if mos == 40:
                want = sp.split_tracks(ref, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen)
                for w, g in zip(want, got):
                    assert np.array_equal(w, g, equal_nan=True), (mos, pen)
            assert got[1][0] >= 1


@pytest.mark.parametrize("label", [0.0, 0.3])
def test_widest_window_equals_oracle(handle, label):
    """The 32768-offset window (split_dp_kernel's 1024-thread instantiation, 32 warps in the unit reduction) against
    the oracle on a few runs, at label 0 and 0.3."""
    rng = np.random.RandomState(9)
    R = 40000
    ref = np.where(rng.rand(R) < 0.4, 1.0, label)
    cs = np.array([10.0, 60.0, 120.5, 170.25, 200.0])
    ce = cs + np.array([3.0, 1.5, 7.0, 0.5, 2.0])
    off = np.array([0, 5], np.int64)
    for pen in (0.0, 5.0):
        want = sp.split_tracks(ref, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 16384, pen)
        got = handle.split_tracks(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 16384, pen)
        for w, g in zip(want, got):
            assert np.array_equal(w, g, equal_nan=True), (label, pen, w, g)


def test_absolute_cue_indices(handle):
    """A cue table that starts past 0 (cue_off[0] = 5): cue_offset is indexed by absolute cue in both memspaces,
    equals the oracle, and the entries outside [cue_off[0], cue_off[T]) are left as they were."""
    import torch
    from ffsubsync_b200 import _native
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(21, R=1500, label=0.3)
    pad = 5
    cs, ce = np.concatenate([np.full(pad, 1.0), cs]), np.concatenate([np.full(pad, 2.0), ce])
    keep = np.concatenate([np.ones(pad, np.uint8), keep])
    off = off + pad
    for pen in (0.0, 4.0):
        want = sp.split_tracks(ref, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, 300, pen)
        got = handle.split_tracks(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, 300, pen)
        for w, g in zip(want, got):
            assert np.array_equal(w, g, equal_nan=True), pen
        guard, n = 16, int(off[-1])
        buf = torch.full((guard + n + guard,), -12345, dtype=torch.int32, device="cuda")
        ns = torch.full((len(tv) + 2 * guard,), -12345, dtype=torch.int32, device="cuda")
        sc = torch.full((len(tv) + 2 * guard,), -1.5, dtype=torch.float64, device="cuda")
        outs = [buf.data_ptr() + 4 * guard, ns.data_ptr() + 4 * guard, sc.data_ptr() + 8 * guard]
        handle.split_tracks(torch.from_numpy(ref).cuda().data_ptr(), True, ref_off, tv, cs, ce, keep, off, ratio, 100,
                            0.0, 300, pen, outs=outs, memspace=_native.B2_DEVICE)
        handle.synchronize()
        b, nsh, sch = buf.cpu().numpy(), ns.cpu().numpy(), sc.cpu().numpy()
        assert np.all(b[: guard + pad] == -12345) and np.all(b[guard + n:] == -12345)
        assert np.all(nsh[:guard] == -12345) and np.all(nsh[guard + len(tv):] == -12345)
        assert np.all(sch[:guard] == -1.5) and np.all(sch[guard + len(tv):] == -1.5)
        assert np.array_equal(b[guard + pad: guard + n], want[0][pad:])
        assert np.array_equal(nsh[guard: guard + len(tv)], want[1])
        assert np.array_equal(sch[guard: guard + len(tv)], want[2], equal_nan=True)


def _oracle_over_speech(s, spl, speech, speech_off, c, pen):
    want = sp.split_tracks(np.asarray(speech, np.float64), speech_off, c["track_video"], c["cue_start"], c["cue_end"],
                           None, c["cue_off"], spl["ratio"], 100, 0.0, s.max_offset_samples, pen)
    for w, k in zip(want, ("cue_offset", "n_segments", "split_score")):
        g = spl[k].cpu().numpy() if hasattr(spl[k], "cpu") else spl[k]
        assert np.array_equal(w, g, equal_nan=True), (k, pen)


def test_text_pgs_signal_references_and_ingest_session():
    """The split over the references a sync call wrote equals the oracle over the same signals: a subs_then_ call with
    text, PGS and stored-signal references (host), and an ingest session's device result."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    rng = np.random.RandomState(13)
    kinds = ["audio", "text", "pgs", "sig"]
    c = _sig_corpus([(50.0 + 3 * v, kinds[v % 4], [(GRID[int(rng.randint(0, 3))], int(rng.randint(-400, 400)))
                                                     for _ in range(1 + v % 2)]) for v in range(8)], seed0=31)
    V = len(c["pcm_off"]) - 1
    sv = np.arange(V)
    s = BatchSynchronizer(GRID, vad="subs_then_energy_zcr", non_speech_label=0.0, max_offset_seconds=8)
    host = s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"],
                              speech_video=sv, **_streams(c, ("text", "pgs", "sig"), False))
    for pen in (0.0, 6.0, math.inf):
        spl = s.split_tracks_host(host, c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"], split_penalty=pen)
        assert np.any(spl["n_segments"] > 0)
        _oracle_over_speech(s, spl, host[-2], host[-1], c, pen)
    # an ingest session over the audio videos: its device result goes straight into split_tracks
    a = _sig_corpus([(50.0 + 3 * v, "audio", [(GRID[int(rng.randint(0, 3))], int(rng.randint(-400, 400)))])
                     for v in range(3)], seed0=41)
    s2 = BatchSynchronizer(GRID, non_speech_label=0.0, max_offset_seconds=8)
    sess = s2.ingest(3)
    for v in range(3):
        p = a["pcm"][a["pcm_off"][v]: a["pcm_off"][v + 1]]
        for i in range(0, len(p), 70000):   # pushes that cut windows and calls
            sess.push(v, p[i: i + 70000].tobytes())
    T = len(a["track_video"])
    out = {"best_score": torch.empty(T, dtype=torch.float64, device="cuda"),
           "best_offset": torch.empty(T, dtype=torch.int32, device="cuda"),
           "best_k": torch.empty(T, dtype=torch.int32, device="cuda")}
    out = sess.sync_tracks(a["track_video"], a["cue_start"], a["cue_end"], a["cue_off"], speech_video=np.arange(3),
                           out=out)
    spl = s2.split_tracks(out, a["track_video"], a["cue_start"], a["cue_end"], a["cue_off"], split_penalty=6.0)
    torch.cuda.synchronize()
    assert np.any(spl["n_segments"].cpu().numpy() > 0)
    _oracle_over_speech(s2, spl, out["speech"].cpu().numpy(), out["speech_off"], a, 6.0)
