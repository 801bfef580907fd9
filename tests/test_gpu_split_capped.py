"""GPU tests of the capped split (b2_split_tracks_capped: at most N segments per track, one cluster of N x C CTAs per
track; run on an H100).

Yardsticks: the capped oracle (tests/split_capped.py, itself held to exhaustive enumeration and oracle/split_oracle.py)
bit for bit, b2_split_tracks / b2_split_tracks_wide wherever a track has at most N units, and their +inf penalty at
N = 1.  Also a noisy reference with a planted 90 s break in both directions, dead tracks in a live call, the refusals,
and BatchSynchronizer.split_tracks(max_segments=...)."""
import math

import numpy as np
import pytest

import split_capped as sc
from oracle import raster_oracle as ro
from oracle import split_oracle as sp
from test_gpu_sig_ref import _sig_corpus
from test_gpu_split import _request
from test_gpu_split_wide import _mos_for_width

pytestmark = pytest.mark.gpu

CTA = 16384   # offsets of one CTA


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _check(want, got, what, names=("cue_offset", "n_segments", "split_score", "split_profile")):
    for w, g, name in zip(want, got, names):
        assert np.array_equal(np.asarray(w), np.asarray(g).reshape(np.shape(w)), equal_nan=True), (what, name, w, g)


def _device(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, N):
    import torch
    from ffsubsync_b200 import _native
    T = len(off) - 1
    outs = [torch.full((max(int(off[-1]), 1),), 7, dtype=torch.int32, device="cuda"),
            torch.full((T,), 7, dtype=torch.int32, device="cuda"),
            torch.zeros(T, dtype=torch.float64, device="cuda"),
            torch.zeros((T, N), dtype=torch.float64, device="cuda")]
    d_ref = torch.from_numpy(np.ascontiguousarray(ref)).cuda()
    handle.split_tracks_capped(d_ref.data_ptr(), f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, N,
                               outs=[o.data_ptr() for o in outs], memspace=_native.B2_DEVICE)
    handle.synchronize()
    return outs[0].cpu().numpy()[:int(off[-1])], outs[1].cpu().numpy(), outs[2].cpu().numpy(), outs[3].cpu().numpy()


@pytest.fixture(scope="module")
def cmax(handle):
    """The widest cluster of the capped kernel on this device: a one-CTA window at N segments (N x 1 CTAs) is refused
    exactly when N exceeds it, with nothing launched before the refusal."""
    from ffsubsync_b200._native import NativeError
    cs, ce = np.array([1.0, 5.0]), np.array([2.0, 6.0])
    n0 = handle.launch_count
    for N in range(16, 0, -1):
        try:
            handle.split_tracks_capped(np.zeros(3000), True, [0, 3000], [0], cs, ce, None, [0, 2], [1.0], 100, 0.0,
                                       100, 1.0, N)
            return N
        except NativeError as e:
            assert handle.launch_count == n0 and "B2_ERR_UNSUPPORTED" in str(e), str(e)
    raise AssertionError("no cluster of the capped kernel fits")


@pytest.mark.parametrize("N", [1, 2, 3, 8, 16])
@pytest.mark.parametrize("seed", range(4))
def test_capped_equals_oracle(handle, cmax, seed, N):
    """Seeded two-level references (labels 0, 0.3, -0.5; float64 and float32), skipped tracks, kept-cue masks; windows
    of one CTA, and of two CTAs wherever N x 2 fits the device's clusters; both memspaces."""
    label = [0.0, 0.3, -0.5][seed % 3]
    f64 = seed % 2 == 0
    for R, mos in ((1600 + 300 * seed, 500), (21000, 16384)):
        ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed, R=R, label=label, f64=f64)
        S_max = max(len(ro.rasterize(cs[off[t]:off[t + 1]], ce[off[t]:off[t + 1]], None, 100, 0,
                                     ratio[t] if ratio[t] == ratio[t] else 1.0)[0]) for t in range(len(tv)))
        C = -(-(mos + S_max + 1) // CTA)
        if N * C > cmax:
            continue
        for pen in (0.0, 3.0, math.inf):
            want = sc.split_tracks(ref.astype(np.float64), ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen,
                                   N)
            got = handle.split_tracks_capped(ref, f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, N)
            _check(want, got, (seed, N, R, pen, "host"))
            d = _device(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, N)
            _check(want, d, (seed, N, R, pen, "device"))
            assert np.all(got[1][got[1] > 0] <= N)


@pytest.mark.parametrize("seed", range(4))
def test_equals_uncapped_entry_points(handle, seed):
    """Tracks of at most 16 units: N = 16 gives b2_split_tracks' and b2_split_tracks_wide's results bit for bit; any
    tracks: N = 1 gives their results at penalty +inf."""
    rng = np.random.RandomState(40 + seed)
    label = [0.0, 0.3][seed % 2]
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed + 10, R=2500, label=label, f64=True)
    few = np.concatenate([np.arange(off[t], min(off[t + 1], off[t] + int(rng.randint(0, 17)))) for t in range(len(tv))])
    lens = [np.count_nonzero((few >= off[t]) & (few < off[t + 1])) for t in range(len(tv))]
    off16 = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    cs16, ce16, keep16 = cs[few], ce[few], keep[few]
    mos = [300, 900][seed % 2]
    for pen in (0.0, 2.0, 7.5):
        got = handle.split_tracks_capped(ref, True, ref_off, tv, cs16, ce16, keep16, off16, ratio, 100, 0.0, mos, pen,
                                         16)
        for fn in (handle.split_tracks, handle.split_tracks_wide):
            _check(fn(ref, True, ref_off, tv, cs16, ce16, keep16, off16, ratio, 100, 0.0, mos, pen), got[:3],
                   (seed, pen, "16"))
        one = handle.split_tracks_capped(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, 1)
        for fn in (handle.split_tracks, handle.split_tracks_wide):
            _check(fn(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, math.inf), one[:3],
                   (seed, pen, "1"))
        live = one[1] > 0
        assert np.array_equal(one[3][live, 0], one[2][live])   # one segment: the profile is the plain score


def _noisy_break(removal, n=120, cut=60, flip=0.1, seed=6):
    """n cues from 30 s; a reference of the cues shifted into place with a fixed fraction of its frames flipped.  A
    break (removal False): the video has 90 s the subtitles do not have, cues [0, cut) at +3 s and [cut, n) at +93 s.
    A removal: the subtitles have 90 s the video does not, cues [0, cut) at +93 s, the cues of the next 90 s nowhere,
    the rest at +3 s.  Returns (ref, cue starts, cue ends, [(first cue, end cue, offset)])."""
    rng = np.random.RandomState(seed)
    cs = np.round(30 + np.cumsum(rng.uniform(1.0, 4.0, n)), 2)
    ce = np.round(cs + rng.uniform(0.5, 2.0, n), 2)
    if removal:
        back = int(np.searchsorted(cs, cs[cut] + 90.0))
        parts = [(0, cut, 9300), (back, n, 300)]
    else:
        parts = [(0, cut, 300), (cut, n, 9300)]
    R = int(ce[-1] * 100) + 9300 + 600
    ref = np.zeros(R)
    for a, b, d in parts:
        g = np.flatnonzero(ro.rasterize(cs[a:b], ce[a:b], None, 100, 0, 1.0)[0] > 0) + d
        ref[g[(g >= 0) & (g < R)]] = 1.0
    fl = rng.rand(R) < flip
    ref[fl] = 1.0 - ref[fl]
    return ref, cs, ce, parts


@pytest.mark.parametrize("removal", [False, True], ids=["break", "removal"])
def test_noisy_planted_break(handle, removal):
    """10 % of the reference's frames flipped and a 90 s break: at penalty 2 the uncapped split returns dozens of
    segments; max_segments = 2 at the same penalty returns exactly the two planted offsets with the break at the
    planted cue (inside the removed stretch for a removal), equal to the oracle; apply_split takes the result."""
    ref, cs, ce, parts = _noisy_break(removal)
    R, off = len(ref), np.array([0, len(cs)], np.int64)
    mos, pen = 9800, 2.0
    u = handle.split_tracks_wide(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen)
    assert u[1][0] >= 20, u[1]
    got = handle.split_tracks_capped(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen, 2)
    co = got[0]
    assert got[1][0] == 2
    for a, b, d in parts:
        assert np.all(co[a:b] == d), (a, b, d, co)
    brk = int(np.flatnonzero(np.diff(co))[0]) + 1
    assert parts[0][1] <= brk <= parts[1][0], brk
    assert got[3][0, 1] > got[3][0, 0]
    _check(sc.split_tracks(ref, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen, 2), got, removal)
    su, eu, st = handle.apply_split([1.0], got[1], co, cs, ce, off, 100)
    w = sp.apply_split([1.0], got[1], co, cs, ce, off, 100)
    for x, y in zip(w, (su, eu, st)):
        assert np.array_equal(x, y)


def test_dead_tracks_in_a_live_call(handle):
    """Skipped (NaN ratio) tracks, an empty reference and a three-level video among live tracks: under B2_DEVICE the
    three-level video's tracks get n_segments == -1, the skipped ones 0, all of them NaN scores, NaN profiles and
    offsets 0, the live ones the oracle's results; B2_HOST refuses the three-level video.  A zero window makes every
    track dead."""
    from ffsubsync_b200._native import NativeError
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(21, V=3, T=8, R=2200, label=0.3, f64=True)
    ref = ref.copy()
    bad_v = int(tv[-1])
    ref[ref_off[bad_v] + 77] = 0.6   # a third level
    # an empty fourth video for two tracks
    ref_off = np.concatenate([ref_off, [ref_off[-1]]])
    tv = tv.copy()
    tv[1] = 3
    ratio = ratio.copy()
    ratio[2] = np.nan
    ratio[-1] = 1.0   # a live track on the three-level video
    N, mos = 3, 400
    co, ns, s, pr = _device(handle, ref, True, ref_off, tv, cs, ce, keep, off, ratio, mos, 1.0, N)
    bad = (tv == bad_v) & ~np.isnan(ratio)
    dead = ((tv == 3) | np.isnan(ratio)) & ~bad
    assert bad.any() and dead.any() and (~bad & ~dead).any()
    assert np.all(ns[bad] == -1) and np.all(ns[dead] == 0)
    assert np.all(np.isnan(s[bad | dead])) and np.all(np.isnan(pr[bad | dead]))
    assert np.all(co[np.repeat(bad | dead, np.diff(off))] == 0)
    sel = np.flatnonzero(~bad)
    sub_off = np.concatenate([[0], np.cumsum(np.diff(off)[sel])])
    idx = np.concatenate([np.arange(off[t], off[t + 1]) for t in sel])
    want = sc.split_tracks(ref, ref_off, tv[sel], cs[idx], ce[idx], keep[idx], sub_off, ratio[sel], 100, 0.0, mos, 1.0,
                           N)
    _check(want, (co[idx], ns[sel], s[sel], pr[sel]), "live")
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*video %d: frame 77" % bad_v):
        handle.split_tracks_capped(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, 1.0, N)
    ok = ref.copy()
    ok[ref_off[bad_v] + 77] = 0.3
    got = handle.split_tracks_capped(ok, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, 0, 1.0, N)
    assert np.all(got[1] == 0) and np.all(np.isnan(got[2])) and np.all(np.isnan(got[3])) and not got[0].any()


def test_refusals(handle, cmax):
    """max_segments 0 is B2_ERR_BAD_ARG, 17 B2_ERR_UNSUPPORTED naming 16; at N = 2 the widest window the device's
    clusters hold runs and one more offset is refused naming it; nothing is launched before a refusal."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(3)
    cs = np.sort(np.round(rng.uniform(1.0, 20.0, 3), 2))
    ce = cs + 0.5
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    off = [0, 3]
    limit = CTA * (cmax // 2)
    R = limit + 2000
    ref = np.where(rng.rand(R) < 0.5, 1.0, 0.0)
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_BAD_ARG.*max_segments 0 must be >= 1"):
        handle.split_tracks_capped(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0, 0)
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*max_segments 17 is more than 16"):
        handle.split_tracks_capped(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0, 17)
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than %d at 2 segments"
                       % (limit + 1, limit)):
        handle.split_tracks_capped(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0,
                                   _mos_for_width(R, S, limit + 1), 1.0, 2)
    assert handle.launch_count == n0
    mos = _mos_for_width(R, S, limit)
    got = handle.split_tracks_capped(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, 1.0, 2)
    _check(sc.split_tracks(ref, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, 1.0, 2), got, "envelope")


def test_batch_max_segments():
    """BatchSynchronizer.split_tracks / split_tracks_host with max_segments after sync_device_tracks, sync_host_tracks
    and an ingest session, with and without split_max_offset_seconds: equal to the capped oracle; apply_split and
    apply_split_host take the results; max_segments=None keeps the dict of before."""
    import torch
    from ffsubsync_b200.batch import DEFAULT_APPLY_OFFSET_SECONDS, BatchSynchronizer
    GRID = [1.0, 25 / 24.0, 24 / 25.0]
    rng = np.random.RandomState(23)
    c = _sig_corpus([(200.0 + 7 * v, "audio", [(GRID[int(rng.randint(0, 3))], int(rng.randint(-700, 700)))
                                               for _ in range(1 + v % 2)]) for v in range(4)], seed0=13)
    V = len(c["pcm_off"]) - 1
    sv = np.arange(V)
    s = BatchSynchronizer(GRID, non_speech_label=0.0, max_offset_seconds=8)
    args = (c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])

    def oracle(speech, speech_off, ratio, mos, pen, N):
        return sc.split_tracks(np.asarray(speech, np.float64), speech_off, c["track_video"], c["cue_start"],
                               c["cue_end"], None, c["cue_off"], ratio, 100, 0.0, mos, pen, N)

    host = s.sync_host_tracks(c["pcm"], c["pcm_off"], *args, speech_video=sv)
    out = s.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], *args, speech_video=sv)
    names = ("cue_offset", "n_segments", "split_score", "split_profile")
    for secs, N in ((None, 2), (150.0, 3)):
        mos = s.max_offset_samples if secs is None else abs(int(secs * s.sample_rate))
        pen = 5.0
        h = s.split_tracks_host(host, *args, split_penalty=pen, split_max_offset_seconds=secs, max_segments=N)
        assert h["split_profile"].shape == (len(c["track_video"]), N)
        _check(oracle(host[-2], host[-1], h["ratio"], mos, pen, N), [h[k] for k in names], (secs, N, "host"))
        d = s.split_tracks(out, *args, split_penalty=pen, split_max_offset_seconds=secs, max_segments=N)
        a = s.apply_split(d, c["cue_start"], c["cue_end"], c["cue_off"])
        torch.cuda.synchronize()
        dn = [d[k].cpu().numpy() for k in names]
        assert dn[3].shape == (len(c["track_video"]), N)
        _check(oracle(out["speech"].cpu().numpy(), out["speech_off"], d["ratio"], mos, pen, N), dn, (secs, N))
        want = sp.apply_split(d["ratio"], dn[1], dn[0], c["cue_start"], c["cue_end"], c["cue_off"], 100,
                              DEFAULT_APPLY_OFFSET_SECONDS)
        ah = s.apply_split_host(h, c["cue_start"], c["cue_end"], c["cue_off"])
        wh = sp.apply_split(h["ratio"], h["n_segments"], h["cue_offset"], c["cue_start"], c["cue_end"], c["cue_off"],
                            100, DEFAULT_APPLY_OFFSET_SECONDS)
        for k, w, x in zip(("synced_start_us", "synced_end_us", "status"), want, wh):
            assert np.array_equal(a[k].cpu().numpy(), w) and np.array_equal(ah[k], x), k
    assert "split_profile" not in s.split_tracks(out, *args, split_penalty=5.0)
    # an ingest session's device result
    sess = s.ingest(V)
    for v in range(V):
        p = c["pcm"][c["pcm_off"][v]: c["pcm_off"][v + 1]]
        for i in range(0, len(p), 90000):
            sess.push(v, p[i: i + 90000].tobytes())
    T = len(c["track_video"])
    o = {"best_score": torch.empty(T, dtype=torch.float64, device="cuda"),
         "best_offset": torch.empty(T, dtype=torch.int32, device="cuda"),
         "best_k": torch.empty(T, dtype=torch.int32, device="cuda")}
    o = sess.sync_tracks(*args, speech_video=sv, out=o)
    d = s.split_tracks(o, *args, split_penalty=5.0, split_max_offset_seconds=300.0, max_segments=4)
    a = s.apply_split(d, c["cue_start"], c["cue_end"], c["cue_off"])
    torch.cuda.synchronize()
    dn = [d[k].cpu().numpy() for k in names]
    assert np.any(dn[1] > 0)
    _check(oracle(o["speech"].cpu().numpy(), o["speech_off"], d["ratio"], 30000, 5.0, 4), dn, "ingest")
    want = sp.apply_split(d["ratio"], dn[1], dn[0], c["cue_start"], c["cue_end"], c["cue_off"], 100,
                          DEFAULT_APPLY_OFFSET_SECONDS)
    for k, w in zip(("synced_start_us", "synced_end_us", "status"), want):
        assert np.array_equal(a[k].cpu().numpy(), w), k


def test_envelope_report(cmax):
    """The capped kernel's widest cluster and the widest window at each N, as the refusals state them (for the record;
    K9s's table comes from this)."""
    rows = ["N=%d: %d CTAs per layer, %d offsets" % (N, cmax // N, CTA * (cmax // N)) for N in (1, 2, 4, 8, 16)]
    print("capped split: widest cluster %d CTAs; " % cmax + "; ".join(rows))
    assert 1 <= cmax <= 16
