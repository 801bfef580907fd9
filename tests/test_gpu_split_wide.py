"""GPU tests of the wide per-segment split (b2_split_tracks_wide: one thread-block cluster per track; run on an H100).

Yardsticks: b2_split_tracks (bit for bit wherever both run) and the vectorised oracle (tests/split_wide.py, itself held
to oracle/split_oracle.py).  Windows up to the envelope the device reports (262 144 offsets at 16-CTA clusters, or the
widest cluster it co-schedules), ties across CTAs, mixed cluster sizes with skipped and three-level tracks, planted
breaks of minutes in both directions, and BatchSynchronizer.split_tracks(split_max_offset_seconds=...)."""
import math
import re

import numpy as np
import pytest

import split_wide as sw
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp
from test_gpu_sig_ref import _sig_corpus
from test_gpu_split import _request

pytestmark = pytest.mark.gpu

CTA = 16384   # offsets of one CTA


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _mos_for_width(R, S, W):
    """max_offset_samples that gives a window of exactly W offsets for (R, S): past S the low end clips at -S, so the
    window is mos + S + 1 while the high end is not clipped."""
    mos = W - S - 1
    o_lo, o_hi = ao.offset_range(R, S, mos)
    assert o_hi - o_lo + 1 == W, (R, S, W, o_lo, o_hi)
    return mos


def _few_cues(rng, n, dur):
    cs = np.sort(np.round(rng.uniform(1.0, dur, n), 2))
    return cs, np.round(cs + rng.uniform(0.3, 4.0, n), 2)


@pytest.fixture(scope="module")
def envelope(handle):
    """The widest window b2_split_tracks_wide takes on this device, read from its refusal one past 16 clusters' worth;
    nothing is launched before that refusal."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(1)
    cs, ce = _few_cues(rng, 4, 20.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    R = 16 * CTA + 2000
    mos = _mos_for_width(R, S, 16 * CTA + 1)
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than (\d+)" % (16 * CTA + 1)) as e:
        handle.split_tracks_wide(np.zeros(R), True, [0, R], [0], cs, ce, None, [0, 4], [1.0], 100, 0.0, mos, 1.0)
    assert handle.launch_count == n0
    limit = int(re.search(r"wider than (\d+)", str(e.value)).group(1))
    assert limit % CTA == 0 and 2 * CTA <= limit <= 16 * CTA, limit
    return limit


def _check(want, got, what):
    for w, g, name in zip(want, got, ("cue_offset", "n_segments", "split_score")):
        assert np.array_equal(w, g, equal_nan=True), (what, name, w, g)


def _device(handle, fn, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen):
    import torch
    from ffsubsync_b200 import _native
    T = len(off) - 1
    outs = [torch.full((max(int(off[-1]), 1),), 7, dtype=torch.int32, device="cuda"),
            torch.full((T,), 7, dtype=torch.int32, device="cuda"),
            torch.zeros(T, dtype=torch.float64, device="cuda")]
    d_ref = torch.from_numpy(np.ascontiguousarray(ref)).cuda()
    fn(d_ref.data_ptr(), f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen,
       outs=[o.data_ptr() for o in outs], memspace=_native.B2_DEVICE)
    handle.synchronize()
    n = int(off[-1])
    return outs[0].cpu().numpy()[:n], outs[1].cpu().numpy(), outs[2].cpu().numpy()


@pytest.mark.parametrize("seed", range(6))
def test_wide_equals_narrow(handle, seed):
    """Windows up to 32 768 offsets (clusters of 1 and 2 CTAs), both memspaces: b2_split_tracks_wide equals
    b2_split_tracks bit for bit."""
    label = [0.0, 0.3, -0.5][seed % 3]
    f64 = seed % 2 == 0
    mos = [16384, 300, 9000][seed % 3]
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed, R=1200 + 400 * (seed % 3) + 20000 * (seed % 2),
                                                          label=label, f64=f64)
    for pen in (0.0, 3.0, math.inf):
        a = handle.split_tracks(ref, f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen)
        b = handle.split_tracks_wide(ref, f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen)
        _check(a, b, (seed, pen, "host"))
        d = _device(handle, handle.split_tracks_wide, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen)
        _check(a, d, (seed, pen, "device"))


@pytest.mark.parametrize("W", [32769, 49153, 131072, 262144])
@pytest.mark.parametrize("label,f64", [(0.0, True), (0.3, False)])
def test_wide_window_equals_oracle(handle, envelope, W, label, f64):
    """Exact window widths: past one cluster of two, a last CTA with one offset, 8 and 16 CTAs (at most the device's
    envelope), and a short reference that clips the window on both sides; labels 0 and 0.3, float64 and float32."""
    W = min(W, envelope)
    rng = np.random.RandomState(W % 1000 + int(10 * label))
    cs, ce = _few_cues(rng, 7, 40.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    R = W + 3000
    mos = _mos_for_width(R, S, W)
    ref = np.where(rng.rand(R) < 0.4, 1.0, label).astype(np.float64 if f64 else np.float32)
    short = np.where(rng.rand(9000) < 0.4, 1.0, label).astype(ref.dtype)   # the window clipped to [-S, R + ...]
    both = np.concatenate([ref, short])
    ref_off = np.array([0, R, R + len(short)])
    off = np.array([0, 7, 14], np.int64)
    cs2, ce2 = np.concatenate([cs, cs]), np.concatenate([ce, ce])
    for pen in (0.0, 5.0):
        want = sw.split_tracks(both.astype(np.float64), ref_off, [0, 1], cs2, ce2, None, off, [1.0, 1.0], 100, 0.0,
                               mos, pen)
        got = handle.split_tracks_wide(both, f64, ref_off, [0, 1], cs2, ce2, None, off, [1.0, 1.0], 100, 0.0, mos, pen)
        _check(want, got, (W, pen, "host"))
        d = _device(handle, handle.split_tracks_wide, both, f64, ref_off, [0, 1], cs2, ce2, None, off, [1.0, 1.0],
                    mos, pen)
        _check(want, d, (W, pen, "device"))


def test_past_the_envelope(handle, envelope):
    """The envelope runs; one more offset is B2_ERR_UNSUPPORTED naming it, with nothing launched."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(3)
    cs, ce = _few_cues(rng, 3, 20.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    R = envelope + 2000
    ref = np.where(rng.rand(R) < 0.5, 1.0, 0.0)
    off = [0, 3]
    got = handle.split_tracks_wide(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0,
                                   _mos_for_width(R, S, envelope), 2.0)
    assert got[1][0] >= 1
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than %d" % (envelope + 1, envelope)):
        handle.split_tracks_wide(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0,
                                 _mos_for_width(R, S, envelope + 1), 2.0)
    assert handle.launch_count == n0


def test_ties_across_ctas(handle, envelope):
    """A reference periodic at 20 000 frames (more than one CTA's 16 384 offsets): every unit's maximum is attained at
    offsets in different CTAs, and the largest of them wins, as in the oracle."""
    rng = np.random.RandomState(5)
    P, reps = 20000, 5
    base = (rng.rand(P) < 0.5).astype(np.float64)
    ref = np.tile(base, reps)
    R = len(ref)
    cs, ce = _few_cues(rng, 6, 30.0)
    mask = ro.rasterize(cs, ce, None, 100, 0, 1.0)[0] > 0
    S = len(mask)
    W = min(envelope, 4 * CTA)
    mos = _mos_for_width(R, S, W)
    o_lo, o_hi = ao.offset_range(R, S, mos)
    m, beta = sp.ref_levels(ref)
    units = sp.units_of(sp.runs_of(mask), S)
    U = sw.unit_table(m, units, list(range(o_lo, o_hi + 1)), sp.levels(1.0, beta))
    tot = U.sum(axis=0)   # +-1: exact integers
    best = np.flatnonzero(tot == tot.max()) + o_lo
    assert (best.max() - best.min()) >= CTA, best   # tied maxima in different CTAs
    for pen in (math.inf, 4.0, 0.0):
        want = sw.split_tracks(ref, [0, R], [0], cs, ce, None, [0, 6], [1.0], 100, 0.0, mos, pen)
        got = handle.split_tracks_wide(ref, True, [0, R], [0], cs, ce, None, [0, 6], [1.0], 100, 0.0, mos, pen)
        _check(want, got, pen)
        if pen == math.inf:
            assert np.all(got[0] == best.max()), (got[0], best)


def test_mixed_clusters_skips_and_three_levels(handle, envelope):
    """One call whose tracks take 1, 2 and up to 16 CTAs (references of different lengths clip the shared window),
    with NaN-ratio tracks and a video whose reference has a third level.  Under B2_DEVICE that video's tracks get
    n_segments == -1 and the others equal the oracle; B2_HOST refuses the call naming the video and frame."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(8)
    mos = envelope - 6000   # windows of mos + S + 1 offsets on the long video (the low end clips at -S)
    lens = [envelope + 5000, 12000, 30000, 5000, 60000]
    refs = [np.where(rng.rand(L) < 0.45, 1.0, 0.3) for L in lens]
    refs[3][1234] = 0.7   # a third level
    ref = np.concatenate(refs)
    ref_off = np.concatenate([[0], np.cumsum(lens)])
    tv = np.array([0, 1, 2, 3, 3, 4, 0, 2, 1])
    T = len(tv)
    cs, ce, off = [], [], [0]
    for t in range(T):
        a, b = _few_cues(rng, int(rng.randint(0, 8)), 45.0)
        cs.append(a)
        ce.append(b)
        off.append(off[-1] + len(a))
    cs, ce, off = np.concatenate(cs), np.concatenate(ce), np.array(off, np.int64)
    ratio = np.array([1.0, 25 / 24.0, 1.0, 1.0, 24 / 25.0, np.nan, 24 / 25.0, np.nan, 1.0])
    widths = []
    for t in range(T):
        S = len(ro.rasterize(cs[off[t]:off[t + 1]], ce[off[t]:off[t + 1]], None, 100, 0, ratio[t] if ratio[t] == ratio[t] else 1.0)[0])
        o_lo, o_hi = ao.offset_range(lens[tv[t]], S, mos)
        widths.append(o_hi - o_lo + 1)
    ctas = {-(-w // CTA) for w, r in zip(widths, ratio) if r == r}
    assert 1 in ctas and len(ctas) >= 3 and max(ctas) == envelope // CTA, (widths, ctas)
    for pen in (0.0, 6.0):
        co, ns, sc = _device(handle, handle.split_tracks_wide, ref, True, ref_off, tv, cs, ce, None, off, ratio, mos,
                             pen)
        ok = tv != 3
        bad_cues = np.repeat(~ok, np.diff(off))
        assert np.all(ns[~ok] == -1) and np.all(np.isnan(sc[~ok])) and np.all(co[bad_cues] == 0)
        sel = np.flatnonzero(ok)
        sub_off = np.concatenate([[0], np.cumsum(np.diff(off)[sel])])
        idx = np.concatenate([np.arange(off[t], off[t + 1]) for t in sel])
        want = sw.split_tracks(ref, ref_off, tv[sel], cs[idx], ce[idx], None, sub_off, ratio[sel], 100, 0.0, mos, pen)
        _check(want, (co[idx], ns[sel], sc[sel]), pen)
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*video 3: frame 1234"):
        handle.split_tracks_wide(ref, True, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, 6.0)


def _planted(shifts, n=40, seed=4):
    """n cues over about 100 s from 30 s, cut into len(shifts) equal parts; part i sits shifted by shifts[i] frames in
    a clean reference (1.0 under the shifted cue frames, 0.0 elsewhere)."""
    rng = np.random.RandomState(seed)
    cs = np.round(30 + np.cumsum(rng.uniform(1.0, 4.0, n)), 2)
    ce = np.round(cs + rng.uniform(0.5, 2.0, n), 2)
    m = ro.rasterize(cs, ce, None, 100, 0, 1.0)[0] > 0
    R = len(m) + max(shifts) + 600
    ref = np.zeros(R)
    f = np.arange(len(m))
    k = len(shifts)
    cuts = [0] + [int(round(cs[n * i // k] * 100)) for i in range(1, k)] + [len(m)]
    for i, d in enumerate(shifts):
        g = f[cuts[i]:cuts[i + 1]][m[cuts[i]:cuts[i + 1]]] + d
        ref[g[(g >= 0) & (g < R)]] = 1.0
    return ref, cs, ce, [n * i // k for i in range(k + 1)]


BREAKS = [(300, 300 + 18000), (300 + 18000, 300), (300, 300 + 48000), (300 + 48000, 300), (300, 300 + 120000),
          (300 + 120000, 300), (300, 300 + 24000, 300 + 48000, 300 + 72000)]


@pytest.mark.parametrize("shifts", BREAKS, ids=lambda s: "_".join(map(str, s)))
def test_planted_breaks(handle, envelope, shifts):
    """3, 8 and 20 min the subtitles do not have (the later cues sit later) and the reverse, and three cumulative
    4 min breaks: every part is found at its exact offset with the break at the planted cue, equal to the oracle;
    apply_split then equals split_oracle.apply_split with offsets far past +-60 s."""
    ref, cs, ce, parts = _planted(shifts)
    R = len(ref)
    mos = max(shifts) + 500
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    o_lo, o_hi = ao.offset_range(R, S, mos)
    if o_hi - o_lo + 1 > envelope:
        pytest.skip("window of %d offsets past this device's envelope of %d" % (o_hi - o_lo + 1, envelope))
    off = np.array([0, len(cs)], np.int64)
    for pen in (10.0, 50.0):
        co, ns, sc = handle.split_tracks_wide(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen)
        assert ns[0] == len(shifts), (pen, ns)
        for i, d in enumerate(shifts):
            assert np.all(co[parts[i]:parts[i + 1]] == d), (pen, i, co)
        want = sw.split_tracks(ref, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen)
        _check(want, (co, ns, sc), pen)
    su, eu, st = handle.apply_split([1.0], ns, co, cs, ce, off, 100)
    w = sp.apply_split([1.0], ns, co, cs, ce, off, 100)
    for a, b in zip(w, (su, eu, st)):
        assert np.array_equal(a, b)


def test_batch_split_max_offset_seconds():
    """BatchSynchronizer.split_tracks / split_tracks_host with split_max_offset_seconds, after sync_device_tracks,
    sync_host_tracks and an ingest session: equal to the oracle at abs(int(s * sample_rate)) samples; None gives the
    calls of before (b2_split_tracks at the synchroniser's window) exactly; apply_split equals the oracle's."""
    import torch
    from ffsubsync_b200.batch import DEFAULT_APPLY_OFFSET_SECONDS, BatchSynchronizer
    GRID = [1.0, 25 / 24.0, 24 / 25.0]
    rng = np.random.RandomState(17)
    c = _sig_corpus([(200.0 + 7 * v, "audio", [(GRID[int(rng.randint(0, 3))], int(rng.randint(-700, 700)))
                                               for _ in range(1 + v % 2)]) for v in range(4)], seed0=9)
    V = len(c["pcm_off"]) - 1
    sv = np.arange(V)
    s = BatchSynchronizer(GRID, non_speech_label=0.0, max_offset_seconds=8)
    args = (c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])

    def oracle(speech, speech_off, ratio, mos, pen):
        return sw.split_tracks(np.asarray(speech, np.float64), speech_off, c["track_video"], c["cue_start"],
                               c["cue_end"], None, c["cue_off"], ratio, 100, 0.0, mos, pen)

    host = s.sync_host_tracks(c["pcm"], c["pcm_off"], *args, speech_video=sv)
    out = s.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], *args, speech_video=sv)
    for secs in (None, 150.0, -600.0):
        mos = s.max_offset_samples if secs is None else abs(int(secs * s.sample_rate))
        for pen in (5.0, math.inf):
            h = s.split_tracks_host(host, *args, split_penalty=pen, split_max_offset_seconds=secs)
            _check(oracle(host[-2], host[-1], h["ratio"], mos, pen), (h["cue_offset"], h["n_segments"],
                                                                     h["split_score"]), (secs, pen, "host"))
            d = s.split_tracks(out, *args, split_penalty=pen, split_max_offset_seconds=secs)
            a = s.apply_split(d, c["cue_start"], c["cue_end"], c["cue_off"])
            torch.cuda.synchronize()
            dn = [d[k].cpu().numpy() for k in ("cue_offset", "n_segments", "split_score")]
            _check(oracle(out["speech"].cpu().numpy(), out["speech_off"], d["ratio"], mos, pen), dn, (secs, pen))
            want = sp.apply_split(d["ratio"], dn[1], dn[0], c["cue_start"], c["cue_end"], c["cue_off"], 100,
                                  DEFAULT_APPLY_OFFSET_SECONDS)
            if secs is None:   # today's call, unchanged
                base = s.handle.split_tracks(out["speech"].cpu().numpy(), True, out["speech_off"], sv[c["track_video"]],
                                             c["cue_start"], c["cue_end"], None, c["cue_off"], d["ratio"], 100, 0.0,
                                             s.max_offset_samples, pen)
                _check(base, dn, (secs, pen, "unchanged"))
            ah = s.apply_split_host({k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in d.items()},
                                    c["cue_start"], c["cue_end"], c["cue_off"])
            for k, w in zip(("synced_start_us", "synced_end_us", "status"), want):
                assert np.array_equal(a[k].cpu().numpy(), w) and np.array_equal(ah[k], w), k
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
    d = s.split_tracks(o, *args, split_penalty=5.0, split_max_offset_seconds=300.0)
    torch.cuda.synchronize()
    dn = [d[k].cpu().numpy() for k in ("cue_offset", "n_segments", "split_score")]
    assert np.any(dn[1] > 0)
    _check(oracle(o["speech"].cpu().numpy(), o["speech_off"], d["ratio"], 30000, 5.0), dn, "ingest")
