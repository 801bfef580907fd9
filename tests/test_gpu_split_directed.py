"""GPU tests of the directed split (b2_split_tracks_directed: segment offsets that only grow, direction +1, or only
shrink, -1, along the track; run on an H100).

Yardsticks: the directed restatement (tests/split_directed.py, itself held to exhaustive enumeration of monotone paths,
to oracle/split_oracle.py at penalty +inf, and to its argmax form) bit for bit, and b2_split_tracks_wide at penalty
+inf.  Also ties across CTAs, monotone paths on a noisy reference, planted edits on a clean one, dead tracks, the
refusals, and BatchSynchronizer.split_tracks(split_direction=...)."""
import math
import re

import numpy as np
import pytest

import split_directed as sd
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp
from test_gpu_sig_ref import _sig_corpus
from test_gpu_split import _request
from test_gpu_split_capped import _noisy_break
from test_gpu_split_wide import _few_cues, _mos_for_width, _planted

pytestmark = pytest.mark.gpu

CTA = 16384   # offsets of one CTA


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _check(want, got, what):
    for w, g, name in zip(want, got, ("cue_offset", "n_segments", "split_score")):
        assert np.array_equal(np.asarray(w), np.asarray(g), equal_nan=True), (what, name, w, g)


def _device(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, d):
    import torch
    from ffsubsync_b200 import _native
    T = len(off) - 1
    outs = [torch.full((max(int(off[-1]), 1),), 7, dtype=torch.int32, device="cuda"),
            torch.full((T,), 7, dtype=torch.int32, device="cuda"),
            torch.zeros(T, dtype=torch.float64, device="cuda")]
    d_ref = torch.from_numpy(np.ascontiguousarray(ref)).cuda()
    handle.split_tracks_directed(d_ref.data_ptr(), f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, d,
                                 outs=[o.data_ptr() for o in outs], memspace=_native.B2_DEVICE)
    handle.synchronize()
    n = int(off[-1])
    return outs[0].cpu().numpy()[:n], outs[1].cpu().numpy(), outs[2].cpu().numpy()


def _both(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, d, what):
    """Host and device calls, each equal to the restatement; returns the host results."""
    want = sd.split_tracks(np.asarray(ref, np.float64), ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, d)
    got = handle.split_tracks_directed(ref, f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, d)
    _check(want, got, what + ("host",))
    _check(want, _device(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, d), what + ("device",))
    return got


@pytest.fixture(scope="module")
def envelope(handle):
    """The widest window b2_split_tracks_directed takes on this device, read from its refusal one past 16 clusters'
    worth; nothing is launched before that refusal."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(1)
    cs, ce = _few_cues(rng, 4, 20.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    R = 16 * CTA + 2000
    mos = _mos_for_width(R, S, 16 * CTA + 1)
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than (\d+)" % (16 * CTA + 1)) as e:
        handle.split_tracks_directed(np.zeros(R), True, [0, R], [0], cs, ce, None, [0, 4], [1.0], 100, 0.0, mos, 1.0,
                                     1)
    assert handle.launch_count == n0
    limit = int(re.search(r"wider than (\d+)", str(e.value)).group(1))
    assert limit % CTA == 0 and 2 * CTA <= limit <= 16 * CTA, limit
    return limit


@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("seed", range(4))
def test_directed_equals_restatement(handle, seed, d):
    """Seeded requests: two-level references (labels 0, 0.3, -0.5; float64 and float32), kept-cue masks, skipped
    tracks, ratios other than 1; windows of one and two CTAs; both memspaces; penalties that split and +inf."""
    label = [0.0, 0.3, -0.5][seed % 3]
    f64 = seed % 2 == 0
    for R, mos in ((1600 + 300 * seed, 500), (21000, 16384)):
        ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed, R=R, label=label, f64=f64)
        for pen in (0.0, 3.0, math.inf):
            got = _both(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, d, (seed, d, R, pen))
            assert np.all(got[1][~np.isnan(ratio)] >= 0)


@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("W", [9000, 2 * CTA, 8 * CTA, 16 * CTA])
@pytest.mark.parametrize("label,f64,ratio", [(0.0, True, 1.0), (0.3, False, 25 / 24.0)])
def test_wide_windows_equal_restatement(handle, envelope, W, label, f64, ratio, d):
    """Exact window widths of 1, 2, 8 and 16 CTAs (16: 262 144 offsets, when the device's envelope holds them),
    beside a short reference that clips the window; label 0.3 (beta != 0) with a ratio != 1 and float32, label 0 with
    float64; both memspaces."""
    if W > envelope:
        pytest.skip("%d offsets past this device's envelope of %d" % (W, envelope))
    rng = np.random.RandomState(W % 1000 + int(10 * label))
    cs, ce = _few_cues(rng, 7, 40.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, ratio)[0])
    R = W + 3000
    mos = _mos_for_width(R, S, W)
    ref = np.where(rng.rand(R) < 0.4, 1.0, label).astype(np.float64 if f64 else np.float32)
    short = np.where(rng.rand(9000) < 0.4, 1.0, label).astype(ref.dtype)
    both = np.concatenate([ref, short])
    ref_off = np.array([0, R, R + len(short)])
    off = np.array([0, 7, 14], np.int64)
    cs2, ce2 = np.concatenate([cs, cs]), np.concatenate([ce, ce])
    for pen in (0.0, 5.0):
        _both(handle, both, f64, ref_off, [0, 1], cs2, ce2, None, off, [ratio, ratio], mos, pen, d, (W, pen, d))


@pytest.mark.parametrize("d", [1, -1])
def test_ties_across_ctas(handle, envelope, d):
    """A reference periodic at 20 000 frames (more than one CTA's offsets): the units' prefix and suffix maxima are
    equal at offsets in different CTAs, and the rules (staying wins, records, the largest offset) decide as in the
    restatement."""
    rng = np.random.RandomState(5)
    P, reps = 20000, 5
    ref = np.tile((rng.rand(P) < 0.5).astype(np.float64), reps)
    R = len(ref)
    cs, ce = _few_cues(rng, 6, 30.0)
    mask = ro.rasterize(cs, ce, None, 100, 0, 1.0)[0] > 0
    S = len(mask)
    W = min(envelope, 4 * CTA)
    mos = _mos_for_width(R, S, W)
    o_lo, o_hi = ao.offset_range(R, S, mos)
    m, beta = sp.ref_levels(ref)
    units = sp.units_of(sp.runs_of(mask), S)
    import split_wide as sw
    U = sw.unit_table(m, units, list(range(o_lo, o_hi + 1)), sp.levels(1.0, beta))
    best = np.flatnonzero(U[0] == U[0].max())
    assert best.max() - best.min() >= CTA, best   # unit 0's maximum tied in different CTAs
    for pen in (math.inf, 4.0, 0.0):
        _both(handle, ref, True, [0, R], [0], cs, ce, None, [0, 6], [1.0], mos, pen, d, (pen, d))


@pytest.mark.parametrize("seed", range(3))
def test_infinite_penalty_equals_wide(handle, seed):
    """At penalty +inf the directed call never switches: every output equals b2_split_tracks_wide's, both memspaces."""
    label = [0.0, 0.3, -0.5][seed % 3]
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed + 30, R=3000 + 20000 * (seed % 2), label=label,
                                                          f64=True)
    mos = [300, 16384, 9000][seed]
    want = handle.split_tracks_wide(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, math.inf)
    for d in (1, -1):
        _check(want, handle.split_tracks_directed(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos,
                                                  math.inf, d), (seed, d, "host"))
        _check(want, _device(handle, ref, True, ref_off, tv, cs, ce, keep, off, ratio, mos, math.inf, d),
               (seed, d, "device"))


def _start_frames(cs, ratio, S):
    """Each cue's rasterised start frame, clamped into [0, S) as the kernels place cues."""
    f = np.array([int(round(ro.scale_seconds(float(c), ratio) * 100)) for c in cs])
    return np.clip(f, 0, S - 1)


def test_monotone_on_a_noisy_batch(handle):
    """Tracks over references with 10 % of their frames flipped, at penalties that split the undirected call many
    times: every track's cue offsets, in rasterised-start order, only grow (d = +1) or only shrink (d = -1), and equal
    the restatement."""
    refs, cs_all, ce_all, off = [], [], [], [0]
    for s, removal in enumerate((False, True, False, True)):
        ref, cs, ce, _ = _noisy_break(removal, n=80, cut=40, seed=20 + s)
        refs.append(ref)
        cs_all.append(cs)
        ce_all.append(ce)
        off.append(off[-1] + len(cs))
    ref = np.concatenate(refs)
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])])
    cs, ce, off = np.concatenate(cs_all), np.concatenate(ce_all), np.array(off, np.int64)
    tv = np.arange(4)
    ratio = np.array([1.0, 1.0, 25 / 24.0, 24 / 25.0])
    mos = 9800
    u = handle.split_tracks_wide(ref, True, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, 2.0)
    assert np.all(u[1] >= 10), u[1]
    for d in (1, -1):
        for pen in (0.0, 2.0):
            co, ns, _ = _both(handle, ref, True, ref_off, tv, cs, ce, None, off, ratio, mos, pen, d, (d, pen))
            for t in range(4):
                c = slice(off[t], off[t + 1])
                S = len(ro.rasterize(cs[c], ce[c], None, 100, 0, ratio[t])[0])
                order = np.argsort(_start_frames(cs[c], ratio[t], S), kind="stable")
                steps = np.diff(co[c][order])
                assert np.all(steps * d >= 0), (d, pen, t, co[c][order])


@pytest.mark.parametrize("removal", [True, False], ids=["removal", "insertion"])
def test_planted_edit(handle, removal):
    """A clean reference with 90 s of video removed (the subtitles' later cues sit 90 s earlier; found with d = -1) or
    90 s inserted (found with d = +1): exactly two segments at the planted offsets with the break at the planted cue,
    equal to the restatement; the wrong direction cannot reach the second offset; apply_split takes the result.  The
    removed stretch's cues have no speech anywhere in the video, so below a penalty of about 5 000 they take segments
    of their own at offsets between the two (2 000: three segments, in the restatement too)."""
    ref, cs, ce, parts = _noisy_break(removal, flip=0.0)
    R, off = len(ref), np.array([0, len(cs)], np.int64)
    d = -1 if removal else 1
    mos = 9800
    for pen in ((5000.0,) if removal else (200.0, 1000.0, 5000.0)):
        co, ns, sc = _both(handle, ref, True, [0, R], [0], cs, ce, None, off, [1.0], mos, pen, d, (removal, pen))
        assert ns[0] == 2, (pen, ns)
        for a, b, o in parts:
            assert np.all(co[a:b] == o), (pen, a, b, o, co)
        brk = int(np.flatnonzero(np.diff(co))[0]) + 1
        assert parts[0][1] <= brk <= parts[1][0], brk
        wrong = handle.split_tracks_directed(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, mos, pen, -d)
        assert not (np.all(wrong[0][parts[0][0]:parts[0][1]] == parts[0][2]) and
                    np.all(wrong[0][parts[1][0]:parts[1][1]] == parts[1][2]))
    su, eu, st = handle.apply_split([1.0], ns, co, cs, ce, off, 100)
    w = sp.apply_split([1.0], ns, co, cs, ce, off, 100)
    for x, y in zip(w, (su, eu, st)):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("d", [1, -1])
def test_three_cumulative_breaks(handle, envelope, d):
    """Three cumulative 4 min breaks in one direction on a clean reference: four segments at their exact offsets, the
    breaks at the planted cues."""
    steps = [300, 300 + 24000, 300 + 48000, 300 + 72000]
    shifts = steps if d > 0 else steps[::-1]
    ref, cs, ce, parts = _planted(shifts)
    R = len(ref)
    mos = max(shifts) + 500
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    o_lo, o_hi = ao.offset_range(R, S, mos)
    if o_hi - o_lo + 1 > envelope:
        pytest.skip("window of %d offsets past this device's envelope of %d" % (o_hi - o_lo + 1, envelope))
    off = np.array([0, len(cs)], np.int64)
    for pen in (10.0, 50.0):
        co, ns, sc = _both(handle, ref, True, [0, R], [0], cs, ce, None, off, [1.0], mos, pen, d, (d, pen))
        assert ns[0] == 4, (pen, ns)
        for i, o in enumerate(shifts):
            assert np.all(co[parts[i]:parts[i + 1]] == o), (pen, i, co)


def test_refusals(handle, envelope):
    """Directions other than +-1 are B2_ERR_BAD_ARG; the envelope runs and one more offset is B2_ERR_UNSUPPORTED
    naming it; nothing is launched before a refusal."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(3)
    cs, ce = _few_cues(rng, 3, 20.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    R = envelope + 2000
    ref = np.where(rng.rand(R) < 0.5, 1.0, 0.0)
    off = [0, 3]
    n0 = handle.launch_count
    for bad in (0, 2, -2):
        with pytest.raises(NativeError, match=r"B2_ERR_BAD_ARG.*direction %d must be \+1" % bad):
            handle.split_tracks_directed(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0, bad)
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than %d" % (envelope + 1, envelope)):
        handle.split_tracks_directed(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0,
                                     _mos_for_width(R, S, envelope + 1), 2.0, -1)
    assert handle.launch_count == n0
    mos = _mos_for_width(R, S, envelope)
    for d in (1, -1):
        _both(handle, ref, True, [0, R], [0], cs, ce, None, off, [1.0], mos, 2.0, d, ("envelope", d))


def test_dead_tracks_and_three_levels(handle):
    """Skipped (NaN ratio) tracks, an empty reference and a three-level video among live tracks: under B2_DEVICE the
    three-level video's tracks get n_segments == -1, the skipped ones 0, all of them NaN scores and offsets 0, the
    live ones the restatement's results; B2_HOST refuses the three-level video.  A zero window makes every track
    dead."""
    from ffsubsync_b200._native import NativeError
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(21, V=3, T=8, R=2200, label=0.3, f64=True)
    ref = ref.copy()
    bad_v = int(tv[-1])
    ref[ref_off[bad_v] + 77] = 0.6   # a third level
    ref_off = np.concatenate([ref_off, [ref_off[-1]]])   # an empty fourth video
    tv = tv.copy()
    tv[1] = 3
    ratio = ratio.copy()
    ratio[2] = np.nan
    ratio[-1] = 1.0
    mos = 400
    for d in (1, -1):
        co, ns, s = _device(handle, ref, True, ref_off, tv, cs, ce, keep, off, ratio, mos, 1.0, d)
        bad = (tv == bad_v) & ~np.isnan(ratio)
        dead = ((tv == 3) | np.isnan(ratio)) & ~bad
        assert bad.any() and dead.any() and (~bad & ~dead).any()
        assert np.all(ns[bad] == -1) and np.all(ns[dead] == 0)
        assert np.all(np.isnan(s[bad | dead]))
        assert np.all(co[np.repeat(bad | dead, np.diff(off))] == 0)
        sel = np.flatnonzero(~bad)
        sub_off = np.concatenate([[0], np.cumsum(np.diff(off)[sel])])
        idx = np.concatenate([np.arange(off[t], off[t + 1]) for t in sel])
        want = sd.split_tracks(ref, ref_off, tv[sel], cs[idx], ce[idx], keep[idx], sub_off, ratio[sel], 100, 0.0, mos,
                               1.0, d)
        _check(want, (co[idx], ns[sel], s[sel]), ("live", d))
        with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*video %d: frame 77" % bad_v):
            handle.split_tracks_directed(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, 1.0, d)
        ok = ref.copy()
        ok[ref_off[bad_v] + 77] = 0.3
        got = handle.split_tracks_directed(ok, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, 0, 1.0, d)
        assert np.all(got[1] == 0) and np.all(np.isnan(got[2])) and not got[0].any()


def test_batch_split_direction():
    """BatchSynchronizer.split_tracks / split_tracks_host with split_direction after sync_device_tracks,
    sync_host_tracks and an ingest session, at the sync window and at split_max_offset_seconds: equal to the
    restatement; apply_split and apply_split_host take the results; max_segments with split_direction and a bad
    direction raise ValueError."""
    import torch
    from ffsubsync_b200.batch import DEFAULT_APPLY_OFFSET_SECONDS, BatchSynchronizer
    GRID = [1.0, 25 / 24.0, 24 / 25.0]
    rng = np.random.RandomState(29)
    c = _sig_corpus([(200.0 + 7 * v, "audio", [(GRID[int(rng.randint(0, 3))], int(rng.randint(-700, 700)))
                                               for _ in range(1 + v % 2)]) for v in range(4)], seed0=17)
    V = len(c["pcm_off"]) - 1
    sv = np.arange(V)
    s = BatchSynchronizer(GRID, non_speech_label=0.0, max_offset_seconds=8)
    args = (c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])
    names = ("cue_offset", "n_segments", "split_score")

    def oracle(speech, speech_off, ratio, mos, pen, d):
        return sd.split_tracks(np.asarray(speech, np.float64), speech_off, c["track_video"], c["cue_start"],
                               c["cue_end"], None, c["cue_off"], ratio, 100, 0.0, mos, pen, d)

    host = s.sync_host_tracks(c["pcm"], c["pcm_off"], *args, speech_video=sv)
    out = s.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], *args, speech_video=sv)
    for secs, d in ((None, 1), (150.0, -1)):
        mos = s.max_offset_samples if secs is None else abs(int(secs * s.sample_rate))
        pen = 5.0
        h = s.split_tracks_host(host, *args, split_penalty=pen, split_max_offset_seconds=secs, split_direction=d)
        _check(oracle(host[-2], host[-1], h["ratio"], mos, pen, d), [h[k] for k in names], (secs, d, "host"))
        dv = s.split_tracks(out, *args, split_penalty=pen, split_max_offset_seconds=secs, split_direction=d)
        a = s.apply_split(dv, c["cue_start"], c["cue_end"], c["cue_off"])
        torch.cuda.synchronize()
        dn = [dv[k].cpu().numpy() for k in names]
        _check(oracle(out["speech"].cpu().numpy(), out["speech_off"], dv["ratio"], mos, pen, d), dn, (secs, d))
        want = sp.apply_split(dv["ratio"], dn[1], dn[0], c["cue_start"], c["cue_end"], c["cue_off"], 100,
                              DEFAULT_APPLY_OFFSET_SECONDS)
        ah = s.apply_split_host(h, c["cue_start"], c["cue_end"], c["cue_off"])
        wh = sp.apply_split(h["ratio"], h["n_segments"], h["cue_offset"], c["cue_start"], c["cue_end"], c["cue_off"],
                            100, DEFAULT_APPLY_OFFSET_SECONDS)
        for k, w, x in zip(("synced_start_us", "synced_end_us", "status"), want, wh):
            assert np.array_equal(a[k].cpu().numpy(), w) and np.array_equal(ah[k], x), k
    with pytest.raises(ValueError, match="cannot be combined"):
        s.split_tracks(out, *args, split_penalty=5.0, max_segments=2, split_direction=1)
    with pytest.raises(ValueError, match="cannot be combined"):
        s.split_tracks_host(host, *args, split_penalty=5.0, max_segments=2, split_direction=-1)
    with pytest.raises(ValueError, match="split_direction must be"):
        s.split_tracks(out, *args, split_penalty=5.0, split_direction=0)
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
    dv = s.split_tracks(o, *args, split_penalty=5.0, split_max_offset_seconds=300.0, split_direction=1)
    torch.cuda.synchronize()
    dn = [dv[k].cpu().numpy() for k in names]
    assert np.any(dn[1] > 0)
    _check(oracle(o["speech"].cpu().numpy(), o["speech_off"], dv["ratio"], 30000, 5.0, 1), dn, "ingest")


def test_envelope_report(envelope):
    """The directed kernel's widest window on this device (for the record)."""
    print("directed split: widest cluster %d CTAs, %d offsets" % (envelope // CTA, envelope))
    assert CTA <= envelope <= 16 * CTA
