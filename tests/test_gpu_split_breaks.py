"""GPU tests of the split along stated breaks (b2_split_tracks_breaks: at most n breaks, the i-th moving the offset the
i-th stated way, with the best objective at every exact break count; run on an H100).

Yardsticks: the restatement (tests/split_breaks.py, itself held to exhaustive enumeration of pattern-following paths,
to oracle/split_oracle.py at penalty +inf and to the directed restatement on uniform patterns) bit for bit, cells
through split_profile, paths through cue_offset and n_segments, and split_score; b2_split_tracks_wide at penalty +inf;
b2_split_tracks_directed on uniform patterns.  Also windows of 1 to 16 CTAs, ties across threads and CTAs, planted
breaks on a noisy reference, dead and three-level tracks, the refusals, and
BatchSynchronizer.split_tracks(split_breaks=...)."""
import math
import re

import numpy as np
import pytest

import split_breaks as sb
import split_directed as sd
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import split_oracle as sp
from test_gpu_sig_ref import _sig_corpus
from test_gpu_split import _request
from test_gpu_split_capped import _noisy_break
from test_gpu_split_wide import _few_cues, _mos_for_width, _planted

pytestmark = pytest.mark.gpu

PATTERNS = [(-1,), (1,), (1, -1), (1, 1, 1), (-1, 1, -1, 1, 1, -1, -1), (1, -1) * 7 + (1,)]


def _cta(nb):
    """Offsets of one CTA at nb breaks: 512 threads of 32 // (nb + 1) offsets."""
    return 512 * (32 // (nb + 1))


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _check(want, got, what):
    for w, g, name in zip(want, got, ("cue_offset", "n_segments", "split_score", "split_profile")):
        assert np.array_equal(np.asarray(w), np.asarray(g), equal_nan=True), (what, name, w, g)


def _device(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, breaks):
    import torch
    from ffsubsync_b200 import _native
    T = len(off) - 1
    outs = [torch.full((max(int(off[-1]), 1),), 7, dtype=torch.int32, device="cuda"),
            torch.full((T,), 7, dtype=torch.int32, device="cuda"),
            torch.zeros(T, dtype=torch.float64, device="cuda"),
            torch.full((T, len(breaks) + 1), 7.0, dtype=torch.float64, device="cuda")]
    d_ref = torch.from_numpy(np.ascontiguousarray(ref)).cuda()
    handle.split_tracks_breaks(d_ref.data_ptr(), f64, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen, breaks,
                               outs=[o.data_ptr() for o in outs], memspace=_native.B2_DEVICE)
    handle.synchronize()
    n = int(off[-1])
    return outs[0].cpu().numpy()[:n], outs[1].cpu().numpy(), outs[2].cpu().numpy(), outs[3].cpu().numpy()


def _both(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, breaks, what):
    """Host and device calls, each equal to the restatement; returns the host results."""
    want = sb.split_tracks(np.asarray(ref, np.float64), ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, pen,
                           breaks)
    got = handle.split_tracks_breaks(ref, True if f64 else False, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos,
                                     pen, breaks)
    _check(want, got, what + ("host",))
    _check(want, _device(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, breaks),
           what + ("device",))
    return got


_ENVELOPES = {}


def _envelope(handle, nb):
    """The widest window b2_split_tracks_breaks takes at nb breaks on this device, read from its refusal one past 16
    CTAs' worth; nothing is launched before that refusal."""
    if nb in _ENVELOPES:
        return _ENVELOPES[nb]
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(1)
    cs, ce = _few_cues(rng, 4, 20.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    W = 16 * _cta(nb) + 1
    R = W + 2000
    mos = _mos_for_width(R, S, W)
    n0 = handle.launch_count
    with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than (\d+), the widest at %d "
                                          r"breaks" % (W, nb)) as e:
        handle.split_tracks_breaks(np.zeros(R), True, [0, R], [0], cs, ce, None, [0, 4], [1.0], 100, 0.0, mos, 1.0,
                                   (1,) * nb)
    assert handle.launch_count == n0
    limit = int(re.search(r"wider than (\d+)", str(e.value)).group(1))
    assert limit % _cta(nb) == 0 and _cta(nb) <= limit <= 16 * _cta(nb), (nb, limit)
    _ENVELOPES[nb] = limit
    return limit


@pytest.mark.parametrize("breaks", PATTERNS, ids=lambda b: "".join("+" if d > 0 else "-" for d in b))
@pytest.mark.parametrize("seed", range(3))
def test_breaks_equal_restatement(handle, seed, breaks):
    """Seeded requests: two-level references (labels 0, 0.3, -0.5; float64 and float32), kept-cue masks, skipped
    tracks, ratios other than 1; a short window and one of several CTAs; both memspaces; penalties that split and
    +inf."""
    label = [0.0, 0.3, -0.5][seed % 3]
    f64 = seed % 2 == 0
    for R, mos in ((1600 + 300 * seed, 500), (21000, 6000)):
        ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed, R=R, label=label, f64=f64)
        for pen in (0.0, 3.0, math.inf):
            got = _both(handle, ref, f64, ref_off, tv, cs, ce, keep, off, ratio, mos, pen, breaks,
                        (seed, breaks, R, pen))
            live = got[1] > 0
            assert np.all(got[1][live] <= len(breaks) + 1)


@pytest.mark.parametrize("ctas", [1, 2, 8, 16])
@pytest.mark.parametrize("nb", [1, 2, 3, 7, 15])
@pytest.mark.parametrize("label,f64,ratio", [(0.0, True, 1.0), (0.3, False, 25 / 24.0)])
def test_windows_of_1_to_16_ctas(handle, nb, ctas, label, f64, ratio):
    """Exact window widths of 1, 2, 8 and 16 CTAs at 1, 2, 3, 7 and 15 breaks (when the device's envelope holds
    them), beside a short reference that clips the window; label 0.3 (beta != 0) with a ratio != 1 and float32, label
    0 with float64; cue tables starting past cue 0; both memspaces."""
    W = ctas * _cta(nb)
    if W > _envelope(handle, nb):
        pytest.skip("%d offsets past this device's envelope at %d breaks" % (W, nb))
    rng = np.random.RandomState(W % 1000 + nb + int(10 * label))
    span = min(40.0, W / 300.0)   # seconds: the mask within a third of the window, so its width is exact
    cs = np.sort(np.round(rng.uniform(0.2, 0.7 * span, 7), 2))
    ce = np.round(cs + rng.uniform(0.05, 0.3 * span, 7), 2)
    S = len(ro.rasterize(cs, ce, None, 100, 0, ratio)[0])
    R = W + 3000
    mos = _mos_for_width(R, S, W)
    ref = np.where(rng.rand(R) < 0.4, 1.0, label).astype(np.float64 if f64 else np.float32)
    short = np.where(rng.rand(9000) < 0.4, 1.0, label).astype(ref.dtype)
    both = np.concatenate([ref, short])
    ref_off = np.array([0, R, R + len(short)])
    junk = np.array([0.5, 2.5])   # cues the call does not own: its tables start at cue 2
    off = np.array([2, 9, 16], np.int64)
    cs2, ce2 = np.concatenate([junk, cs, cs]), np.concatenate([junk + 1, ce, ce])
    breaks = tuple(int(x) for x in rng.choice([1, -1], nb))
    for pen in (0.0, 5.0):
        want = sb.split_tracks(np.asarray(both, np.float64), ref_off - 0, [0, 1], cs2[2:], ce2[2:], None, off - 2,
                               [ratio, ratio], 100, 0.0, mos, pen, breaks)
        got = handle.split_tracks_breaks(both, f64, ref_off, [0, 1], cs2, ce2, None, off, [ratio, ratio], 100, 0.0,
                                         mos, pen, breaks)
        _check((want[0],), (got[0][2:],), (nb, ctas, pen, "host cues"))
        _check(want[1:], got[1:], (nb, ctas, pen, "host"))
        dev = _device(handle, both, f64, ref_off, [0, 1], cs2, ce2, None, off, [ratio, ratio], mos, pen, breaks)
        _check((want[0],), (dev[0][2:],), (nb, ctas, pen, "device cues"))
        _check(want[1:], dev[1:], (nb, ctas, pen, "device"))


@pytest.mark.parametrize("breaks", [(1,), (-1,), (1, -1, 1), (-1,) * 7])
def test_ties_across_threads_and_ctas(handle, breaks):
    """A reference periodic at 2 000 frames, shorter than one CTA's offsets and a multiple of every thread's: the
    layers' prefix and suffix maxima tie at offsets in different threads and CTAs, and the rules (staying wins,
    records, the largest offset, then the smallest layer) decide as in the restatement."""
    nb = len(breaks)
    rng = np.random.RandomState(5 + nb)
    P, reps = 2000, 45
    ref = np.tile((rng.rand(P) < 0.5).astype(np.float64), reps)
    R = len(ref)
    cs, ce = _few_cues(rng, 6, 15.0)
    mask = ro.rasterize(cs, ce, None, 100, 0, 1.0)[0] > 0
    S = len(mask)
    W = min(_envelope(handle, nb), 4 * _cta(nb))
    mos = _mos_for_width(R, S, W)
    o_lo, o_hi = ao.offset_range(R, S, mos)
    m, beta = sp.ref_levels(ref)
    units = sp.units_of(sp.runs_of(mask), S)
    import split_wide as sw
    U = sw.unit_table(m, units, list(range(o_lo, o_hi + 1)), sp.levels(1.0, beta))
    best = np.flatnonzero(U[0] == U[0].max())
    assert best.max() - best.min() >= _cta(nb), best   # unit 0's maximum tied in different CTAs
    for pen in (math.inf, 4.0, 0.0):
        _both(handle, ref, True, [0, R], [0], cs, ce, None, [0, 6], [1.0], mos, pen, breaks, (pen, breaks))


@pytest.mark.parametrize("seed", range(3))
def test_infinite_penalty_equals_wide(handle, seed):
    """At penalty +inf the call never breaks: cue_offset, n_segments and split_score equal b2_split_tracks_wide's,
    split_profile[:, 0] is finite on live tracks and the other columns -inf; both memspaces."""
    label = [0.0, 0.3, -0.5][seed % 3]
    ref, ref_off, tv, cs, ce, keep, off, ratio = _request(seed + 30, R=3000 + 20000 * (seed % 2), label=label,
                                                          f64=True)
    mos = [300, 6000, 9000][seed]
    want = handle.split_tracks_wide(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, math.inf)
    for breaks in ((1,), (-1, 1), (1, 1, -1, -1, 1)):
        for got in (handle.split_tracks_breaks(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos,
                                               math.inf, breaks),
                    _device(handle, ref, True, ref_off, tv, cs, ce, keep, off, ratio, mos, math.inf, breaks)):
            _check(want, got[:3], (seed, breaks))
            live = got[1] > 0
            assert live.any()
            assert np.all(np.isfinite(got[3][live, 0])) and np.all(got[3][live, 1:] == -np.inf)
            assert np.all(np.isnan(got[3][~live]))


@pytest.mark.parametrize("d", [1, -1])
@pytest.mark.parametrize("seed", range(4))
def test_uniform_pattern_equals_directed(handle, seed, d):
    """(d,) * n on tracks of at most n + 1 units (a few cues each), with +-1 signals so every value is an integer: the
    largest split_profile entry is the directed optimum, split_score - penalty x (n_segments - 1) of the directed call;
    wherever the two restatements choose the same path, the two GPU calls return the same outputs."""
    rng = np.random.RandomState(400 + seed)
    T = 6
    cs, ce, off = [], [], [0]
    for t in range(T):
        k = int(rng.randint(1, 5))
        a, b = _few_cues(rng, k, 12.0)
        cs.append(a)
        ce.append(b)
        off.append(off[-1] + k)
    cs, ce, off = np.concatenate(cs), np.concatenate(ce), np.array(off, np.int64)
    R = 2500
    ref = (rng.rand(2 * R) < 0.5).astype(np.float64)
    ref_off, tv, ratio = [0, R, 2 * R], np.arange(T) % 2, np.ones(T)
    nb = 5   # at least the units of every track less one (k cues make at most k units)
    mos = 700
    for pen in (0.0, 2.0, 7.0):
        got = _both(handle, ref, True, ref_off, tv, cs, ce, None, off, ratio, mos, pen, (d,) * nb, (seed, d, pen))
        dg = handle.split_tracks_directed(ref, True, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, d)
        want_b = sb.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, (d,) * nb)
        want_d = sd.split_tracks(ref, ref_off, tv, cs, ce, None, off, ratio, 100, 0.0, mos, pen, d)
        for t in range(T):
            assert got[3][t].max() == dg[2][t] - pen * (dg[1][t] - 1), (seed, d, pen, t)
            c = slice(off[t], off[t + 1])
            if np.array_equal(want_b[0][c], want_d[0][c]) and want_b[1][t] == want_d[1][t]:
                assert np.array_equal(got[0][c], dg[0][c]) and got[1][t] == dg[1][t] and got[2][t] == dg[2][t]


def _flip(ref, frac, seed):
    ref = ref.copy()
    fl = np.random.RandomState(seed).rand(len(ref)) < frac
    ref[fl] = 1.0 - ref[fl]
    return ref


def _planted_check(handle, ref, cs, ce, parts, mos, pen, breaks):
    R, off = len(ref), np.array([0, len(cs)], np.int64)
    co, ns, sc, pr = _both(handle, ref, True, [0, R], [0], cs, ce, None, off, [1.0], mos, pen, breaks,
                           ("planted", breaks, pen))
    return co, ns, pr


def test_planted_removal(handle):
    """90 s of video removed and 10 % of the reference's frames flipped: (-1,) at penalty 2 returns exactly the two
    planted offsets, the break inside the removed stretch, and the profile gains from the break; apply_split takes
    the result."""
    ref, cs, ce, parts = _noisy_break(True)
    co, ns, pr = _planted_check(handle, ref, cs, ce, parts, 9800, 2.0, (-1,))
    assert ns[0] == 2, ns
    for a, b, o in parts:
        assert np.all(co[a:b] == o), (a, b, o, co)
    brk = int(np.flatnonzero(np.diff(co))[0]) + 1
    assert parts[0][1] <= brk <= parts[1][0], brk
    assert pr[0, 1] > pr[0, 0]
    off = np.array([0, len(cs)], np.int64)
    su, eu, st = handle.apply_split([1.0], ns, co, cs, ce, off, 100)
    w = sp.apply_split([1.0], ns, co, cs, ce, off, 100)
    for x, y in zip(w, (su, eu, st)):
        assert np.array_equal(x, y)


def test_planted_three_ad_breaks(handle):
    """Three 60 s ad breaks (offsets growing three times) and 10 % of the frames flipped: (+1,) * 3 returns four
    segments at their exact offsets, the breaks at the planted cues."""
    shifts = [300, 300 + 6000, 300 + 12000, 300 + 18000]
    ref, cs, ce, parts = _planted(shifts)
    ref = _flip(ref, 0.1, 11)
    co, ns, pr = _planted_check(handle, ref, cs, ce, parts, max(shifts) + 500, 2.0, (1, 1, 1))
    assert ns[0] == 4, ns
    for i, o in enumerate(shifts):
        assert np.all(co[parts[i]:parts[i + 1]] == o), (i, co)
    assert np.all(np.diff(pr[0]) > 0), pr


def test_planted_removal_then_insertion(handle):
    """A removal (the offset falls by 120 s) followed by an insertion (it grows by 90 s), 10 % of the frames flipped:
    (-1, +1) returns the three planted offsets; the profile gains at each break."""
    shifts = [12300, 300, 9300]
    ref, cs, ce, parts = _planted(shifts, n=45)
    ref = _flip(ref, 0.1, 12)
    co, ns, pr = _planted_check(handle, ref, cs, ce, parts, max(shifts) + 500, 2.0, (-1, 1))
    assert ns[0] == 3, ns
    for i, o in enumerate(shifts):
        assert np.all(co[parts[i]:parts[i + 1]] == o), (i, co)
    assert pr[0, 2] > pr[0, 1] > pr[0, 0], pr


def test_refusals(handle):
    """n_breaks < 1 and entries other than +-1 are B2_ERR_BAD_ARG, 16 breaks B2_ERR_UNSUPPORTED; one offset past the
    envelope is B2_ERR_UNSUPPORTED naming it, and the envelope itself runs; nothing is launched before a refusal.  The
    envelope holds the capped call's at the same number of layers: 16 layers at +-60 s, 8 at +-150 s (100 Hz)."""
    from ffsubsync_b200._native import NativeError
    rng = np.random.RandomState(3)
    cs, ce = _few_cues(rng, 3, 20.0)
    S = len(ro.rasterize(cs, ce, None, 100, 0, 1.0)[0])
    assert _envelope(handle, 15) >= 12001 and _envelope(handle, 7) >= 30001
    R = 4000
    ref = np.where(rng.rand(R) < 0.5, 1.0, 0.0)
    off = [0, 3]
    n0 = handle.launch_count
    for bad, what in (((), "n_breaks 0 must be"), ((1, 0), r"breaks\[1\] = 0 must be"),
                      ((2,), r"breaks\[0\] = 2 must be"), ((-1, 1, -3), r"breaks\[2\] = -3 must be")):
        with pytest.raises(NativeError, match="B2_ERR_BAD_ARG.*" + what):
            handle.split_tracks_breaks(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0, bad)
    with pytest.raises(NativeError, match="B2_ERR_UNSUPPORTED.*16 breaks is more than 15"):
        handle.split_tracks_breaks(ref, True, [0, R], [0], cs, ce, None, off, [1.0], 100, 0.0, 100, 1.0, (1,) * 16)
    for nb in (1, 4, 15):
        env = _envelope(handle, nb)
        Rw = env + 2000
        refw = np.where(rng.rand(Rw) < 0.5, 1.0, 0.0)
        with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*%d offsets is wider than %d, the widest at %d "
                                              r"breaks" % (env + 1, env, nb)):
            handle.split_tracks_breaks(refw, True, [0, Rw], [0], cs, ce, None, off, [1.0], 100, 0.0,
                                       _mos_for_width(Rw, S, env + 1), 2.0, (-1,) * nb)
        assert handle.launch_count == n0
    nb = 4
    env = _envelope(handle, nb)
    Rw = env + 2000
    refw = np.where(rng.rand(Rw) < 0.5, 1.0, 0.0)
    _both(handle, refw, True, [0, Rw], [0], cs, ce, None, off, [1.0], _mos_for_width(Rw, S, env), 2.0,
          (1, -1, 1, -1), ("envelope",))


def test_dead_tracks_and_three_levels(handle):
    """Skipped (NaN ratio) tracks, an empty reference and a three-level video among live tracks: under B2_DEVICE the
    three-level video's tracks get n_segments == -1, the skipped ones 0, all of them NaN scores and profile rows and
    offsets 0, the live ones the restatement's results; B2_HOST refuses the three-level video.  A zero window makes
    every track dead."""
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
    for breaks in ((1, -1), (-1,) * 9):
        co, ns, s, pr = _device(handle, ref, True, ref_off, tv, cs, ce, keep, off, ratio, mos, 1.0, breaks)
        bad = (tv == bad_v) & ~np.isnan(ratio)
        dead = ((tv == 3) | np.isnan(ratio)) & ~bad
        assert bad.any() and dead.any() and (~bad & ~dead).any()
        assert np.all(ns[bad] == -1) and np.all(ns[dead] == 0)
        assert np.all(np.isnan(s[bad | dead])) and np.all(np.isnan(pr[bad | dead]))
        assert np.all(co[np.repeat(bad | dead, np.diff(off))] == 0)
        sel = np.flatnonzero(~bad)
        sub_off = np.concatenate([[0], np.cumsum(np.diff(off)[sel])])
        idx = np.concatenate([np.arange(off[t], off[t + 1]) for t in sel])
        want = sb.split_tracks(ref, ref_off, tv[sel], cs[idx], ce[idx], keep[idx], sub_off, ratio[sel], 100, 0.0, mos,
                               1.0, breaks)
        _check(want, (co[idx], ns[sel], s[sel], pr[sel]), ("live", breaks))
        with pytest.raises(NativeError, match=r"B2_ERR_UNSUPPORTED.*video %d: frame 77" % bad_v):
            handle.split_tracks_breaks(ref, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, mos, 1.0, breaks)
        ok = ref.copy()
        ok[ref_off[bad_v] + 77] = 0.3
        got = handle.split_tracks_breaks(ok, True, ref_off, tv, cs, ce, keep, off, ratio, 100, 0.0, 0, 1.0, breaks)
        assert np.all(got[1] == 0) and np.all(np.isnan(got[2])) and not got[0].any() and np.all(np.isnan(got[3]))


def test_batch_split_breaks():
    """BatchSynchronizer.split_tracks / split_tracks_host with split_breaks after sync_device_tracks,
    sync_host_tracks and an ingest session, at the sync window and at split_max_offset_seconds: equal to the
    restatement, split_profile included; apply_split and apply_split_host take the results; split_breaks with
    max_segments or split_direction, and a bad pattern, raise ValueError; split_breaks=None keeps the plain call."""
    import torch
    from ffsubsync_b200.batch import DEFAULT_APPLY_OFFSET_SECONDS, BatchSynchronizer
    GRID = [1.0, 25 / 24.0, 24 / 25.0]
    rng = np.random.RandomState(31)
    c = _sig_corpus([(200.0 + 7 * v, "audio", [(GRID[int(rng.randint(0, 3))], int(rng.randint(-700, 700)))
                                               for _ in range(1 + v % 2)]) for v in range(4)], seed0=19)
    V = len(c["pcm_off"]) - 1
    sv = np.arange(V)
    s = BatchSynchronizer(GRID, non_speech_label=0.0, max_offset_seconds=8)
    args = (c["track_video"], c["cue_start"], c["cue_end"], c["cue_off"])
    names = ("cue_offset", "n_segments", "split_score", "split_profile")

    def oracle(speech, speech_off, ratio, mos, pen, breaks):
        return sb.split_tracks(np.asarray(speech, np.float64), speech_off, c["track_video"], c["cue_start"],
                               c["cue_end"], None, c["cue_off"], ratio, 100, 0.0, mos, pen, breaks)

    host = s.sync_host_tracks(c["pcm"], c["pcm_off"], *args, speech_video=sv)
    out = s.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], *args, speech_video=sv)
    for secs, breaks in ((None, (1,)), (150.0, (-1, 1)), (60.0, [1, 1, 1])):
        mos = s.max_offset_samples if secs is None else abs(int(secs * s.sample_rate))
        pen = 5.0
        h = s.split_tracks_host(host, *args, split_penalty=pen, split_max_offset_seconds=secs, split_breaks=breaks)
        assert h["split_profile"].shape == (len(c["track_video"]), len(breaks) + 1)
        _check(oracle(host[-2], host[-1], h["ratio"], mos, pen, tuple(breaks)), [h[k] for k in names],
               (secs, breaks, "host"))
        dv = s.split_tracks(out, *args, split_penalty=pen, split_max_offset_seconds=secs, split_breaks=breaks)
        a = s.apply_split(dv, c["cue_start"], c["cue_end"], c["cue_off"])
        torch.cuda.synchronize()
        dn = [dv[k].cpu().numpy() for k in names]
        _check(oracle(out["speech"].cpu().numpy(), out["speech_off"], dv["ratio"], mos, pen, tuple(breaks)), dn,
               (secs, breaks))
        want = sp.apply_split(dv["ratio"], dn[1], dn[0], c["cue_start"], c["cue_end"], c["cue_off"], 100,
                              DEFAULT_APPLY_OFFSET_SECONDS)
        ah = s.apply_split_host(h, c["cue_start"], c["cue_end"], c["cue_off"])
        wh = sp.apply_split(h["ratio"], h["n_segments"], h["cue_offset"], c["cue_start"], c["cue_end"], c["cue_off"],
                            100, DEFAULT_APPLY_OFFSET_SECONDS)
        for k, w, x in zip(("synced_start_us", "synced_end_us", "status"), want, wh):
            assert np.array_equal(a[k].cpu().numpy(), w) and np.array_equal(ah[k], x), k
    plain = s.split_tracks_host(host, *args, split_penalty=5.0, split_breaks=None)
    assert "split_profile" not in plain
    for kw in ({"max_segments": 2}, {"split_direction": 1}):
        with pytest.raises(ValueError, match="cannot be combined"):
            s.split_tracks(out, *args, split_penalty=5.0, split_breaks=(1,), **kw)
        with pytest.raises(ValueError, match="cannot be combined"):
            s.split_tracks_host(host, *args, split_penalty=5.0, split_breaks=(-1,), **kw)
    for bad in ((), (0,), (True,)):
        with pytest.raises(ValueError, match="split_breaks"):
            s.split_tracks(out, *args, split_penalty=5.0, split_breaks=bad)
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
    dv = s.split_tracks(o, *args, split_penalty=5.0, split_max_offset_seconds=150.0, split_breaks=(1, -1))
    torch.cuda.synchronize()
    dn = [dv[k].cpu().numpy() for k in names]
    assert np.any(dn[1] > 0)
    _check(oracle(o["speech"].cpu().numpy(), o["speech_off"], dv["ratio"], 15000, 5.0, (1, -1)), dn, "ingest")


def test_envelope_report(handle):
    """The kernel's widest window at every break count on this device (for the record)."""
    for nb in range(1, 16):
        env = _envelope(handle, nb)
        print("split along %d breaks: %d offsets a CTA, widest cluster %d CTAs, %d offsets" %
              (nb, _cta(nb), env // _cta(nb), env))
        assert _cta(nb) <= env <= 16 * _cta(nb)
