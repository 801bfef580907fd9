"""The run path of the aligner (csrc/runcorr.cu) checked at EVERY offset of the window against exact
integer counts.

Under B2_ALIGN_PATH=runs, b2_capture_nominations records what run_corr_kernel scored (its float64 score
at every offset, rounded to float32), the job's (maximum, epsilon) and the candidate count.  The oracle
builds the same score from the four overlap counts in int64:
    c11 = sum_j u[j] m[j + o] (FFT correlation of the 0/1 arrays, rounded), Mwin and Uov from prefix sums,
    score = hi*c11 - c01 + hi*alpha*c10 - alpha*c00
with m = (VAD output == 1.0f) of the same PCM (oracle/vad_oracle.py) and u the oracle's cue raster.  Per job:
  * the window equals aligner_oracle.offset_range;
  * +-1 jobs (level 1, label 0) score the exact integer at every offset; all others stay within eps / 2
    (plus half a float32 ulp of the score);
  * the captured maximum is the row's maximum and epsilon is rc_eps(min(R, S)), recomputed here;
  * the candidate count lies between #{exact >= max} and #{exact >= max - 2 eps} (exact for +-1 jobs) and
    is -1 exactly where winner-only pruning must drop the ratio;
  * the per-ratio outputs of a call without capture pick the exact maximum among the 32 largest-offset
    nominees (ties: the largest offset) and equal B2_ALIGN_PATH=tiled bit for bit wherever the tiled
    capture nominates at most 32 offsets.
The shapes sit where this kernel can go wrong: window widths around lane, warp and CTA sizes (up to
1 024 threads in one call with narrow jobs, so that most CTAs have idle threads), windows that run off
both ends of the reference, lengths around word boundaries, run counts around the 4-bit counter flushes,
the largest run table, references that fill the counters, ties across lane and warp boundaries, plateaus
of 32 and 33 tied offsets, and the winner-only pruning around equal maxima."""
import contextlib
import os
import time

import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

FPW = 160
K_CAND = 32
BENCH = [1.0, 24.0 / 23.976, 25.0 / 24.0, 23.976 / 24.0, 24.0 / 25.0]
LEVEL_RATIOS = BENCH + [2.0, 4.0]   # levels 0.5 (hi = 0) and 0.25 (hi = -0.5)
LABELS = [0.0, 0.3, 0.5, 1.0, -0.5]


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module", autouse=True)
def report_time():
    t0 = time.time()
    yield
    print("test_gpu_runcorr_exact: %.1f s" % (time.time() - t0))


@contextlib.contextmanager
def _env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ------------------------------------------------------------------------------------------ inputs

def _cues(runs, S=None):
    """Cue list whose raster at ratio 1 is the frame runs [a, b) (times 0.3 frame early, so that round()
    lands on a and b and the last run may end at S - 1, the last frame a cue can reach).  S: mask length,
    set by one extra cue that cue_keep drops (then every run must end by S - 2)."""
    st = [0.0 if a == 0 else (a - 0.3) / 100.0 for a, _ in runs]
    en = [(b - 0.3) / 100.0 for _, b in runs]
    keep = [1] * len(runs)
    if S is not None:
        assert all(b <= S - 2 for _, b in runs), S
        st.append((S - 3.5) / 100.0)
        en.append((S - 1.5) / 100.0)
        keep.append(0)
    return dict(st=np.array(st, np.float64), en=np.array(en, np.float64), keep=np.array(keep, np.uint8))


def _track(v, runs=(), S=None, **kw):
    t = _cues(list(runs), S)
    t.update(kw)
    t["video"] = v
    return t


def _pcm(handle, cls, seed, tail=0):
    """PCM of the window classes (0 silence, 1 speech, 2 hiss) and `tail` samples of a partial last window."""
    cls = np.asarray(cls, np.uint8)
    if tail:
        cls = np.concatenate([cls, [1]]).astype(np.uint8)
    pcm = handle.synth_pcm(cls, len(cls), FPW, seed)
    return pcm[: len(pcm) - (FPW - tail)] if tail else pcm


def _mask_cls(m, rng, hiss=0.05):
    """Window classes whose VAD output is the 0/1 array m (speech where m, silence or hiss elsewhere)."""
    m = np.asarray(m, bool)
    return np.where(m, 1, np.where(rng.rand(len(m)) < hiss, 2, 0)).astype(np.uint8)


def _vad(pcm, label):
    """The oracle VAD in 60 s pieces (windows are independent; memory stays small for 2 h inputs)."""
    step = 6000 * FPW
    parts = [vo.energy_zcr_detect(pcm[i:i + step], 100, 16000, label) for i in range(0, len(pcm), step)]
    return np.concatenate(parts) if parts else np.zeros(0)


def _raster(t, ratio, start_seconds):
    return ro.rasterize(t["st"], t["en"], t["keep"].astype(bool), 100, start_seconds, ratio)[0]


# ------------------------------------------------------------------------------------------ oracle

def _xcorr_int(u, m, o_lo, W):
    """c[o] = sum_j u[j] m[j + o] for o = o_lo .. o_lo + W - 1, exact (int64)."""
    S, R = len(u), len(m)
    n = 1
    while n < R + S:
        n *= 2
    fu = np.fft.rfft(u.astype(np.float64)[::-1], n)
    fm = np.fft.rfft(m.astype(np.float64), n)
    full = np.rint(np.fft.irfft(fu * fm, n)).astype(np.int64)  # full[k] = sum_j u[j] m[k - (S-1) + j]
    o = np.arange(o_lo, o_lo + W, dtype=np.int64)
    idx = o + S - 1
    ok = (o < R) & (o > -S)
    out = np.zeros(W, np.int64)
    out[ok] = full[idx[ok]]
    return out


class _Job:
    """Exact scores of one (track, ratio) job over its window."""

    def __init__(self, m, u, level, label, mos):
        self.R, self.S = len(m), len(u)
        self.hi = 2.0 * float(np.float32(level)) - 1.0
        self.alpha = 2.0 * float(np.float32(label)) - 1.0
        self.pm1 = self.hi == 1.0 and self.alpha == -1.0
        self.o_lo, self.o_hi = ao.offset_range(self.R, self.S, mos)
        self.live = self.R > 0 and self.S > 0 and self.o_lo <= self.o_hi
        self.m, self.u = m, u
        if not self.live:
            return
        W = self.o_hi - self.o_lo + 1
        o = np.arange(self.o_lo, self.o_hi + 1, dtype=np.int64)
        uu, mm = np.asarray(u, np.int64), np.asarray(m, np.int64)
        j_lo = np.maximum(0, -o)
        j_hi = np.minimum(self.S, self.R - o)
        live = j_hi > j_lo
        n_ov = np.where(live, j_hi - j_lo, 0)
        U = np.concatenate([[0], np.cumsum(uu)])
        M = np.concatenate([[0], np.cumsum(mm)])
        uo = np.where(live, U[np.clip(j_hi, 0, self.S)] - U[np.clip(j_lo, 0, self.S)], 0)
        mw = np.where(live, M[np.clip(j_hi + o, 0, self.R)] - M[np.clip(j_lo + o, 0, self.R)], 0)
        c11 = _xcorr_int(uu, mm, self.o_lo, W)
        c01, c10, c00 = mw - c11, uo - c11, n_ov - mw - uo + c11
        assert (c01 >= 0).all() and (c10 >= 0).all() and (c00 >= 0).all()
        self.no_overlap = ~live
        if self.pm1:
            self.exact = c11 - c01 - c10 + c00          # int64, exact
            self.exact_f = self.exact.astype(np.float64)
        else:
            ld = np.longdouble
            hi, al = ld(self.hi), ld(self.alpha)
            self.exact = hi * c11.astype(ld) - c01.astype(ld) + hi * al * c10.astype(ld) - al * c00.astype(ld)
            self.exact_f = self.exact.astype(np.float64)
        self.max = self.exact.max()
        self.eps = _rc_eps(float(min(self.R, self.S)), self.hi, self.alpha)
        self.norm = float(np.sqrt(self.S * max(self.hi ** 2, 1.0) * self.R * max(self.alpha ** 2, 1.0)))


def _rc_eps(n, hi, alpha):
    """runcorr.cuh rc_eps, the same float64 operations in the same order."""
    u = 1.1102230246251565e-16
    c = max(abs(hi), 1.0) * max(abs(alpha), 1.0)
    k = n + 32.0
    gamma = k * u / (1.0 - k * u)
    return 2.02 * (gamma + 8.0 * u) * n * c


def _check_capture(cap, jobs, K, mos, winner_only, where):
    """cap: a run-path capture; jobs[j]: _Job.  Checks every offset, the stat, the count and the pruning."""
    for j, jb in enumerate(jobs):
        w0, n = (int(v) for v in cap["win"][j])
        mx, eps = cap["stat"][j]
        cand = int(cap["cand"][j])
        at = (where, j, jb.R, jb.S, jb.hi, jb.alpha)
        if not jb.live:
            assert n == 0 and cand == 0 and mx == -np.inf, at
            continue
        assert (w0, n) == (jb.o_lo, jb.o_hi - jb.o_lo + 1), (at, w0, n)
        f = cap["scores"][j, :n]
        if jb.pm1:
            bad = np.flatnonzero(f.astype(np.int64) != jb.exact)
            assert len(bad) == 0, (at, "offsets", (w0 + bad[:8]).tolist(), f[bad[:8]].tolist(), jb.exact[bad[:8]].tolist())
        else:
            ulp = np.maximum(np.spacing(np.abs(f)), np.spacing(np.abs(jb.exact_f).astype(np.float32))) / 2
            err = np.abs(f.astype(np.float64) - jb.exact_f)
            bad = np.flatnonzero(err > jb.eps / 2 + ulp.astype(np.float64))
            assert len(bad) == 0, (at, "offsets", (w0 + bad[:8]).tolist(), err[bad[:8]].tolist(), jb.eps)
        assert np.all(f[jb.no_overlap] == 0.0), at
        assert mx == f.max(), (at, mx, f.max())
        assert eps == np.float32(jb.eps), (at, eps, jb.eps)
        if cand == -1:
            assert winner_only, at
            continue
        if jb.pm1:
            assert cand == int(np.sum(jb.exact == jb.max)), (at, cand)
        else:
            lo = int(np.sum(jb.exact >= jb.max))
            hi = int(np.sum(jb.exact >= jb.max - 2 * np.longdouble(jb.eps)))
            assert lo <= cand <= hi, (at, lo, cand, hi)
    if winner_only:
        _check_pruning(cap, jobs, K, mos, where)


def _check_pruning(cap, jobs, K, mos, where):
    """-1 exactly where max((float)max, max) + eps < max_k (max_k - eps_k): for +-1 jobs, the ratio's exact
    maximum below the track's best; other jobs are checked where the exact maxima decide the rule."""
    for b in range(len(jobs) // K):
        js = [jobs[b * K + k] for k in range(K)]
        live = [jb for jb in js if jb.live]
        if not live:
            continue
        t_lo, t_hi = min(jb.o_lo for jb in live), max(jb.o_hi for jb in live)
        no_prune = mos is not None and max(abs(t_lo), abs(t_hi)) > mos
        # the kernel's maxima lie within eps / 2 of the exact ones: bounds of both sides of the rule
        floor_lo = max(float(x.max) - 1.5 * x.eps for x in live)
        floor_hi = max(float(x.max) - 0.5 * x.eps for x in live)
        for k, jb in enumerate(js):
            if not jb.live:
                continue
            got = int(cap["cand"][b * K + k]) == -1
            at = (where, b, k, float(jb.max), floor_lo, floor_hi)
            ulp = float(np.spacing(np.float32(abs(float(jb.max)))))
            if no_prune:
                assert not got, at
            elif all(x.pm1 for x in live):
                assert got == (jb.max < max(x.max for x in live)), at
            elif float(jb.max) + 1.5 * jb.eps + ulp < floor_lo:
                assert got, at
            elif float(jb.max) + 0.5 * jb.eps >= floor_hi:
                assert not got, at


def _check_outputs(out, jobs, K, tiled_out, tiled_cap, where):
    """Per-ratio outputs of a want_all call without capture."""
    _, _, _, all_score, all_offset = out
    for j, jb in enumerate(jobs):
        if not jb.live:
            continue
        at = (where, j, jb.R, jb.S)
        m = int(all_offset[j]) - jb.o_lo
        assert 0 <= m <= jb.o_hi - jb.o_lo, at
        if jb.pm1:
            nom = np.flatnonzero(jb.exact == jb.max)[::-1][:K_CAND]
            assert m == int(nom[0]), (at, int(all_offset[j]), jb.o_lo + int(nom[0]))   # ties: the largest offset
            assert float(all_score[j]) == float(jb.max), at
        else:
            near = np.flatnonzero(jb.exact >= jb.max - 2 * np.longdouble(jb.eps))
            assert m in set(near.tolist()), at
            tol = 1e-9 * jb.norm
            assert abs(float(all_score[j]) - jb.exact_f[m]) <= tol, (at, float(all_score[j]), jb.exact_f[m])
            top = near[::-1][:K_CAND]
            assert jb.exact_f[m] >= jb.exact_f[top].max() - tol or len(near) > K_CAND, at
    if tiled_out is None:
        return
    for j, jb in enumerate(jobs):
        if jb.live and int(tiled_cap["cand"][j]) <= K_CAND:
            assert all_score[j] == tiled_out[3][j] and all_offset[j] == tiled_out[4][j], (where, j)
    for b in range(len(jobs) // K):
        if all(int(tiled_cap["cand"][b * K + k]) <= K_CAND for k in range(K)):
            for i in range(3):
                assert out[i][b] == tiled_out[i][b], (where, "track", b)


# ------------------------------------------------------------------------------------------ calls

class _Call:
    def __init__(self, handle, pcms, tracks, ratios, label, mos, start_seconds=0.0):
        order = sorted(range(len(tracks)), key=lambda i: tracks[i]["video"])
        self.tracks = [tracks[i] for i in order]
        self.h, self.pcms, self.ratios, self.label, self.mos, self.ss = handle, pcms, list(ratios), label, mos, start_seconds
        self.K = len(ratios)
        self.pcm = np.concatenate(pcms)
        self.pcm_off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
        self.tv = np.array([t["video"] for t in self.tracks], np.int32)
        self.cs = np.concatenate([t["st"] for t in self.tracks])
        self.ce = np.concatenate([t["en"] for t in self.tracks])
        self.keep = np.concatenate([t["keep"] for t in self.tracks])
        self.cue_off = np.concatenate([[0], np.cumsum([len(t["st"]) for t in self.tracks])]).astype(np.int64)
        refs = {}
        self.jobs = []
        for t in self.tracks:
            v = t["video"]
            if v not in refs:
                refs[v] = _vad(pcms[v], label).astype(np.float32) == np.float32(1.0)
            for r in self.ratios:
                u = _raster(t, r, start_seconds) != 0
                self.jobs.append(_Job(refs[v], u, min(1.0 / r, 1.0), label, mos))
        self.refs = refs
        self.stride = max([jb.o_hi - jb.o_lo + 1 for jb in self.jobs if jb.live] + [1])

    def run(self, want_all=True, batch=False):
        n0 = self.h.launch_count
        if batch:   # b2_sync_batch: each track with its own copy of its video's PCM
            pcm = np.concatenate([self.pcms[v] for v in self.tv])
            off = np.concatenate([[0], np.cumsum([len(self.pcms[v]) for v in self.tv])]).astype(np.int64)
            out = self.h.sync_batch(pcm, off, 16000, 100, self.label, 100000, -1, -1, self.cs, self.ce, self.keep,
                                    self.cue_off, self.ratios, self.ss, self.mos, want_all=want_all)
        else:
            out = self.h.sync_tracks(self.pcm, self.pcm_off, self.tv, 16000, 100, self.label, 100000, -1, -1,
                                     self.cs, self.ce, self.keep, self.cue_off, self.ratios, self.ss, self.mos,
                                     want_all=want_all)
        return out, self.h.launch_count - n0

    def capture(self, want_all=True, batch=False):
        with self.h.capture_nominations(len(self.jobs), self.stride) as cap:
            out, n = self.run(want_all, batch)
        return cap, out, n


def _same(a, b, where):
    for x, y in zip(a, b):
        if x is None and y is None:
            continue
        assert np.array_equal(np.asarray(x), np.asarray(y)), where


def _check_call(call, where, batch=False, tiled=True, n_sub=1):
    """The whole check of one call on the run path (forced), with the tiled path as the second opinion.
    n_sub: sub-batches of the pipeline (one capture launch each)."""
    with _env(B2_ALIGN_PATH="runs"):
        cap, out_c, n_c = call.capture(True, batch)
        cap_w, out_w, _ = call.capture(False, batch)
        out, n = call.run(True, batch)
        out_nw, _ = call.run(False, batch)
    assert n_c == n + n_sub, (where, n_c, n)   # the run path plus the capture kernel
    _check_capture(cap, call.jobs, call.K, call.mos, False, where)
    assert (cap["cand"] != -1).all(), where
    _check_capture(cap_w, call.jobs, call.K, call.mos, True, where + ("winner-only",))
    _same(out, out_c, where)
    _same(out_nw[:3], out[:3], where)
    _same(out_w[:3], out[:3], where)
    tiled_out = tiled_cap = None
    if tiled:
        with _env(B2_ALIGN_PATH="tiled"):
            tiled_cap, _, _ = call.capture(True, batch)
            tiled_out, n_t = call.run(True, batch)
        assert n_t != n, (where, n_t, n)
    _check_outputs(out, call.jobs, call.K, tiled_out, tiled_cap, where)
    return cap, out


def _assert_falls_back(call, where):
    """The run path cannot take the call: forcing it gives the tiled path's launches and outputs."""
    with _env(B2_ALIGN_PATH="runs"):
        forced, n_f = call.run(True)
    with _env(B2_ALIGN_PATH="tiled"):
        tiled, n_t = call.run(True)
    assert n_f == n_t, (where, n_f, n_t)
    _same(forced, tiled, where)


# ------------------------------------------------------------------------------------------ shapes

def _s_for_width(R, w, mos, s_range):
    """A mask length S in s_range whose window against a reference of R frames has exactly w offsets."""
    for S in s_range:
        lo, hi = ao.offset_range(R, S, mos)
        if hi - lo + 1 == w:
            return S
    raise AssertionError((R, w, mos))


def _random_runs(rng, S, n_runs, max_len=40):
    """n_runs separated runs inside [0, S - 2)."""
    cuts = np.sort(rng.choice(np.arange(1, (S - 4) // 2), 2 * n_runs, replace=False)) * 2
    return [(int(a), int(min(b, a + max_len))) for a, b in zip(cuts[::2], cuts[1::2])]


WIDTH_MOS = 16384
WIDTHS = [31, 32, 33, 1023, 1024, 1025, 32767, 32768]


def _width_call(handle, label):
    """The widths around lane, warp and CTA sizes in one call (K = 1): the widest job sets 1 024 threads for
    every CTA, so most CTAs have idle threads.  Against a reference of 10 000 frames (padded length 16 384) the
    mask corner leaves the offsets -S .. 0 (S + 1 of them); 32 767 and 32 768 come from the clipped and the
    plain mask of a 40 000-frame reference.  (Widths 1 and 2 are in the edge matrix.)"""
    rng = np.random.RandomState(11 + int(10 * label))
    R_big, R_mid = 40000, 10000
    pcms = [_pcm(handle, _mask_cls(rng.rand(R_big) < 0.45, rng), 1),
            _pcm(handle, _mask_cls(rng.rand(R_mid) < 0.5, rng), 2)]
    tracks = []
    for w in WIDTHS:
        v, R, s_range = (0, R_big, range(16000, 24000)) if w >= 32767 else (1, R_mid, range(2, 2000))
        S = _s_for_width(R, w, WIDTH_MOS, s_range)
        runs = _random_runs(rng, S, min(40, max(1, S // 12)))
        if S >= 64:
            runs.append((S - 20, S - 2))
        tracks.append(_track(v, runs, S=S))
    return _Call(handle, pcms, tracks, [1.0], label, WIDTH_MOS)


@pytest.mark.parametrize("label", [0.0, 0.3])
def test_every_width_in_one_call(handle, label):
    call = _width_call(handle, label)
    widths = sorted(jb.o_hi - jb.o_lo + 1 for jb in call.jobs)
    assert widths == WIDTHS, widths
    _check_call(call, ("widths", label))


def test_width_above_one_cta_falls_back(handle):
    rng = np.random.RandomState(3)
    R = 40000
    pcms = [_pcm(handle, _mask_cls(rng.rand(R) < 0.45, rng), 5)]
    S = 20000
    call = _Call(handle, pcms, [_track(0, _random_runs(rng, S - 10, 60), S=S)], [1.0], 0.0, WIDTH_MOS + 1)
    assert call.jobs[0].o_hi - call.jobs[0].o_lo + 1 == 32770
    _assert_falls_back(call, "32770 offsets")


def _edges_call(handle, label, ratios):
    """Windows off both ends of the reference and lengths at word boundaries:
    R in {1, 31, 32, 33, 63, 64, 65} (and PCM ending in a partial window), S mod 32 in {0, 1, 31} with a run
    in the mask's last word, R << S and S << R with a mask wider than the padded length (every offset
    -S .. N - 1 - S), cues at frame 0, one-frame runs one frame apart, touching and overlapping cues, a
    track whose cues are all dropped."""
    rng = np.random.RandomState(71)
    pcms, tracks = [], []
    for i, R in enumerate([1, 31, 32, 33, 63, 64, 65]):
        tail = 37 if i % 2 else 0
        R_full = R - 1 if tail else R
        pcms.append(_pcm(handle, _mask_cls(rng.rand(R_full) < 0.5, rng), 20 + i, tail))
        for S in (32 * 9, 32 * 9 + 1, 32 * 10 - 1):
            tracks.append(_track(i, [(0, 3), (5, 6), (7, 8), (9, 10), (40, 77), (S - 30, S - 2)], S=S))
    # R << S and S << R, mask wider than the padded length
    v = len(pcms)
    pcms.append(_pcm(handle, _mask_cls(rng.rand(400) < 0.5, rng), 40, 100))
    tracks.append(_track(v, [(0, 1)] + [(a, a + 1) for a in range(2, 400, 2)] + [(450, 700), (900, 1199)]))
    tracks.append(_track(v, [(0, 2), (2, 9), (5, 20), (30, 31), (31, 60), (100, 129)], S=160))
    tracks.append(_track(v, [(3, 10), (20, 31)], S=33))
    v += 1
    pcms.append(_pcm(handle, _mask_cls(rng.rand(3000) < 0.5, rng), 41))
    tracks.append(_track(v, [(0, 5), (10, 11), (12, 13)], S=64))
    for S in (3192, 3193):                # windows of 1 and 2 offsets (mask corner, padded length 8 192)
        tracks.append(_track(v, [(0, 7), (S - 40, S - 2)], S=S))
    t = _track(v, [(10, 20), (30, 40)], S=96)
    t["keep"][:] = 0                      # every cue dropped: an empty mask of 96 frames
    tracks.append(t)
    return _Call(handle, pcms, tracks, ratios, label, 5000)


@pytest.mark.parametrize("label", LABELS)
def test_edges_levels_and_labels(handle, label):
    call = _edges_call(handle, label, LEVEL_RATIOS)
    Rs = sorted({len(r) for r in call.refs.values()})
    assert {1, 31, 32, 33, 63, 64, 65} <= set(Rs), Rs
    Ss = {jb.S % 32 for jb in call.jobs[::call.K]}
    assert {0, 1, 31} <= Ss, Ss
    wide = [jb for jb in call.jobs if jb.live and jb.o_lo == -jb.S and jb.o_hi == ao.padded_length(jb.R, jb.S) - 1 - jb.S]
    assert len(wide) >= 2
    assert {1, 2} <= {jb.o_hi - jb.o_lo + 1 for jb in call.jobs if jb.live}
    _check_call(call, ("edges", label))


def test_edges_start_seconds_wrap(handle):
    """Cues before start_seconds: the raster's slice wraps them to the end of the mask."""
    rng = np.random.RandomState(5)
    pcms = [_pcm(handle, _mask_cls(rng.rand(2000) < 0.5, rng), 50)]
    t = _track(0, [(50, 80), (120, 130), (300, 400), (900, 1000)])
    t["st"] = np.concatenate([[0.10, 0.20], t["st"]])   # frames -40 .. -35 and -30 .. -20 relative to the start
    t["en"] = np.concatenate([[0.15, 0.30], t["en"]])
    t["keep"] = np.concatenate([[1, 1], t["keep"]]).astype(np.uint8)
    call = _Call(handle, pcms, [t], BENCH, 0.0, 3000, start_seconds=0.5)
    u = call.jobs[0].u
    assert u[-40:-35].all() and u[-30:-20].all(), "no run wrapped to the end of the mask"
    _check_call(call, ("start-seconds",))


def _complement_ref(u, R, o_star, rng):
    """Reference bits m with m[j + o*] = 1 - u[j]: speech just after every run end, silence at every run start,
    so every run adds 2 to the same 4-bit counter of the thread that owns o*."""
    m = rng.rand(R) < 0.5
    m[o_star:o_star + len(u)] = ~u
    return m


@pytest.mark.parametrize("n_runs", [1, 6, 7, 8, 13, 14, 15])
def test_counter_flush_boundaries(handle, n_runs):
    """Run counts around the flushes of the 4-bit counters, each against the complement of its own mask (the
    input that fills a counter) and against random, all-speech, all-silence and alternating references."""
    rng = np.random.RandomState(100 + n_runs)
    S = 800
    runs = [(40 + 50 * i, 40 + 50 * i + 1 + (i % 3)) for i in range(n_runs)]
    u = _raster(_track(0, runs, S=S), 1.0, 0.0) != 0
    R, o_star = 3000, 1234
    refs = [_complement_ref(u, R, o_star, rng), rng.rand(R) < 0.5, np.ones(R, bool), np.zeros(R, bool),
            np.arange(R) % 2 == 0]
    pcms = [_pcm(handle, _mask_cls(m, rng, hiss=0.0), 60 + i) for i, m in enumerate(refs)]
    tracks = [_track(v, runs, S=S) for v in range(len(refs))]
    call = _Call(handle, pcms, tracks, [1.0, 25.0 / 24.0], 0.0, 2000)
    assert np.array_equal(call.refs[0], refs[0]) and np.array_equal(call.refs[4], refs[4])
    jb = call.jobs[0]
    assert jb.exact[o_star - jb.o_lo] == jb.exact.min() == -S     # the planted offset: every frame disagrees
    _check_call(call, ("flush", n_runs))


def test_largest_run_table(handle):
    """Exactly 16 384 one-frame cues one frame apart in one job (192 KB of run table); 16 385 fall back."""
    rng = np.random.RandomState(8)
    runs = [(2 * i + 1, 2 * i + 2) for i in range(16384)]
    u = _raster(_track(0, runs), 1.0, 0.0) != 0
    R = 40000
    m = rng.rand(R) < 0.5
    m[5000:5000 + len(u)] = u
    pcms = [_pcm(handle, _mask_cls(m, rng), 70)]
    call = _Call(handle, pcms, [_track(0, runs), _track(0, runs[:300], S=len(u))], [1.0, 25.0 / 24.0], 0.0, 6000)
    assert len(call.tracks[0]["st"]) == 16384 and int(u.sum()) == 16384
    _check_call(call, ("16384 runs",))
    more = [(2 * i + 1, 2 * i + 2) for i in range(16385)]
    over = _Call(handle, pcms, [_track(0, more)], [1.0], 0.0, 6000)
    _assert_falls_back(over, "16385 cues")


# ------------------------------------------------------------------------------------------ ties

def _tie_video(R, P, Lb):
    m = np.zeros(R, bool)
    m[P:P + Lb] = True
    return m


def _tie_call(handle, label=0.0):
    """+-1 jobs with a plateau of k tied maxima: a run of L frames against a speech block of Lb < L frames
    ties at the offsets [P + Lb - L, P] (k = L - Lb + 1).  Placed across a lane boundary (m = 32 t + 31 /
    32 t + 32), a warp boundary (m = 1024 t - 1 / 1024 t), and plateaus of 32 and 33."""
    rng = np.random.RandomState(12)
    mos, R, S = 6000, 30000, 700
    L = 400
    o_lo, _ = ao.offset_range(R, S, mos)
    # (k, first tied m): a lane boundary, a warp boundary, plateaus of 32 and 33 (block starts P >= L)
    specs = [(2, 32 * 100 + 31), (2, 1024 * 5 - 1), (32, 32 * 60 + 5), (33, 32 * 150 + 31), (33, 1024 * 6 - 16)]
    pcms, tracks, plan = [], [], []
    for i, (k, m_first) in enumerate(specs):
        Lb = L - k + 1
        P = o_lo + m_first + k - 1                       # plateau [P - k + 1, P] = m_first .. m_first + k - 1
        pcms.append(_pcm(handle, _mask_cls(_tie_video(R, P, Lb), rng, hiss=0.0), 80 + i))
        tracks.append(_track(i, [(0, L)], S=S))
        plan.append((k, m_first))
    return _Call(handle, pcms, tracks, [1.0, 24.0 / 25.0], label, mos), plan


def test_ties_across_lane_and_warp_boundaries(handle):
    call, plan = _tie_call(handle)
    for i, (k, m_first) in enumerate(plan):
        jb = call.jobs[i * call.K]
        assert jb.pm1
        tied = np.flatnonzero(jb.exact == jb.max)
        assert tied.tolist() == list(range(m_first, m_first + k)), (i, tied[:40].tolist())
    _check_call(call, ("ties",))


# ------------------------------------------------------------------------------------------ pruning

PRUNE_RATIOS = [1.0, 25.0 / 24.0, 23.976 / 24.0, 24.0 / 25.0]   # levels 1, 0.96, 1, 1


def test_winner_only_pruning(handle):
    """Winner-only pruning at its edges.  A track whose cues are all dropped, its mask 0.2 s long: S = 22, 22,
    21, 21 frames at the four ratios, every frame silent, so against a reference with a long silence the
    maxima are 22 (+-1), 22 (two-level, equal in exact arithmetic: within 2 eps), 21 and 21 (1 below, equal to
    each other).  Random tracks beside it, and a negative mask width (every offset beyond the mask: no_prune)."""
    rng = np.random.RandomState(21)
    R = 6000
    m = rng.rand(R) < 0.5
    m[1000:1100] = False
    pcms = [_pcm(handle, _mask_cls(m, rng), 90)]
    silent = _track(0, [])
    silent.update(st=np.array([0.1]), en=np.array([0.2]), keep=np.array([0], np.uint8))
    tracks = [silent, _track(0, _random_runs(rng, 1500, 30), S=1500), _track(0, [(20, 21)], S=40)]
    call = _Call(handle, pcms, tracks, PRUNE_RATIOS, 0.0, 2000)
    assert [jb.S for jb in call.jobs[:4]] == [22, 22, 21, 21]
    assert [float(jb.max) for jb in call.jobs[:4]] == [22.0, 22.0, 21.0, 21.0]
    assert not call.jobs[1].pm1
    _check_call(call, ("pruning",))
    # mask width -100: the window of a 200-frame mask against a 10-frame reference is offsets -155 .. -100
    corner = _Call(handle, [_pcm(handle, _mask_cls(rng.rand(10) < 0.5, rng), 91)],
                   [_track(0, [(3, 20), (30, 31), (150, 190)], S=200)], PRUNE_RATIOS, 0.0, -100)
    assert (corner.jobs[0].o_lo, corner.jobs[0].o_hi) == (-155, -100)
    _check_call(corner, ("no_prune",))


# ------------------------------------------------------------------------------------------ call modes

def test_matrix_sub_batches_and_sync_batch(handle):
    """The edge matrix once more through the sub-batch pipeline and through b2_sync_batch."""
    call = _edges_call(handle, 0.3, BENCH)
    with _env(B2_SUBBATCHES=3, B2_VAD_SMS=60):
        _, out = _check_call(call, ("edges", "sub-batches"), tiled=False, n_sub=3)
    _, out_b = _check_call(call, ("edges", "sync_batch"), batch=True, tiled=False)
    _same(out_b, out, "sync_batch vs sync_tracks")
    call0 = _edges_call(handle, 0.0, [1.0, 24.0 / 25.0])
    _check_call(call0, ("edges", "sync_batch", 0.0), batch=True)


def test_bench_shape_two_hours(handle):
    """One two-hour video x 5 tracks at +-60 s with the bench ratios, captured in full."""
    dur = 7200.0
    st, en = cases.synthetic_cues(4242, dur)
    mask = ro.rasterize(st, en, None, 100, 0, 1.0)[0] != 0
    n = int(dur * 100)
    rng = np.random.RandomState(4243)
    m = np.zeros(n, bool)
    m[: min(n, len(mask))] = mask[:n]
    m ^= rng.rand(n) < 0.10
    pcms = [_pcm(handle, _mask_cls(m, rng), 4244)]
    tracks = []
    for i, (k, delta) in enumerate([(0, 250), (2, -700), (4, 0), (1, 1234), (3, -5999)]):
        r = np.random.RandomState(100 + i)
        keep = r.rand(len(st)) >= 0.1
        s = (st - delta / 100.0) / BENCH[k]
        e = (en - delta / 100.0) / BENCH[k]
        keep &= s >= 0
        tracks.append(dict(video=0, st=np.round(s[keep], 3), en=np.round(e[keep], 3),
                           keep=np.ones(int(keep.sum()), np.uint8)))
    call = _Call(handle, pcms, tracks, BENCH, 0.0, 6000)
    assert all(jb.o_hi - jb.o_lo + 1 == 12000 for jb in call.jobs)
    _check_call(call, ("bench shape",))
