"""The aligner's nomination stage against a float64 correlation at EVERY offset of the window.

The aligner scores all surviving offsets in fp32 (overlap-save tiles, corr.cu, or one large four-step
FFT per signal, bigfft.cu), takes the fp32 maximum and the round-off bound tau, and re-scores every
offset within tau of the maximum exactly (DESIGN.md section 4, "Round-off bound").  That argument
needs |fp32 score - exact score| <= tau at every offset; the final (score, offset) alone hides any
fp32 error smaller than the winner's margin.  b2_capture_nominations exposes the fp32 window,
(maximum, tau) and the candidate count of every (pair, ratio), and these tests check them against
oracle/aligner_oracle.correlation (complex128) on the signals the kernels were given:
  * the surviving window equals the oracle's;
  * the captured maximum is the maximum of the captured scores;
  * max |fp32 - exact| <= tau (tau is the kernels' own bound, never loosened here);
  * the candidate count is #{fp32 >= max - tau} (cut in float32), B2_ALIGN_CAND_OVERFLOW iff > 32;
  * the returned offset is the exact argmax over the 32 largest-offset candidates, the score exact;
  * winner-only b2_sync_batch: B2_ALIGN_APPROX exactly for the ratios whose max + tau lies below
    another ratio's max - tau.
Shapes: every block length L / 2048 = 8 .. 16, 1 to 7 overlap-save tiles, split block ranges,
every large-FFT size 2^17 .. 2^23, several groups on the large-window path, plateaus of exactly 32 and
33 tied candidates across selection chunk boundaries."""
import numpy as np
import pytest

import cases
from oracle import aligner_oracle as ao
from oracle import raster_oracle as ro
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

K_CAND = 32
WORST = {}   # (path, subtitle encoding) -> worst max |fp32 - exact| / tau


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for key in sorted(WORST):
        print("nomination error / tau, worst [%s, %s]: %.3g" % (key + WORST[key][:1]), *WORST[key][1:])


# ------------------------------------------------------------------------------------------ oracle

class _Exact:
    """float64 correlation of a (ref, sub) pair, computed once per pair of signals."""

    def __init__(self):
        self.memo = {}

    def window(self, ref, sub, w0, n):
        key = (id(ref), id(sub))
        if key not in self.memo:
            conv = ao.correlation(ref, sub)
            if _binary(ref) and _binary(sub):
                conv = np.round(conv)          # +-1 products: the exact scores are integers
            self.memo[key] = (conv, ref, sub)  # keep the arrays alive: their ids are the key
        conv = self.memo[key][0]
        N, S = len(conv), len(sub)
        o = w0 + np.arange(n)
        # aligners.py:47; offsets where the signals do not overlap score exactly 0 (no FFT round-off)
        return np.where((o > -S) & (o < len(ref)), conv[N - 1 - S - o], 0.0)


def _binary(x):
    return bool(np.all((x == 0) | (x == 1)))


def _norm(x):
    return float(np.sqrt(np.sum((2.0 * np.asarray(x, np.float64) - 1.0) ** 2)))


def _check_jobs(cap, sigs, mos, exact, key, out=None, winner_only=False, K=1):
    """sigs[j] = (ref, sub) float64 arrays of global job j as the kernels saw them; out = (score, offset,
    status) per job (None in winner-only calls).  Returns the per-job fp32 maxima / taus."""
    stats = []
    for j, (ref, sub) in enumerate(sigs):
        w0, n = (int(v) for v in cap["win"][j])
        mx, tau = (np.float32(v) for v in cap["stat"][j])
        cand = int(cap["cand"][j])
        o_lo, o_hi = ao.offset_range(len(ref), len(sub), mos)
        where = (key, j, len(ref), len(sub), mos)
        if o_lo > o_hi:
            assert n == 0 and cand == 0 and mx == -np.inf, where
            stats.append((mx, tau, None))
            continue
        assert (w0, n) == (o_lo, o_hi - o_lo + 1), where
        f = cap["scores"][j, :n]
        assert mx == f.max(), where
        ex = exact.window(ref, sub, w0, n)
        err = float(np.abs(f.astype(np.float64) - ex).max())
        assert err <= float(tau), (where, err, float(tau))
        WORST[key] = max(WORST.get(key, (0.0,)), (err / float(tau), "N=%d" % ao.padded_length(len(ref), len(sub)),
                                                   "R=%d S=%d" % (len(ref), len(sub)), "mos=%s" % mos))
        cut = np.float32(mx - tau)           # float32 subtraction, as the selection kernels do
        hits = np.flatnonzero(f >= cut)
        if cand != -1:
            assert cand == len(hits), (where, cand, len(hits))
        if out is not None:
            score, offset, status = (None if a is None else a[j] for a in out)
            assert cand != -1, where
            if status is not None:           # b2_sync_batch does not return the per-ratio status
                assert bool(status & 4) == (cand > K_CAND), (where, status, cand)
            top = hits[::-1][:K_CAND]        # largest offsets first
            best = ex[top].max()
            m = int(offset) - w0
            assert m in set(top.tolist()), (where, int(offset))
            tol = 1e-9 * (_norm(ref) * _norm(sub) + 1.0)
            assert ex[m] >= best - tol and abs(float(score) - ex[m]) <= tol, (where, float(score), ex[m], best)
            if _binary(ref) and _binary(sub):   # integer scores: the tie rule is checkable exactly
                assert m == int(top[np.flatnonzero(ex[top] == best)[0]]), where
        stats.append((mx, tau, (w0, n, f)))
    if winner_only:
        _check_approx(cap, stats, mos, K, key)
    return stats


def _check_approx(cap, stats, mos, K, key):
    """Winner-only pruning: cand == -1 exactly when max + tau < max_k (max_k - tau_k) and no surviving
    offset of the pair exceeds the mask width (no_prune)."""
    for b in range(len(stats) // K):
        js = range(b * K, b * K + K)
        floor = max(np.float32(stats[j][0] - stats[j][1]) for j in js)
        no_prune = mos is not None and any(
            stats[j][2] is not None and max(abs(stats[j][2][0]), abs(stats[j][2][0] + stats[j][2][1] - 1)) > mos
            for j in js)
        for j in js:
            mx, tau, w = stats[j]
            if w is None:
                continue
            want = (not no_prune) and np.float32(mx + tau) < floor
            assert (int(cap["cand"][j]) == -1) == want, (key, b, j, float(mx), float(tau), float(floor))


# ------------------------------------------------------------------------------- b2_align_batch

def _width(R, S, mos):
    o_lo, o_hi = ao.offset_range(R, S, mos)
    return max(1, o_hi - o_lo + 1)


def _align(handle, pairs, K, mos):
    """pairs: list of (ref, [sub_0 .. sub_{K-1}]) float32.  Returns capture, outputs, job signals."""
    refs = [p[0] for p in pairs]
    subs = [s for p in pairs for s in p[1]]
    ref_off = np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.int64)
    sub_off = np.concatenate([[0], np.cumsum([len(s) for s in subs])]).astype(np.int64)
    stride = max(_width(len(pairs[j // K][0]), len(s), mos) for j, s in enumerate(subs))
    with handle.capture_nominations(len(subs), stride) as cap:
        out = handle.align_batch(np.concatenate(refs), ref_off, np.concatenate(subs), sub_off, len(pairs), K, mos)
    sigs = [(pairs[j // K][0].astype(np.float64), s.astype(np.float64)) for j, s in enumerate(subs)]
    return cap, out, sigs


def _tiled_q_mos(q):
    """Mask width whose +-window makes the planner pick L = q * 2048 + 1024 (q < 16): offsets per tile
    Wt = 32 ceil((2 mos - 1) / 32) + 1 = 31 745 - 2048 q, L = 2^15 - Wt + 1."""
    return 15872 - 1024 * q


_LEVEL_MIX = [  # (reference family, subtitle family, subtitle level)
    ("random", "random", 1.0), ("random", "random", 0.96), ("wide", "wide", 1.0), ("ones", "random", 1.0),
    ("sparse", "sparse", 0.96), ("random", "ones", 1.0), ("period_block", "random", 0.96), ("sparse", "random", 1.0),
]


def _make_pair(rng, fam_r, R, sub_specs):
    """Reference of family fam_r and one subtitle signal per (family, S, level, shift) in sub_specs.  Each
    subtitle carries a copy of the reference (delayed by shift) on half of its frames, so that the window
    holds a real peak next to the family's own landscape ("wide" subtitles stay pure noise)."""
    ref = cases.signal_family(fam_r, R, rng)
    subs = []
    for fam_s, S, level, shift in sub_specs:
        sub = cases.signal_family(fam_s, S, rng, level)
        src = np.arange(S) - shift
        ok = (src >= 0) & (src < R) & (np.arange(S) % 2 == 0)
        if fam_s != "wide":
            sub[ok] = (ref[src[ok]] != 0) * np.float32(level)
        subs.append(sub)
    return ref, subs


def _mixed_pairs(rng, dims, salt, shift_max):
    """dims: [(R, [S_0, ..])]; signal families and levels rotate through _LEVEL_MIX."""
    pairs = []
    for b, (R, S_list) in enumerate(dims):
        specs = [_LEVEL_MIX[(salt + 3 * b + k) % len(_LEVEL_MIX)][1:] + (S, int(rng.randint(-shift_max, shift_max + 1)))
                 for k, S in enumerate(S_list)]
        pairs.append(_make_pair(rng, _LEVEL_MIX[(salt + 3 * b) % len(_LEVEL_MIX)][0], R,
                                [(f, S, lv, sh) for f, lv, S, sh in specs]))
    return pairs


def _assert_tile_width(cap, K, L):
    """The planner's offsets per tile, from the widest pair window (union over the pair's ratios)."""
    max_w = 1
    for b in range(len(cap["cand"]) // K):
        w = [(int(a), int(a) + int(n) - 1) for a, n in cap["win"][b * K:(b + 1) * K] if n > 0]
        if w:
            max_w = max(max_w, max(h for _, h in w) - min(lo for lo, _ in w) + 1)
    assert 32 * ((max_w + 30) // 32) + 1 == 32768 - L + 1, (max_w, L)


@pytest.mark.parametrize("q", list(range(8, 16)))
def test_tiled_float_every_block_length(handle, q):
    """b2_align_batch with the planner's block length L = q * 2048 + 1024 for q = 8 .. 15: K = 4 subtitle
    lengths around block multiples per pair, references much longer / much shorter than the subtitles
    (blocks pruned at both ends, windows reaching offsets without overlap) and mixed signal levels."""
    L = q * 2048 + 1024
    mos = _tiled_q_mos(q)
    rng = np.random.RandomState(100 + q)
    S_list = [2 * L - 1, 2 * L, 2 * L + 1, 3 * L + 5]
    dims = [(R, S_list) for R in (5 * L + 777, min(L // 2, mos // 2) + 3, 3 * L)]
    cap, out, sigs = _align(handle, _mixed_pairs(rng, dims, q, mos // 2), 4, mos)
    _assert_tile_width(cap, 4, L)
    _check_jobs(cap, sigs, mos, _Exact(), ("tiled", "float"), out=out)


def test_tiled_float_single_offset_window(handle):
    """L / 2048 = 16 (L = 2^15, one offset per tile) needs a one-offset window: the negative-slice corner
    mos = N - S with N >= 2 S + 1 leaves only offset -S (no overlap, score 0).  Only the subtitle's partial
    last block meets the reference there, so the planner, not a full-block first pass, is what runs."""
    L = 32768
    rng = np.random.RandomState(16)
    for S in (2 * L - 1, 2 * L, 2 * L + 1, 3 * L + 5):
        R = S + 5000
        N = ao.padded_length(R, S)
        assert N >= 2 * S + 1
        ref = cases.signal_family("random", R, rng)
        sub = cases.signal_family("random", S, rng, 0.96)
        cap, out, sigs = _align(handle, [(ref, [sub])], 1, N - S)
        assert int(cap["win"][0][1]) == 1
        _check_jobs(cap, sigs, N - S, _Exact(), ("tiled", "float"), out=out)


@pytest.mark.parametrize("mos, env", [
    (10000, {}), (20000, {}), (32000, {}),                                         # 2, 3, 4 tiles (default path)
    (50000, {"B2_ALIGN_PATH": "tiled"}),                                           # 7 tiles
    (5000, {"B2_ALIGN_SPLIT": "1"}), (5000, {"B2_ALIGN_SPLIT": "2"}), (5000, {"B2_ALIGN_SPLIT": "7"}),
    (5000, {"B2_ALIGN_SPLIT": "64"}),                                              # more chunks than blocks
    (20000, {"B2_ALIGN_SPLIT": "1"}), (20000, {"B2_ALIGN_SPLIT": "2"}), (20000, {"B2_ALIGN_SPLIT": "7"}),
    (20000, {"B2_ALIGN_SPLIT": "64"}),
], ids=lambda v: str(v) if not isinstance(v, dict) else "-".join("%s=%s" % kv for kv in v.items()) or "default")
def test_tiled_float_tiles_and_splits(handle, monkeypatch, mos, env):
    """Multi-tile windows and split block ranges (partial score arrays merged by window_max_kernel at
    (split * n_tiles + tile) * Wt)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.RandomState(mos)
    pairs = _mixed_pairs(rng, [(150000, [120000, 97000]), (60000, [130000, 125001])], mos // 1000, mos - 1)
    cap, out, sigs = _align(handle, pairs, 2, mos)
    _check_jobs(cap, sigs, mos, _Exact(), ("tiled", "float"), out=out)


# ------------------------------------------------------------------ large-window path, float signals

def test_large_window_float_every_transform_size(handle):
    """Unmasked: transform sizes 2^17 .. 2^22 in one batch (one group per size), including a pair whose
    two ratios have different padded lengths (2^17 and 2^18)."""
    rng = np.random.RandomState(1717)
    pairs = [(70000, [60000, 62000])]
    for lg in range(17, 23):
        n = 1 << lg
        pairs.append((int(0.42 * n), [int(0.33 * n), int(0.21 * n) + 7]))
    cap, out, sigs = _align(handle, _mixed_pairs(rng, pairs, 1, 20000), 2, None)
    sizes = [ao.padded_length(len(r), len(s)) for r, s in sigs]
    assert sizes[:2] == [1 << 17, 1 << 18] and set(sizes) == {1 << lg for lg in range(17, 23)}
    _check_jobs(cap, sigs, None, _Exact(), ("large-window", "float"), out=out)


def test_large_window_float_largest_transform(handle):
    """N = 2^23 (the largest four-step factorisation), one pair."""
    rng = np.random.RandomState(23)
    ref = (rng.rand(3000000) > 0.5).astype(np.float32)
    sub = np.concatenate([np.zeros(4321, np.float32), ref])[:2500001]
    cap, out, sigs = _align(handle, [(ref, [sub])], 1, None)
    assert ao.padded_length(len(ref), len(sub)) == 1 << 23
    _check_jobs(cap, sigs, None, _Exact(), ("large-window", "float"), out=out)
    assert int(out[1][0]) == -4321


@pytest.mark.parametrize("mos, env", [(100000, {}), (None, {"B2_BIG_WS_MB": "64"})],
                         ids=["clipped-mask", "several-groups"])
def test_large_window_float_masks_and_groups(handle, monkeypatch, mos, env):
    """A mask that clips the window inside N, and a 64 MB workspace budget that splits four pairs of
    the same transform size (2^20) into two groups (group-local score_off, score workspace reused)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.RandomState(2020)
    dims = [(200000, [180000, 150000])] if mos is not None else [(600000, [400000, 380000])] * 4
    cap, out, sigs = _align(handle, _mixed_pairs(rng, dims, 2, 50000), 2, mos)
    _check_jobs(cap, sigs, mos, _Exact(), ("large-window", "float"), out=out)


# ------------------------------------------------------------------------------ selection edges

def _plateau_ref(R, centre, width):
    """Reference that is speech only on `width` frames around `centre`: against a one-frame subtitle
    signal (score(o) = r'[o]) exactly `width` offsets tie at the maximum +1, all others score 0 or -1."""
    ref = np.zeros(R, np.float32)
    ref[centre - width // 2: centre - width // 2 + width] = 1.0
    return ref


@pytest.mark.parametrize("path", ["tiled", "tiled-chunk", "large-window"])
def test_selection_plateaus_of_32_and_33(handle, path):
    """Plateaus of exactly 32 (fits the re-score budget) and 33 (B2_ALIGN_CAND_OVERFLOW) tied candidates
    across the boundaries of the selection's walk: on the tiled path a 256-offset step of the ordered
    compaction ("tiled") and the boundary m = 4 096 of the 4 096-offset counting chunks ("tiled-chunk"),
    on the large-window path the chunk boundary m = 32 768."""
    sub = np.ones(1, np.float32)
    if path.startswith("tiled"):
        mos, R = 6000, 70000
        o_lo, o_hi = ao.offset_range(R, 1, mos)
        if path == "tiled":
            centre = o_hi - 256 * 10 + 1     # offsets o_hi - 256 k and o_hi - 256 k + 1 are in different steps
        else:
            centre = o_lo + 4096             # m = offset - o_lo (the window's first offset is m = 0)
    else:
        mos, R = None, 70000
        centre = 32768 - 1 + 1               # m = offset + 1: the chunk boundary m = 32 768 is offset 32 767
    pairs = [(_plateau_ref(R, centre, w), [sub]) for w in (32, 33)]
    cap, out, sigs = _align(handle, pairs, 1, mos)
    _check_jobs(cap, sigs, mos, _Exact(), ("tiled" if path.startswith("tiled") else path, "float"), out=out)
    assert list(cap["cand"]) == [32, 33]
    assert [int(s) & 4 for s in out[2]] == [0, 4]
    for b, w in enumerate((32, 33)):
        top = centre - w // 2 + w - 1        # largest offset of the plateau: the reference's tie rule
        assert int(out[1][b]) == top and out[0][b] == 1.0


# ----------------------------------------------------------------- b2_sync_batch (bit-mask signals)

def _sync_inputs(seeds_durs, ratios, delta_max):
    """Synthetic PCM + cue lists: the reference mask is the subtitle mask at one of the ratios, delayed,
    with 10 % of its frames flipped."""
    fpw = 160
    cls_all, pcm_off, cs, ce, cue_off = [], [0], [], [], [0]
    rng = np.random.RandomState(seeds_durs[0][0])
    for seed, dur in seeds_durs:
        st, en = cases.synthetic_cues(seed, dur)
        mask = ro.rasterize(st, en, None, 100, 0, ratios[seed % len(ratios)])[0] != 0
        n = int(dur * 100)
        delta = int(rng.randint(-delta_max, delta_max + 1))
        ref = np.zeros(n, dtype=bool)
        src = np.arange(n) - delta
        ok = (src >= 0) & (src < len(mask))
        ref[ok] = mask[src[ok]]
        ref ^= rng.rand(n) < 0.10
        cls_all.append(np.where(ref, 1, np.where(rng.rand(n) < 0.05, 2, 0)).astype(np.uint8))
        pcm_off.append(pcm_off[-1] + n * fpw)
        cs.append(st)
        ce.append(en)
        cue_off.append(cue_off[-1] + len(st))
    pcm = vo.synth_pcm(np.concatenate(cls_all), fpw, seed=seeds_durs[0][0])
    refs = [vo.energy_zcr_detect(pcm[pcm_off[b]:pcm_off[b + 1]], 100, 16000, 0.0) for b in range(len(seeds_durs))]
    subs = []
    for b in range(len(seeds_durs)):
        for r in ratios:
            x = ro.rasterize(cs[b], ce[b], None, 100, 0, r)[0]
            subs.append((x != 0) * float(np.float32(min(1.0 / r, 1.0))))   # the level the kernels use
    sigs = [(refs[j // len(ratios)], subs[j]) for j in range(len(subs))]
    return (pcm, pcm_off, np.concatenate(cs), np.concatenate(ce), cue_off), sigs


def _sync(handle, inp, ratios, mos, want_all, stride):
    pcm, pcm_off, cs, ce, cue_off = inp
    J = (len(pcm_off) - 1) * len(ratios)
    with handle.capture_nominations(J, stride) as cap:
        res = handle.sync_batch(pcm, pcm_off, 16000, 100, 0.0, 100000, -1, -1, cs, ce, None, cue_off, ratios, 0.0,
                                mos, want_all=want_all)
    return cap, res


def _sync_all_modes(handle, monkeypatch, inp, sigs, ratios, mos, path, extra_envs=()):
    """want_all, winner-only, the float-signal (B2_FUSED_RASTER=0) path and extra settings on the same
    inputs: every capture checked against the oracle, the final outputs identical."""
    K = len(ratios)
    exact = _Exact()
    stride = max(_width(len(r), len(s), mos) for r, s in sigs)
    cap, res = _sync(handle, inp, ratios, mos, True, stride)
    _check_jobs(cap, sigs, mos, exact, (path, "bits"), out=(res[3], res[4], None), K=K)
    cap_w, res_w = _sync(handle, inp, ratios, mos, False, stride)
    _check_jobs(cap_w, sigs, mos, exact, (path, "bits"), winner_only=True, K=K)
    for a, b in zip(res_w[:3], res[:3]):
        assert np.array_equal(a, b), path
    for env in ({"B2_FUSED_RASTER": "0"},) + tuple(extra_envs):
        with monkeypatch.context() as mp:
            for k, v in env.items():
                mp.setenv(k, v)
            cap_e, res_e = _sync(handle, inp, ratios, mos, True, stride)
        _check_jobs(cap_e, sigs, mos, exact, (path, "float" if env.get("B2_FUSED_RASTER") == "0" else "bits"), K=K)
        for a, b in zip(res_e, res):
            assert np.array_equal(a, b), (path, env)
    return cap


@pytest.mark.parametrize("q", list(range(8, 16)))
def test_sync_batch_bits_every_block_length(handle, monkeypatch, q):
    """The bit-mask first pass is instantiated per L / 2048; subtitles longer than 2 L take it on full
    blocks.  Ratios 1 (binary level) and 24/25, 25/24 (level 0.96 for the latter)."""
    L = q * 2048 + 1024
    mos = _tiled_q_mos(q)
    ratios = [1.0, 25.0 / 24.0, 24.0 / 25.0]
    dur = 3.0 * L / 100.0
    inp, sigs = _sync_inputs([(300 + 3 * q + i, dur + 40.0 * i) for i in range(3)], ratios, mos // 2)
    assert all(len(s) > 2 * L for _, s in sigs)
    extra = ({"B2_SUBBATCHES": "3"},) if q in (8, 13) else ()
    cap = _sync_all_modes(handle, monkeypatch, inp, sigs, ratios, mos, "tiled", extra)
    _assert_tile_width(cap, len(ratios), L)


def test_sync_batch_bits_single_offset_window(handle, monkeypatch):
    """L = 2^15 on the bit-mask path (one-offset window, the negative-slice corner)."""
    inp, sigs = _sync_inputs([(416, 700.0)], [1.0], 0)
    R, S = len(sigs[0][0]), len(sigs[0][1])
    assert S > 2 * 32768 and ao.padded_length(R, S) >= 2 * S + 1
    cap = _sync_all_modes(handle, monkeypatch, inp, sigs, [1.0], ao.padded_length(R, S) - S, "tiled")
    _assert_tile_width(cap, 1, 32768)


def test_sync_batch_bits_large_window(handle, monkeypatch):
    """Unmasked b2_sync_batch: bit-mask subtitle signals through the four-step FFT at 2^17 and 2^19 (one
    group per size), winner-only and per-ratio runs, and a 64 MB workspace budget."""
    ratios = [1.0, 25.0 / 24.0]
    inp, sigs = _sync_inputs([(517, 560.0), (519, 2300.0), (518, 655.0)], ratios, 3000)
    sizes = sorted({ao.padded_length(len(r), len(s)) for r, s in sigs})
    assert sizes[0] == 1 << 17 and (1 << 19) in sizes, sizes
    _sync_all_modes(handle, monkeypatch, inp, sigs, ratios, None, "large-window", ({"B2_BIG_WS_MB": "64"},))


# ----------------------------------------------------------------------- the capture itself

def test_capture_changes_no_output_and_adds_one_launch(handle):
    """With the capture set, outputs are bit-identical and the tiled path issues exactly one extra launch;
    a window longer than the stride is refused."""
    from ffsubsync_b200 import _native
    ref, (sub,) = _make_pair(np.random.RandomState(5), "random", 90000, [("random", 70000, 1.0, 1234)])
    ref_off, sub_off = np.array([0, len(ref)]), np.array([0, len(sub)])
    n0 = handle.launch_count
    plain = handle.align_batch(ref, ref_off, sub, sub_off, 1, 1, 6000)
    n1 = handle.launch_count
    with handle.capture_nominations(1, 12000) as cap:
        got = handle.align_batch(ref, ref_off, sub, sub_off, 1, 1, 6000)
        n2 = handle.launch_count
    for a, b in zip(plain, got):
        assert np.array_equal(a, b)
    assert n2 - n1 == (n1 - n0) + 1
    assert int(cap["win"][0][1]) == 12000
    with pytest.raises(_native.NativeError, match="B2_ERR_BAD_ARG"):
        with handle.capture_nominations(1, 11999):
            handle.align_batch(ref, ref_off, sub, sub_off, 1, 1, 6000)
    n3 = handle.launch_count
    again = handle.align_batch(ref, ref_off, sub, sub_off, 1, 1, 6000)   # capture cleared on exit
    assert handle.launch_count - n3 == n1 - n0
    for a, b in zip(plain, again):
        assert np.array_equal(a, b)
