"""Exact per-window features of the VAD (K1) on every kernel variant (run on an H100).

The other VAD tests check decisions on synthetic speech / hiss / silence, whose windows sit far from every
threshold: a kernel that miscounts a window's sign changes by a few, or its energy by one, passes them.
Here every call's decisions are compared with plain int64 numpy (``oracle.vad_oracle.window_features``)
at settings that make each decision a probe of one exact feature:

* crossing sweep: energy threshold 0 and band ``[v, v]`` for every crossing count v the input has (and
  fpw - 1, fpw): a window reads 1.0 exactly when its Z is v, which pins every full window's Z;
* energy edges: windows built with E = fpw*T + d, d in {-1, 0, +1}, band wide open: the decision is
  E >= fpw*T, which pins E at the threshold, across 2^31, 2^32 and at full scale.

Each call writes into a device output prefilled with NaN (every window must be written), label 0.5; a
partial last window must read 0.5.

Variant matrix, from the planner in b2i_vad_launch (which kernel runs is not observable from Python):

| input                                   | kernel / path                                          |
|-----------------------------------------|--------------------------------------------------------|
| 16 kHz, aligned                         | lane <20,1>; with B2_VAD_WPL=2: <20,2>                 |
| 8 kHz, aligned                          | lane <10,2>; with B2_VAD_WPL=2: <10,4>                 |
| 16 kHz, B2_VAD_LAYOUT=group             | group fast <5,4>                                       |
| 48 kHz                                  | group fast <15,4>                                      |
| 8 kHz, group layout                     | runtime CPL 5, G = 2                                   |
| 24 kHz                                  | runtime CPL 15, G = 2                                  |
| 32 kHz                                  | runtime CPL 5, G = 8                                   |
| 96 kHz                                  | runtime CPL 15, G = 8                                  |
| 25.6 kHz                                | runtime CPL 1, G = 32                                  |
| 27.2 kHz                                | runtime CPL 17, G = 2: the 16-chunk partial-sum flush  |
| 44.1, 22.05, 11.025 kHz                 | 16-bit path (window not a multiple of 8 samples)       |
| 16 or 48 kHz, a pcm_off not a multiple of 8 | 16-bit path, head_bytes 2 ... 14                   |

("aligned": every signal starts at a multiple of 8 samples, i.e. 16 bytes.)
"""
import math

import numpy as np
import pytest

from oracle import auditok_oracle as au
from oracle import vad_oracle as vo

pytestmark = pytest.mark.gpu

LABEL = 0.5
INT16_MAX = 32767

# id -> (frame_rate, signal starts "aligned" / "ragged", environment, chunks per lane of the group layout)
VARIANTS = {
    "16k-lane": (16000, "aligned", {}, 5),
    "16k-lane-wpl2": (16000, "aligned", {"B2_VAD_WPL": "2"}, 5),
    # a shallow ring and every producer batch size, 16 only legal because the batch is capped at the ring
    "16k-lane-stages4-batch1": (16000, "aligned", {"B2_VAD_STAGES": "4", "B2_VAD_BATCH": "1"}, 5),
    "16k-lane-stages4-batch4": (16000, "aligned", {"B2_VAD_STAGES": "4", "B2_VAD_BATCH": "4"}, 5),
    "16k-lane-stages4-batch16": (16000, "aligned", {"B2_VAD_STAGES": "4", "B2_VAD_BATCH": "16"}, 5),
    "8k-lane": (8000, "aligned", {}, 5),
    "8k-lane-wpl2": (8000, "aligned", {"B2_VAD_WPL": "2"}, 5),
    "16k-group": (16000, "aligned", {"B2_VAD_LAYOUT": "group"}, 5),
    "16k-group-1cta-2stages": (16000, "aligned", {"B2_VAD_LAYOUT": "group", "B2_VAD_CTAS_FORCE": "1",
                                                   "B2_VAD_STAGES": "2"}, 5),
    "8k-group": (8000, "aligned", {"B2_VAD_LAYOUT": "group"}, 5),
    "48k": (48000, "aligned", {}, 15),
    "48k-1cta-2stages": (48000, "aligned", {"B2_VAD_CTAS_FORCE": "1", "B2_VAD_STAGES": "2"}, 15),
    "24k": (24000, "aligned", {}, 15),
    "32k": (32000, "aligned", {}, 5),
    "96k": (96000, "aligned", {}, 15),
    "25.6k": (25600, "aligned", {}, 1),
    "27.2k": (27200, "aligned", {}, 17),
    "44.1k": (44100, "ragged", {}, 1),
    "44.1k-1cta-2stages": (44100, "ragged", {"B2_VAD_CTAS_FORCE": "1", "B2_VAD_STAGES": "2"}, 1),
    "22.05k": (22050, "ragged", {}, 1),
    "11.025k": (11025, "ragged", {}, 1),
    "16k-unaligned": (16000, "ragged", {}, 1),
    "48k-unaligned": (48000, "ragged", {}, 1),
}
_KNOBS = ("B2_VAD_LAYOUT", "B2_VAD_WPL", "B2_VAD_STAGES", "B2_VAD_BATCH", "B2_VAD_CTAS_FORCE", "B2_VAD_WPT")


@pytest.fixture(scope="module")
def handle():
    """The library handle, enqueueing on torch's current stream (so NaN prefills and comparisons are ordered
    around its launches)."""
    import torch
    from ffsubsync_b200 import _native
    h = _native.get_handle()
    h.set_stream(torch.cuda.current_stream().cuda_stream)
    yield h
    h.set_stream(None)


def _set_knobs(monkeypatch, env):
    for k in _KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ----------------------------------------------------------------------------------------- PCM families

def _family_rows(fpw, n, cpl, rng):
    """n windows of int16 PCM (shape (n, fpw)) from families aimed at where the kernels go wrong, shuffled."""
    i = np.arange(fpw)
    edge = (3 * fpw) // 8   # the default band's upper edge

    def flip(m):
        return rng.rand(m, 1) < 0.5

    def signed(neg):   # random magnitudes below a per-window amplitude 2^0 .. 2^15, sign as given (0 is >= 0)
        amp = 2 ** rng.randint(0, 16, (len(neg), 1))
        mag = (rng.random_sample(neg.shape) * amp).astype(np.int64)
        return np.where(neg, -1 - mag, mag)

    def crossings_at(mask):   # mask[w, k]: a sign change between samples k - 1 and k of window w
        mask = np.array(mask, dtype=bool)
        mask[:, 0] = False
        return signed((np.cumsum(mask, axis=1) & 1).astype(bool) ^ flip(len(mask)))

    def exact_z(zs):   # zs[w] sign changes at random positions
        keys = rng.rand(len(zs), fpw)
        keys[:, 0] = 2.0
        return crossings_at(keys.argsort(1).argsort(1) < zs[:, None])

    def full(m):
        return rng.randint(-32768, 32768, (m, fpw))

    families = [
        full,                                                                      # full-range random
        lambda m: np.where(rng.rand(m, fpw) < 0.03, full(m), 0),                   # sparse
        lambda m: rng.randint(-2, 3, (m, fpw)),                                    # small, many zeros
        lambda m: -(rng.rand(m, fpw) < 0.5).astype(np.int64),                      # 0 against -1
        lambda m: np.tile(np.where(i % 2 == 0, -32768, INT16_MAX), (m, 1)),        # Z = fpw - 1, maximal E
        lambda m: np.array([255, 256, -256, -257])[rng.randint(0, 4, (m, fpw))],   # lo8 / hi8 split
        lambda m: signed(np.broadcast_to(flip(m), (m, fpw))),                      # crossings across windows only
        lambda m: crossings_at(np.broadcast_to(i % (8 * cpl) == 0, (m, fpw))),     # at lane-chunk starts only
        lambda m: crossings_at(np.broadcast_to(i % 8 == 0, (m, fpw))),             # at 16-byte chunk starts only
        lambda m: crossings_at((rng.rand(m, fpw) < 0.3) & (i % 2 == 1)),           # inside 32-bit words only
        lambda m: crossings_at((rng.rand(m, fpw) < 0.3) & (i % 2 == 0)),           # across 32-bit words only
    ]
    # exact counts (every k in 1..fpw-1 for the single crossing; every Z, and Z around the band edge)
    m_exact = max(fpw, min(2000, n // 20))
    rows = [crossings_at(i[None, :] == 1 + (np.arange(m_exact) % (fpw - 1))[:, None]),
            exact_z(rng.randint(0, fpw, m_exact)),
            exact_z(np.clip(edge + rng.randint(-4, 5, m_exact), 0, fpw - 1))]
    m = max(1, (n - 3 * m_exact) // len(families) + 1)
    rows = [r.astype(np.int16) for r in rows] + [f(m).astype(np.int16) for f in families]
    out = np.concatenate(rows)
    return out[rng.permutation(len(out))][:max(n, 1)]


# ------------------------------------------------------------------------------------- energy edges

def _squares(r, k):
    """k non-negative ints <= 32767 whose squares add up to r (greedy, with backtracking), or None."""
    if r < 0 or r > k * INT16_MAX ** 2:
        return None
    if k == 1:
        a = math.isqrt(r)
        return [a] if a * a == r else None
    a = min(math.isqrt(r), INT16_MAX)
    if k == 2:
        while 2 * a * a >= r:
            b = math.isqrt(r - a * a)
            if b * b == r - a * a:
                return [a, b]
            a -= 1
        return None
    for _ in range(200):
        if a < 0:
            break
        rest = _squares(r - a * a, k - 1)
        if rest is not None:
            return [a] + rest
        a -= 1
    return None


def _window_with_energy(e, n, pos, rng):
    """n int16 samples with sum of squares exactly e: all but len(pos) samples at random, the remainder a
    sum of len(pos) squares placed at the sample indices pos (lane-chunk and 32-bit word boundaries)."""
    x = np.zeros(n, np.int64)
    rem = e
    free = [j for j in range(n) if j not in set(pos)]
    u_lo = 0.5 if e <= n * 2 ** 27 else 0.97   # keep the remainder within len(pos) * 32767^2
    for idx, j in enumerate(free):
        q = int(rem // (n - idx) * rng.uniform(u_lo, 1.0))
        m = min(math.isqrt(q), INT16_MAX)
        x[j] = m if rng.rand() < 0.5 else -m
        rem -= m * m
    sq = _squares(rem, len(pos))
    assert sq is not None, (e, n, rem)
    for j, s in zip(pos, sq):
        x[j] = s if rng.rand() < 0.5 else -s
    assert int((x * x).sum()) == e
    return x.astype(np.int16)


def _thresholds(fpw):
    """Per-sample energy thresholds T (the API's energy_threshold): small, the default, around E = 2^31 and
    2^32 (the sums need 64 bits), large."""
    return [1, 2, 3, 7, 100, 12345, 100000, 2 ** 31 // fpw, -(-2 ** 31 // fpw), 2 ** 32 // fpw,
            -(-2 ** 32 // fpw), 5 * 10 ** 7, 9 * 10 ** 8]


def _edge_rows(fpw, cpl, rng):
    b = 8 * cpl if 8 * cpl < fpw else fpw // 2
    pos = sorted({0, b - 1, b, fpw - 1})
    rows = [_window_with_energy(fpw * t + d, fpw, pos, rng)
            for t in _thresholds(fpw) for d in (-1, 0, 1, -1, 0, 1)]
    rows.append(np.full(fpw, -32768, np.int16))   # E = fpw * 2^30: the largest a window can have
    rows.append(np.where(np.arange(fpw) % 2 == 0, -32768, INT16_MAX).astype(np.int16))
    rows = np.stack(rows)
    return rows[rng.permutation(len(rows))]


# -------------------------------------------------------------------------------------------- batches

class _Batch:
    """Device PCM of a batch of signals, its pcm_off and the oracle's E / Z per output window (-1 for a
    partial last window, which no threshold lets through)."""

    def __init__(self, fr, sigs):
        import torch
        self.fr = fr
        self.fpw = vo.frames_per_window(fr, 100)
        self.sigs = sigs
        self.pcm_off = np.concatenate([[0], np.cumsum([len(s) for s in sigs])]).astype(np.int64)
        e_all, z_all = [], []
        for s in sigs:
            n_full = len(s) // self.fpw
            step = 1 << 16
            for w0 in range(0, n_full, step):   # window_features over window-aligned slices: same result
                e, z = vo.window_features(s[w0 * self.fpw:min(n_full, w0 + step) * self.fpw], self.fpw)
                e_all.append(e)
                z_all.append(z)
            if len(s) % self.fpw:
                e_all.append(np.array([-1], np.int64))
                z_all.append(np.array([-1], np.int64))
        self.E_host = np.concatenate(e_all) if e_all else np.zeros(0, np.int64)
        self.Z_host = np.concatenate(z_all) if z_all else np.zeros(0, np.int64)
        self.n_out = len(self.E_host)
        assert self.n_out == sum(-(-len(s) // self.fpw) for s in sigs)
        self.pcm = torch.from_numpy(np.concatenate(sigs)).cuda()
        self.E = torch.from_numpy(self.E_host).cuda()
        self.Z = torch.from_numpy(self.Z_host).cuda()
        self.out = torch.empty(self.n_out, dtype=torch.float32, device="cuda")

    def run(self, handle, thr, z_lo, z_hi):
        from ffsubsync_b200 import _native
        self.out.fill_(float("nan"))
        handle.vad_energy_zcr(self.pcm.data_ptr(), self.pcm_off, self.fr, 100, LABEL, thr, z_lo, z_hi,
                              out=self.out.data_ptr(), memspace=_native.B2_DEVICE)
        return self.out

    def expect(self, thr, z_lo, z_hi):
        import torch
        if z_lo < 0:
            z_lo = 0
        if z_hi < 0:
            z_hi = (3 * self.fpw) // 8
        speech = (self.E >= self.fpw * thr) & (self.Z >= z_lo) & (self.Z <= z_hi)
        return torch.where(speech, 1.0, LABEL).to(torch.float32)

    def check(self, handle, thr, z_lo, z_hi, what=""):
        import torch
        got = self.run(handle, thr, z_lo, z_hi)
        want = self.expect(thr, z_lo, z_hi)
        if not torch.equal(got, want):
            bad = torch.nonzero((got != want) | torch.isnan(got)).flatten()[:8].cpu().numpy()
            g = got.cpu().numpy()
            raise AssertionError("%s T=%d band [%d, %d]: %d windows differ, e.g. %s" % (
                what, thr, z_lo, z_hi, int(((got != want) | torch.isnan(got)).sum()),
                [(int(w), int(self.E_host[w]), int(self.Z_host[w]), float(g[w])) for w in bad]))
        return got


def _signals(rows, fpw, geometry, rng, n_big):
    """Cut a batch of signals from whole windows (rows): window counts that are no multiple of a tile, partial
    last windows of several residues, an empty and a one-sample signal, a last byte that is no multiple of
    16.  'aligned': every signal starts at a multiple of 8 samples (the lane and vector paths take it);
    'ragged': starts anywhere (the 16-bit path with head_bytes 2 ... 14)."""
    if geometry == "aligned":
        assert fpw % 8 == 0
        res = [8, 8 * (fpw // 16), fpw - 8, 0]
        spec = [(1, res[0]), (0, 0), (31, res[1]), (33, res[3]), (63, res[2]), (65, res[0]), (257, res[3]),
                (1031, res[1]), (n_big, res[2]), (0, 1)]
    else:
        res = [1, 7, fpw // 2 + 3, fpw - 1, 0]
        spec = [(1, res[0]), (0, 0), (31, res[1]), (0, 1), (33, res[4]), (63, res[2]), (65, res[3]), (257, res[1]),
                (1031, res[4]), (n_big, res[3])]
    sigs, k = [], 0
    for n_full, r in spec:
        n_full = max(0, min(n_full, len(rows) - k - 1))
        s = rows[k:k + n_full].ravel()
        k += n_full
        if r:   # the partial window: random samples (every whole row stays a full window)
            s = np.concatenate([s, rng.randint(-32768, 32768, r)])
        sigs.append(np.ascontiguousarray(s, dtype=np.int16))
    return sigs


_CACHE = {}


def _family_batch(fr, geometry, cpl):
    key = ("families", fr, geometry, cpl)
    if key not in _CACHE:
        fpw = vo.frames_per_window(fr, 100)
        rng = np.random.RandomState(fr % 1009 + len(geometry))
        lane = fr in (8000, 16000) and geometry == "aligned"
        if lane:   # every pipeline of every CTA claims several producer batches: 3 x SMs x 2 pipes x 5 x 32
            n_win = 3 * _sm_count() * 2 * 5 * 32 * (160 // fpw)
        else:
            n_win = max(12_000_000 // fpw, 3000)
        rows = _family_rows(fpw, n_win + 16, cpl, rng)
        _CACHE.clear()   # one large batch at a time on the device
        _CACHE[key] = _Batch(fr, _signals(rows, fpw, geometry, rng, n_win - 1500))
    return _CACHE[key]


def _edge_batch(fr, geometry, cpl):
    fpw = vo.frames_per_window(fr, 100)
    rng = np.random.RandomState(fr % 997 + 3)
    rows = _edge_rows(fpw, cpl, rng)
    rows = np.concatenate([rows, _family_rows(fpw, 1500, cpl, rng)])
    return _Batch(fr, _signals(rows, fpw, geometry, rng, len(rows)))


# ---------------------------------------------------------------------------------------------- tests

@pytest.mark.parametrize("variant", list(VARIANTS))
def test_crossing_counts_exact(handle, monkeypatch, variant):
    fr, geometry, env, cpl = VARIANTS[variant]
    _set_knobs(monkeypatch, env)
    b = _family_batch(fr, geometry, cpl)
    fpw = b.fpw
    zs = sorted(set(b.Z_host[b.Z_host >= 0].tolist()) | {fpw - 1, fpw})
    assert len(zs) > fpw // 2   # the families reach most crossing counts
    for v in zs:   # window reads 1.0 <=> its Z is exactly v
        b.check(handle, 0, v, v, variant)
    rng = np.random.RandomState(len(zs))
    for _ in range(4):
        lo, hi = sorted(rng.choice(fpw + 1, 2, replace=False).tolist())
        b.check(handle, 0, lo, hi, variant)
    full = b.E_host[b.Z_host >= 0]
    for q in (0.3, 0.7):   # energy and band together
        b.check(handle, int(np.quantile(full, q)) // fpw, (3 * fpw) // 16, (3 * fpw) // 8, variant)
    b.check(handle, 100000, -1, -1, variant)   # default threshold and band


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_energy_edges_exact(handle, monkeypatch, variant):
    fr, geometry, env, cpl = VARIANTS[variant]
    _set_knobs(monkeypatch, env)
    b = _edge_batch(fr, geometry, cpl)
    fpw = b.fpw
    for t in _thresholds(fpw):
        # the batch holds windows at E = fpw*T - 1, fpw*T, fpw*T + 1
        assert all(np.any(b.E_host == fpw * t + d) for d in (-1, 0, 1)), t
        b.check(handle, t, 0, fpw, variant)
        b.check(handle, t, -1, -1, variant)
    for t in (2 ** 30, 2 ** 30 + 1):   # all samples -32768: E = fpw * 2^30 passes T = 2^30 only
        assert np.any(b.E_host == fpw * 2 ** 30)
        b.check(handle, t, 0, fpw, variant)
    b.check(handle, 100000, -1, -1, variant)


@pytest.mark.parametrize("env", [{"B2_VAD_STAGES": "4", "B2_VAD_BATCH": "4"},
                                 {"B2_VAD_STAGES": "4", "B2_VAD_BATCH": "16"},
                                 {"B2_VAD_WPL": "2", "B2_VAD_BATCH": "16"},
                                 {"B2_VAD_BATCH": "16"}], ids=["stages4-batch4", "stages4-batch16",
                                                               "wpl2-batch16", "batch16"])
def test_lane_producer_batch_deeper_than_the_ring(handle, monkeypatch, env):
    """B2_VAD_BATCH larger than the ring (4 stages; 5 stages per pipeline with B2_VAD_WPL=2; 10 by default) is
    capped at the ring depth: the same output as a batch that fits, on a batch where every CTA claims many."""
    _set_knobs(monkeypatch, env)
    b = _family_batch(16000, "aligned", 5)
    b.check(handle, 100000, -1, -1, str(env))
    b.check(handle, 0, 60, 60, str(env))


# ------------------------------------------------------------------------------------ auditok contract

def _auditok_flags(sig, fpw, max_length):
    """The reference detector with min_length 1, max_continuous_silence 0 and label 0 on one signal: with
    these tokenizer settings its output is the literal energy validator's per-block flags."""
    valid = [au.block_is_valid(blk) for blk in au.read_blocks(sig, fpw)]
    tokens = au.tokenize(valid, 1, max_length, 0)
    media = np.zeros(len(valid) + 1)
    for s, e in tokens:
        media[s] = 1.0
        media[e + 1] = -1.0
    out = np.clip(np.cumsum(media)[:-1], 0.0, 1.0)
    assert np.array_equal(out, np.array(valid, np.float64))
    return out


def _nearest_representable(e, k, step):
    while _squares(e, k) is None:
        e += step
    return e


def _block(e, n, rng):
    if n >= 4:
        return _window_with_energy(e, n, sorted({0, n // 2 - 1, n // 2, n - 1}), rng)
    sq = _squares(e, n)
    return np.array([s if rng.rand() < 0.5 else -s for s in sq], np.int16)


@pytest.mark.parametrize("fr, geometry", [(16000, "aligned"), (48000, "aligned"), (44100, "ragged"),
                                          (16000, "ragged")], ids=["16k-lane", "48k-group", "44.1k", "16k-unaligned"])
def test_auditok_energy_floor_exact(handle, fr, geometry):
    """b2_vad_auditok's per-block decision at the validator's exact integer floor, full blocks and trailing
    partial blocks of sampled lengths (lane kernel's and both group paths' tail_emin branch)."""
    import torch
    from ffsubsync_b200 import _native
    lib = _native.load()
    fpw = lib.b2_auditok_block_size(fr, 100)
    floor = lib.b2_auditok_energy_floor(fpw, 50.0)
    assert floor == au.energy_floor(fpw, 50)
    rng = np.random.RandomState(fr + len(geometry))
    rs = sorted({1, 2, 3, 4, 5, 7, 8, 9, fpw // 2, fpw - 8, fpw - 1} | set(rng.randint(1, fpw, 12).tolist()))
    sigs = []   # (PCM, intended per-block flags): full blocks at F - 1 and F, then a tail just below or at F_r
    for r in rs:
        f_r = lib.b2_auditok_energy_floor(r, 50.0)
        assert f_r == au.energy_floor(r, 50)
        below = _nearest_representable(f_r - 1, r, -1) if r < 4 else f_r - 1
        above = _nearest_representable(f_r, r, 1) if r < 4 else f_r
        for e, on in ((below, 0.0), (above, 1.0)):
            order = [0, 1] if rng.rand() < 0.5 else [1, 0]
            sigs.append((np.concatenate([_block(floor - 1 + k, fpw, rng) for k in order] + [_block(e, r, rng)]),
                         order + [on]))
    # one call per batch of signals; on aligned input only the last signal of a call may end off a 16-byte
    # boundary (it shifts every later start)
    if geometry == "aligned":
        calls = [[s for s in sigs if len(s[0]) % 8 == 0]] + [[s] for s in sigs if len(s[0]) % 8]
    else:
        calls = [sigs]
    max_length = 10 ** 6
    for call in calls:
        pcm_off = np.concatenate([[0], np.cumsum([len(s) for s, _ in call])]).astype(np.int64)
        want = np.concatenate([_auditok_flags(s, fpw, max_length) for s, _ in call])
        # the validator itself puts the blocks where they were built: the edges are pinned
        assert np.array_equal(want, np.concatenate([flags for _, flags in call]))
        pcm = torch.from_numpy(np.concatenate([s for s, _ in call])).cuda()
        out = torch.full((len(want),), float("nan"), dtype=torch.float64, device="cuda")
        handle.vad_auditok(pcm.data_ptr(), pcm_off, fr, 100, 0.0, min_length=1, max_length=max_length,
                           max_continuous_silence=0, out=out.data_ptr(), memspace=_native.B2_DEVICE)
        got = out.cpu().numpy()
        assert np.array_equal(got, want), (fr, geometry, np.nonzero(got != want)[0][:8], len(call))


# ------------------------------------------------------------------------------------------- streaming

@pytest.mark.parametrize("fr", [16000, 48000])
def test_stream_ragged_chunks_crossing_sweep(handle, fr):
    """b2_vad_stream_*: chunks of odd byte counts, of fewer than 16 bytes and of sample counts that are no
    multiple of 8, each detected like one detector call; crossing sweep around the default band edge."""
    fpw = vo.frames_per_window(fr, 100)
    edge = (3 * fpw) // 8
    rng = np.random.RandomState(fr // 1000)
    sizes = [2 * fpw * 700 + 1, 7, 15, 2 * fpw * 40 + 6, 1, 2 * (8 * 90 + 3), 2 * fpw * 333 - 2, 14,
             2 * fpw * 1200 + 3, 2 * fpw, 9, 2 * fpw * 64]
    chunks = []
    for n in sizes:   # every chunk starts at a window of its own, so windows with Z near the edge stay whole
        rows = _family_rows(fpw, n // (2 * fpw) + 1, 5, rng)
        chunks.append(rows.ravel().tobytes()[:n])
    settings = [(0, v, v) for v in range(edge - 3, edge + 4)] + [(100000, -1, -1)]
    n_hits = 0
    for thr, z_lo, z_hi in settings:
        want = np.concatenate([vo.energy_zcr_detect(c[:len(c) // 2 * 2], 100, fr, LABEL, thr,
                                                    None if z_lo < 0 else z_lo, None if z_hi < 0 else z_hi)
                               for c in chunks if len(c) >= 2])
        handle.vad_stream_begin(fr, 100, LABEL, thr, z_lo, z_hi)
        for c in chunks:
            handle.vad_stream_push(c)
        got = handle.vad_stream_end()
        assert np.array_equal(got.astype(np.float64), want), (fr, thr, z_lo, np.nonzero(got != want)[0][:8])
        n_hits += int((want == 1.0).sum()) if thr == 0 else 0
    assert n_hits > 100   # the sweep met windows at every tested count
