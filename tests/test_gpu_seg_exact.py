"""Exact per-window features of the detector on sampled-segment tables (b2_sync_tracks_seg, run on an H100).

tests/test_gpu_seg_ref.py compares whole references of synthetic speech, whose windows sit far from every threshold.
Here the segments' sample ranges are chosen freely inside the videos' PCM - ragged ends in the middle of the buffer,
starts off a multiple of 8 samples, ranges that overlap in PCM or lie inside one another, empty and sub-window ranges,
a range ending at the buffer's last sample, decoded pieces back to back - and every sample no range reads is poison
(full-scale noise that changes sign at every sample).  Each segment starts in a reference span of its own, so every
captured frame (handle.capture_reference) is one window's decision, compared with plain int64 numpy
(oracle.vad_oracle.window_features) and the float64 segment oracle at settings that make it a probe of one feature:

* crossing sweep: energy threshold 0 and band [v, v] for every crossing count v the input has (and fpw - 1, fpw), and
  the band [0, fpw] (every full window 1.0, every partial one the label): pins every full window's Z and which
  windows are full;
* energy edges: windows with E = fpw*T + d, d in {-1, 0, +1}, across 2^31, 2^32 and full scale, band wide open;
* auditok: with min_length 1, max_continuous_silence 0 a frame is its block's flag; every item's short last block
  (items cut by the chunk loop, remainders changing from item to item) holds E = floor - 1 / floor / floor + 1.

At label 0.5 a frame reads 1.0 (speech), 0.5 (non-speech or a partial last window) or 0.0 (no segment owns it); at
label 0 the reference is two-level and may go out as packed bits (compared with sig_oracle.packed_words).  Every
table runs under B2_DEVICE (the PCM tensor is followed by poison past the call's last sample) and B2_HOST, where the
staging workspace first holds a full-scale noise corpus (bytes outside the staged ranges are stale) - and once with
a silent corpus first.

Kernel of the segments' detector launch per variant (vad_layout.h; tests/test_seg_ref_cpu.py confirms each row
through the planner's CPU emulator):

| variant (test_gpu_vad_exact.VARIANTS) | kernel                   |
|---------------------------------------|--------------------------|
| 16k-lane, 16k-lane-wpl2, 16k-lane-stages4-batch{1,4,16}, 8k-lane, 8k-lane-wpl2 | lane-per-window |
| 16k-group, 16k-group-1cta-2stages, 8k-group, 48k, 48k-1cta-2stages, 24k, 32k, 96k, 25.6k, 27.2k | lane-group vector path |
| 44.1k, 44.1k-1cta-2stages, 22.05k, 11.025k, 16k-unaligned, 48k-unaligned | lane-group 16-bit path |
"""
import numpy as np
import pytest

from oracle import auditok_oracle as au
from oracle import segment_oracle as so
from oracle import sig_oracle
from oracle import vad_oracle as vo
from test_gpu_parity import _score_ok
from test_gpu_vad_exact import (VARIANTS, _block, _edge_rows, _family_rows, _nearest_representable, _set_knobs,
                                _thresholds)

pytestmark = pytest.mark.gpu

LABEL = 0.5
MOS = 200
# the kernel each variant's segment launch reaches (vad_layout.h VadKernel: 0 lane, 1 lane-group vector, 2 16-bit)
KERNEL = {v: (2 if geo == "ragged" else 0 if fr in (8000, 16000) and env.get("B2_VAD_LAYOUT") != "group" else 1)
          for v, (fr, geo, env, _) in VARIANTS.items()}
AUDITOK_TOK = dict(min_length=1, max_length=10 ** 6, max_continuous_silence=0)


# ------------------------------------------------------------------------------------------------ tables

def _poison(n, rng):
    """Full-scale noise whose sign changes at every sample."""
    mag = rng.randint(8192, 32768, n)
    sign = (np.arange(n) + rng.randint(2)) % 2
    return np.where(sign == 0, mag, -mag).clip(-32768, 32767).astype(np.int16)


class _Rows:
    """Hands out samples of whole windows (rows), cycling."""

    def __init__(self, rows):
        self.rows, self.k = rows, 0

    def take(self, n, fpw):
        m = -(-n // fpw)
        idx = (self.k + np.arange(m)) % len(self.rows)
        self.k = int((self.k + m) % len(self.rows))
        return self.rows[idx].ravel()[:n]


class _Table:
    """Videos of PCM (poison where no range reads) with a segment table.  add(lo, content or n) places a segment at
    lo of video 0; samples of its range that no earlier segment wrote come from `fill`."""

    def __init__(self, rng):
        self.rng = rng
        self.buf = [_poison(1 << 22, rng)]
        self.written = [np.zeros(1 << 22, bool)]
        self.segs = [[]]   # per video: (lo, hi, frames)

    def add(self, v, lo, n, fill, frames):
        hi = lo + n
        w = self.written[v]
        run = np.flatnonzero(~w[lo:hi]) + lo
        if len(run):   # fresh samples for every run of unwritten ones (a whole unwritten range starts a row)
            cuts = np.flatnonzero(np.diff(run) != 1) + 1
            for part in np.split(run, cuts):
                self.buf[v][part[0]:part[-1] + 1] = fill(len(part))
                w[part[0]:part[-1] + 1] = True
        self.segs[v].append((lo, hi, frames))
        return hi


def _finish(t, fr, lens, tracks=1):
    """The call's inputs from a _Table: video v's PCM is buf[v][:lens[v]]; starts spaced so every segment's frames
    land in a span of their own."""
    pcms = [t.buf[v][:lens[v]] for v in range(len(lens))]
    pcm_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    seg = dict(seg_video=[], seg_total=[], seg_off=[0], seg_start=[], seg_lo=[], seg_hi=[])
    for v in range(len(lens)):
        s = 1
        for lo, hi, frames in t.segs[v]:
            seg["seg_start"].append(s)
            seg["seg_lo"].append(lo)
            seg["seg_hi"].append(hi)
            s += -(-frames // 100) + 1
        seg["seg_video"].append(v)
        seg["seg_total"].append(s + 0.505)
        seg["seg_off"].append(len(seg["seg_start"]))
    seg = {k: np.asarray(x, dtype=np.int32 if k == "seg_video" else np.float64 if k == "seg_total" else np.int64)
           for k, x in seg.items()}
    return _inputs(np.concatenate(pcms), pcm_off, fr, seg, t.rng, tracks)


def _inputs(pcm, pcm_off, fr, seg, rng, tracks=1):
    from ffsubsync_b200.synth import synthetic_cues
    V = len(pcm_off) - 1
    cs, ce, tv, off = [], [], [], [0]
    for v in range(V):
        for k in range(tracks):
            s, e = synthetic_cues(int(rng.randint(1 << 30)), max(30.0, float(seg["seg_total"][v])))
            cs.append(s)
            ce.append(e)
            tv.append(v)
            off.append(off[-1] + len(s))
    L = [so.length(x, 100) for x in seg["seg_total"]]
    return dict(pcm=np.ascontiguousarray(pcm, dtype=np.int16), pcm_off=pcm_off, fr=fr, seg=seg,
                track_video=np.asarray(tv, np.int32), cue_start=np.concatenate(cs), cue_end=np.concatenate(ce),
                cue_off=np.asarray(off, np.int64), L=L, cap=int(sum(L)) + 64, V=V)


def _starts_cycle(aligned):
    """Offsets added to each range's start: 0 on aligned tables, every residue mod 8 on ragged ones."""
    k = [0]

    def nxt():
        k[0] += 1
        return 0 if aligned else [1, 3, 5, 7, 2, 6, 4, 0][k[0] % 8]
    return nxt


def energy_layout(fr, geometry, cpl, seed=0):
    """The energy detector's table for a variant: video 0 holds segments with gaps (bulk windows with ragged ends,
    sub-window and empty ranges, overlaps in PCM); video 1 decoded pieces back to back, the last one ending at the
    buffer's last sample (an odd sample count)."""
    from ffsubsync_b200.batch import segment_table
    fpw = vo.frames_per_window(fr, 100)
    rng = np.random.RandomState(seed + fr % 1013 + len(geometry))
    # (at least 3 fpw family rows: test_gpu_vad_exact's exact-count rows reach most crossing counts)
    rows = np.concatenate([_edge_rows(fpw, cpl, rng), _family_rows(fpw, max(1500, 3 * fpw + 200), cpl, rng)])
    src = _Rows(rows)
    aligned = geometry == "aligned"
    t = _Table(rng)
    fill = lambda n: src.take(n, fpw)   # noqa: E731
    off = _starts_cycle(aligned)
    pos = 24

    def nxt_lo(hi, gap):
        a = hi + gap
        a = -(-a // 8) * 8
        return a + off()

    R = len(rows)
    residues = [1, 2, 3, 4, 5, 6, 7, 11, fpw // 2 + 5, fpw - 1, 0, 8 + 3]
    # bulk windows (every row once), ragged ends mid-buffer: a multiple of 8 plus 1 .. 7, poison right after
    for i, k in enumerate([R // 2, R // 4, R // 8, 61, 33, 17, 9, 5, 3, 2, 1, R // 8]):
        r = residues[i % len(residues)]
        n = k * fpw + r
        hi = t.add(0, pos, n, fill, -(-n // fpw))
        pos = nxt_lo(hi, 8 + 16 * (i % 3))
    # sub-window and empty ranges, k * fpw +- 1
    for n in (0, 1, 7, 8, fpw - 1, fpw, fpw + 1, 2 * fpw - 1, 3 * fpw + 1, 5 * fpw - 1):
        hi = t.add(0, pos, n, fill, -(-n // fpw))
        pos = nxt_lo(hi, 16)
    # overlaps in PCM: B starts inside A and runs past its end, C lies inside A
    n_a = 20 * fpw + 5
    lo_a = pos
    hi_a = t.add(0, lo_a, n_a, fill, 21)
    lo_b = lo_a + 8 * 3 + off()
    n_b = hi_a + 40 - lo_b
    t.add(0, lo_b, n_b, fill, -(-n_b // fpw))
    lo_c = lo_a + 8 * 7 + off()
    n_c = hi_a - 9 - lo_c
    t.add(0, lo_c, n_c, fill, -(-n_c // fpw))
    t.add(0, lo_a, 7 * fpw + 3, fill, 8)   # a range starting where A starts, ending inside it
    len0 = -(-(hi_a + 200) // 8) * 8 + (0 if aligned else 3)
    # video 1: decoded pieces (ffmpeg -ss s -t 1) back to back, the last one short and ending the buffer
    total1 = 40.0
    last = 8 * (fr // 80) + (5 - len0 - 3 * fr) % 8   # the buffer ends 5 samples past a multiple of 8
    pieces = [fr, fr, fr, last]
    n1 = sum(pieces)
    tab1 = segment_table([0, n1], fr, totals=[total1], segment_count=4, segment_duration=1, piece_samples=[pieces])
    t.buf.append(_poison(n1, rng))
    t.written.append(np.zeros(n1, bool))
    t.segs.append([])
    t.buf[1][:] = src.take(n1, fpw)
    c = _finish(t, fr, [len0, n1])
    # video 1 keeps the helper's starts and total
    s = c["seg"]
    n0 = int(s["seg_off"][1])
    s["seg_start"] = np.concatenate([s["seg_start"][:n0], tab1["seg_start"]])
    s["seg_lo"] = np.concatenate([s["seg_lo"][:n0], tab1["seg_lo"]])
    s["seg_hi"] = np.concatenate([s["seg_hi"][:n0], tab1["seg_hi"]])
    s["seg_total"] = np.array([s["seg_total"][0], total1])
    s["seg_off"] = np.array([0, n0, n0 + len(pieces)], np.int64)
    c.update(L=[so.length(x, 100) for x in s["seg_total"]])
    c["cap"] = int(sum(c["L"])) + 64
    assert len(c["pcm"]) % 8 != 0 and c["seg"]["seg_hi"][-1] == n1   # ends at the buffer's last sample
    c["fpw"] = fpw
    return c


def auditok_layout(fr, geometry, seed=0):
    """The auditok table for a variant: segments cut by the chunk loop into items of chunk_samples (remainder r0 =
    chunk_samples mod fpw) and a last item of another remainder; full blocks at E = F - 1 / F, every item's short
    last block at E = f_r - 1 / f_r / f_r + 1 (the nearest sums of r squares for r < 4)."""
    fpw = int(fr * (1.0 / 100))   # auditok's block size
    aligned = geometry == "aligned"
    rng = np.random.RandomState(seed + fr % 997 + len(geometry))
    F = au.energy_floor(fpw, 50)
    cs = 2 * fpw + (40 if aligned else 37)
    t = _Table(rng)
    off = _starts_cycle(aligned)
    flags, k_item = [], [0]
    tail_es = {}

    def item(n):
        out, fl = [], []
        for _ in range(n // fpw):
            e = F - 1 + int(rng.randint(2))
            out.append(_block(e, fpw, rng))
            fl.append(float(e >= F))
        r = n % fpw
        if r:
            f_r = au.energy_floor(r, 50)
            if r not in tail_es:
                tail_es[r] = [(_nearest_representable(f_r - 1, r, -1) if r < 4 else f_r - 1),
                              (_nearest_representable(f_r, r, 1) if r < 4 else f_r),
                              (_nearest_representable(f_r + 1, r, 1) if r < 4 else f_r + 1)]
            e = tail_es[r][k_item[0] % 3]
            k_item[0] += 1
            out.append(_block(e, r, rng))
            fl.append(float(e >= f_r))
        return np.concatenate(out), fl

    pos = 16
    rems = [1, 2, 3, 5, 8, fpw // 2, fpw - 1, 7, cs % fpw, 4, 9, fpw // 3 + 1, 6, 2, fpw - 2]
    for i, r in enumerate(rems):
        m = i % 3   # whole chunks before the last item
        last = (i % 2) * fpw + r
        n = m * cs + last
        parts, fl = [], []
        for c0 in range(0, n, cs):
            x, f = item(min(cs, n - c0))
            parts.append(x)
            fl += f
        content = np.concatenate(parts)
        hi = t.add(0, pos, n, lambda k, x=content: x[:k], len(fl))
        flags.append(fl)
        pos = -(-(hi + 24) // 8) * 8 + off()
    c = _finish(t, fr, [-(-(pos + 64) // 8) * 8 + 5])
    c["fpw"], c["chunk"], c["flags"] = fpw, cs, flags
    return c


# ---------------------------------------------------------------------------------------------- oracle

def _segments(c, v):
    s = c["seg"]
    js = range(int(s["seg_off"][v]), int(s["seg_off"][v + 1]))
    a = int(c["pcm_off"][v])
    return [(int(s["seg_start"][j]), a + int(s["seg_lo"][j]), a + int(s["seg_hi"][j])) for j in js]


def _feature_maps(c):
    """Per video: (owned, E, Z) per reference frame, E = Z = -1 for a partial last window."""
    fpw, maps = c["fpw"], []
    for v in range(c["V"]):
        total = float(c["seg"]["seg_total"][v])
        own, es, zs = [], [], []
        for s, a, b in _segments(c, v):
            e, z = vo.window_features(c["pcm"][a:b], fpw)
            if (b - a) % fpw:
                e, z = np.append(e, -1), np.append(z, -1)
            own.append((s, np.ones(len(e))))
            es.append((s, e.astype(np.float64)))
            zs.append((s, z.astype(np.float64)))
        maps.append((so.assemble(total, 100, own) > 0, so.assemble(total, 100, es), so.assemble(total, 100, zs)))
    return maps


def _expect(maps, fpw, thr, z_lo, z_hi, label):
    z_lo = 0 if z_lo < 0 else z_lo
    z_hi = (3 * fpw) // 8 if z_hi < 0 else z_hi
    out = []
    for own, E, Z in maps:
        speech = (E >= fpw * thr) & (Z >= z_lo) & (Z <= z_hi) & (Z >= 0)
        out.append(np.where(~own, 0.0, np.where(speech, 1.0, label)).astype(np.float32))
    return out


def _oracle_refs(c, det, label, **kw):
    out = []
    for v in range(c["V"]):
        seg = _segments(c, v)
        out.append(so.segment_reference(c["pcm"], float(c["seg"]["seg_total"][v]), [x[0] for x in seg],
                                        [x[1] for x in seg], [x[2] for x in seg], 100, detector=det,
                                        frame_rate=c["fr"], non_speech_label=label, **kw).astype(np.float32))
    return out


# ------------------------------------------------------------------------------------------------ calls

@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


def _device_inputs(c):
    import torch
    if "dpcm" not in c:   # the caller's tensor: the call's samples, then poison past its last one
        tail = _poison(64, np.random.RandomState(5))
        c["dpcm"] = torch.from_numpy(np.concatenate([c["pcm"], tail])).cuda()
        T = len(c["track_video"])
        c["douts"] = [torch.zeros(T, dtype=dt, device="cuda") for dt in (torch.float64, torch.int32, torch.int32)]
        torch.cuda.synchronize()
    return c


def _call(handle, c, memspace, det="energy_zcr", label=LABEL, ratios=(1.0,), want_all=False, **kw):
    from ffsubsync_b200 import _native
    s = c["seg"]
    d = dict(detector=_native.B2_DETECTOR_AUDITOK, chunk_samples=c.get("chunk", 0), **AUDITOK_TOK) \
        if det == "auditok" else dict(detector=_native.B2_DETECTOR_ENERGY_ZCR)
    d.update(kw)
    if memspace == _native.B2_DEVICE:
        _device_inputs(c)
        pcm = c["dpcm"].data_ptr()
        d.update(best_score=c["douts"][0].data_ptr(), best_offset=c["douts"][1].data_ptr(),
                 best_k=c["douts"][2].data_ptr())
    else:
        pcm = c["pcm"]
    return handle.sync_tracks_seg(pcm, c["pcm_off"], c["track_video"], c["fr"], 100, label, s["seg_video"],
                                  s["seg_total"], s["seg_off"], s["seg_start"], s["seg_lo"], s["seg_hi"],
                                  c["cue_start"], c["cue_end"], None, c["cue_off"], list(ratios), 0.0, MOS,
                                  want_all=want_all, memspace=memspace, **d)


def _capture(handle, c, memspace, **kw):
    with handle.capture_reference(c["cap"], c["V"]) as cap:
        _call(handle, c, memspace, **kw)
    return cap


def _compare(c, cap, want, what, maps=None):
    """The capture against per-video expected frames (floats, or packed bits where the call packed them)."""
    n_packed = 0
    for v in range(c["V"]):
        a, b = int(cap["ref_off"][v]), int(cap["ref_off"][v + 1])
        assert b - a == len(want[v]) == c["L"][v], (what, v, b - a, len(want[v]))
        if cap["packed"][v] == 1:
            n_packed += 1
            got = cap["ref"][a: a + (b - a + 31) // 32].view(np.uint32)
            ok = np.array_equal(got, sig_oracle.packed_words(want[v]))
            bad = [] if ok else np.flatnonzero(np.unpackbits(
                (got ^ sig_oracle.packed_words(want[v])).view(np.uint8), bitorder="little"))[:8]
        else:
            got = cap["ref"][a:b]
            ok = np.array_equal(got, want[v])
            bad = [] if ok else np.flatnonzero(got != want[v])[:8]
        if not ok:
            info = [(int(f), float(want[v][f]), None if cap["packed"][v] == 1 else float(got[f]),
                     None if maps is None else (int(maps[v][1][f]), int(maps[v][2][f]))) for f in bad]
            raise AssertionError("%s: video %d differs at frames (frame, want, got, (E, Z)) %s" % (what, v, info))
    return n_packed


_CACHE = {}


def _energy(variant):
    fr, geo, _, cpl = VARIANTS[variant]
    key = ("energy", fr, geo, cpl)
    if key not in _CACHE:
        c = energy_layout(fr, geo, cpl)
        c["maps"] = _feature_maps(c)
        _CACHE[key] = c
    return _CACHE[key]


def _poison_staging(handle, c, silent=False):
    """A B2_HOST call over a corpus of at least the segment call's size: full-scale noise (or silence) fills the
    staging workspace, so every byte the segment call does not stage is stale."""
    from ffsubsync_b200 import _native
    n = int(c["pcm_off"][-1]) + 4096
    x = np.zeros(n, np.int16) if silent else _poison(n, np.random.RandomState(11))
    handle.sync_tracks(x, [0, n], [0], c["fr"], 100, 0.0, 100000, -1, -1, [1.0], [2.0], None, [0, 1], [1.0], 0.0,
                       MOS, memspace=_native.B2_HOST)


_MEMSPACES = ["device", "host"]


def _memspace(name):
    from ffsubsync_b200 import _native
    return _native.B2_DEVICE if name == "device" else _native.B2_HOST


# ---------------------------------------------------------------------------------------------- tests

@pytest.mark.parametrize("ms", _MEMSPACES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_crossing_counts_exact(handle, monkeypatch, variant, ms):
    _set_knobs(monkeypatch, VARIANTS[variant][2])
    c = _energy(variant)
    fpw, maps, memspace = c["fpw"], c["maps"], _memspace(ms)
    if ms == "host":
        _poison_staging(handle, c)
    # the shortcut over the feature maps is the segment oracle
    for thr, lo, hi in ((100000, -1, -1), (0, (3 * fpw) // 8, (3 * fpw) // 8)):
        assert all(np.array_equal(a, b) for a, b in zip(
            _expect(maps, fpw, thr, lo, hi, LABEL),
            _oracle_refs(c, "energy_zcr", LABEL, energy_threshold=thr, z_lo=None if lo < 0 else lo,
                         z_hi=None if hi < 0 else hi)))
    zall = np.concatenate([m[2][m[0]] for m in maps])
    zs = sorted(set(zall[zall >= 0].astype(int).tolist()) | {fpw - 1, fpw})
    assert len(zs) > fpw // 2
    for v in zs:   # a frame reads 1.0 <=> its window is full and its Z is exactly v
        _compare(c, _capture(handle, c, memspace, energy_threshold=0, z_lo=v, z_hi=v),
                 _expect(maps, fpw, 0, v, v, LABEL), "%s %s band [%d, %d]" % (variant, ms, v, v), maps)
    rng = np.random.RandomState(len(zs))
    for lo, hi in [(0, fpw)] + [tuple(sorted(rng.choice(fpw + 1, 2, replace=False).tolist())) for _ in range(3)]:
        _compare(c, _capture(handle, c, memspace, energy_threshold=0, z_lo=lo, z_hi=hi),
                 _expect(maps, fpw, 0, lo, hi, LABEL), "%s %s band [%d, %d]" % (variant, ms, lo, hi), maps)
    _compare(c, _capture(handle, c, memspace, energy_threshold=100000),
             _expect(maps, fpw, 100000, -1, -1, LABEL), "%s %s defaults" % (variant, ms), maps)


@pytest.mark.parametrize("ms", _MEMSPACES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_energy_edges_exact(handle, monkeypatch, variant, ms):
    _set_knobs(monkeypatch, VARIANTS[variant][2])
    c = _energy(variant)
    fpw, maps, memspace = c["fpw"], c["maps"], _memspace(ms)
    if ms == "host":
        _poison_staging(handle, c)
    eall = np.concatenate([m[1][m[0]] for m in maps])
    for t in _thresholds(fpw) + [2 ** 30, 2 ** 30 + 1]:
        if t < 2 ** 30:   # the table holds windows at E = fpw*T - 1, fpw*T, fpw*T + 1
            assert all(np.any(eall == fpw * t + d) for d in (-1, 0, 1)), t
        _compare(c, _capture(handle, c, memspace, energy_threshold=t, z_lo=0, z_hi=fpw),
                 _expect(maps, fpw, t, 0, fpw, LABEL), "%s %s T=%d" % (variant, ms, t), maps)
    assert np.any(eall == fpw * 2 ** 30)


@pytest.mark.parametrize("variant", ["16k-lane", "8k-lane-wpl2", "16k-group", "48k", "27.2k", "44.1k",
                                     "16k-unaligned"])
def test_packed_reference_at_label_zero(handle, monkeypatch, variant):
    """At label 0 the reference is two-level and goes out as the run path's packed bits."""
    _set_knobs(monkeypatch, VARIANTS[variant][2])
    c = _energy(variant)
    fpw, maps = c["fpw"], c["maps"]
    n_packed = 0
    for ms in _MEMSPACES:
        for thr, lo, hi in ((0, 0, fpw), (0, (3 * fpw) // 8, (3 * fpw) // 8), (100000, -1, -1), (12345, 0, fpw)):
            n_packed += _compare(c, _capture(handle, c, _memspace(ms), label=0.0, energy_threshold=thr, z_lo=lo,
                                             z_hi=hi),
                                 _expect(maps, fpw, thr, lo, hi, 0.0), "%s %s label 0 T=%d [%d, %d]" % (
                                     variant, ms, thr, lo, hi), maps)
    assert n_packed > 0


def test_stale_staging_either_order(handle):
    """B2_HOST after a noise corpus and after a silent one: the same captures as B2_DEVICE and the oracle."""
    from ffsubsync_b200 import _native
    for variant in ("16k-lane", "48k", "44.1k"):
        c = _energy(variant)
        fpw, maps = c["fpw"], c["maps"]
        settings = [(0, fpw - 1, fpw - 1), (0, 0, fpw), (0, (3 * fpw) // 8, (3 * fpw) // 8), (100000, -1, -1)]
        for silent in (False, True):
            _poison_staging(handle, c, silent=silent)
            for thr, lo, hi in settings:
                kw = dict(energy_threshold=thr, z_lo=lo, z_hi=hi)
                host = _capture(handle, c, _native.B2_HOST, **kw)
                dev = _capture(handle, c, _native.B2_DEVICE, **kw)
                assert np.array_equal(host["ref"], dev["ref"], equal_nan=True), (variant, silent, thr, lo)
                _compare(c, host, _expect(maps, fpw, thr, lo, hi, LABEL), "%s silent=%s" % (variant, silent), maps)


@pytest.mark.parametrize("ms", _MEMSPACES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_auditok_item_floors_exact(handle, monkeypatch, variant, ms):
    fr, geo, env, _ = VARIANTS[variant]
    _set_knobs(monkeypatch, env)
    key = ("auditok", fr, geo)
    if key not in _CACHE:
        _CACHE[key] = auditok_layout(fr, geo)
    c = _CACHE[key]
    from ffsubsync_b200 import _native
    lib = _native.load()
    assert lib.b2_auditok_block_size(fr, 100) == c["fpw"]
    want = _oracle_refs(c, "auditok", 0.0, chunk_samples=c["chunk"], **AUDITOK_TOK)
    # the validator puts every block where it was built: the frames are the intended flags
    flat = [f for fl in c["flags"] for f in fl]
    assert int((want[0] == 1.0).sum()) == int(sum(flat))
    starts = c["seg"]["seg_start"]
    for s, fl in zip(starts, c["flags"]):
        assert np.array_equal(want[0][100 * s: 100 * s + len(fl)], np.float32(fl)), s
    _compare(c, _capture(handle, c, _memspace(ms), det="auditok", label=0.0), want, "%s %s auditok" % (variant, ms))


# --------------------------------------------------------------------------------------- overlap ownership

def owner_corpus(fr, aligned, seed=0):
    """Segments that overlap in the reference with PCM that decides differently: A all speech (1.0), B one speech
    window then silence (1.0, then the label), so every frame names its owner.  Video 0: B cuts A in two, D runs past
    int(total * 100) + 2 and the total is shorter than the PCM; video 1: the total is longer than the PCM."""
    fpw = vo.frames_per_window(fr, 100)
    rng = np.random.RandomState(seed + fr % 991)
    speech = lambda w: vo.synth_pcm(np.ones(w, np.uint8), fpw, seed=int(rng.randint(1 << 30)))   # noqa: E731
    quiet = lambda w: vo.synth_pcm(np.r_[1, np.zeros(w - 1)].astype(np.uint8), fpw,   # noqa: E731
                                   seed=int(rng.randint(1 << 30)))
    d = 0 if aligned else 3
    parts0 = [(0, speech(1000)), (3, quiet(200)), (8, speech(200)), (9, quiet(50)), (20, speech(3000))]
    parts1 = [(0, speech(500)), (2, quiet(100)), (4, speech(60))]
    pcms, seg = [], dict(seg_video=[0, 1], seg_total=[35.5, 60.25], seg_off=[0], seg_start=[], seg_lo=[], seg_hi=[])
    for parts in (parts0, parts1):
        x, at = [_poison(16 + d, rng)], 16 + d
        for s, p in parts:
            seg["seg_start"].append(s)
            seg["seg_lo"].append(at)
            seg["seg_hi"].append(at + len(p))
            gap = _poison(-(-(len(p) + 40) // 8) * 8 - len(p) + d, rng)
            x += [p, gap]
            at += len(p) + len(gap)
        seg["seg_off"].append(len(seg["seg_start"]))
        pcms.append(np.concatenate(x))
    pcm_off = np.concatenate([[0], np.cumsum([len(p) for p in pcms])]).astype(np.int64)
    seg = {k: np.asarray(v, dtype=np.int32 if k == "seg_video" else np.float64 if k == "seg_total" else np.int64)
           for k, v in seg.items()}
    c = _inputs(np.concatenate(pcms), pcm_off, fr, seg, rng, tracks=2)
    c["fpw"] = fpw
    return c


OWNER_ROWS = ["16k-lane", "8k-group", "48k", "44.1k", "16k-unaligned"]


@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
@pytest.mark.parametrize("variant", OWNER_ROWS)
def test_overlap_ownership(handle, monkeypatch, variant, det):
    fr, geo, env, _ = VARIANTS[variant]
    _set_knobs(monkeypatch, env)
    c = owner_corpus(fr, geo == "aligned")
    kw = dict(chunk_samples=0, **AUDITOK_TOK) if det == "auditok" else dict(energy_threshold=100000)
    for label in (LABEL, 0.0):
        want = _oracle_refs(c, det, label, **kw)
        if label == LABEL:   # every frame names its owner: A 1.0, B's silence the label, no segment 0.0
            w0 = want[0]
            assert len(w0) == 3552 and np.all(w0[:301] == 1.0) and np.all(w0[301:500] == 0.5)
            assert np.all(w0[500:901] == 1.0) and np.all(w0[901:950] == 0.5) and np.all(w0[950:1000] == 1.0)
            assert np.all(w0[1000:2000] == 0.0) and np.all(w0[2000:] == 1.0)
            w1 = want[1]
            assert len(w1) == 6027 and np.all(w1[:201] == 1.0) and np.all(w1[201:300] == 0.5)
            assert np.all(w1[300:500] == 1.0) and np.all(w1[500:] == 0.0)
        for ms in _MEMSPACES:
            _compare(c, _capture(handle, c, _memspace(ms), det=det, label=label, **kw), want,
                     "%s %s %s label %g" % (variant, det, ms, label))


# ----------------------------------------------------------------------------------------------- results

@pytest.mark.parametrize("det", ["energy_zcr", "auditok"])
@pytest.mark.parametrize("variant", ["16k-lane", "48k", "44.1k"])
def test_results_equal_the_oracle_pipeline(handle, monkeypatch, variant, det):
    """best_* / all_* at label 0 against segment oracle -> raster_oracle -> exact_align -> max_score_select.  A
    returned offset must attain the exact maximum (the reference breaks exact ties by its float64 round-off, so only
    the score and tie membership are comparable; the subtitle signal at a ratio other than 1 is float32 in the call,
    so scores compare within test_gpu_parity's tolerance), and the chosen ratio must be one whose score ties the
    best."""
    from ffsubsync_b200 import _native
    from oracle import aligner_oracle as ao
    from oracle import raster_oracle as ro
    fr, geo, env, _ = VARIANTS[variant]
    _set_knobs(monkeypatch, env)
    c = owner_corpus(fr, geo == "aligned", seed=1)
    kw = dict(chunk_samples=0, **AUDITOK_TOK) if det == "auditok" else dict(energy_threshold=100000)
    refs = _oracle_refs(c, det, 0.0, **kw)
    ratios = [1.0, 25 / 24.0]
    K = len(ratios)
    bs, bo, bk, a_s, a_o = _call(handle, c, _native.B2_HOST, det=det, label=0.0, ratios=ratios, want_all=True, **kw)
    for t, v in enumerate(c["track_video"]):
        a, b = c["cue_off"][t], c["cue_off"][t + 1]
        results = []
        for k, r in enumerate(ratios):
            sub = ro.rasterize(c["cue_start"][a:b], c["cue_end"][a:b], None, 100, 0, r)[0]
            best, _ = ao.exact_align(refs[v].astype(np.float64), sub, MOS)
            got_o = int(a_o[t * K + k])
            assert _score_ok(a_s[t * K + k], best), (t, k, a_s[t * K + k], best)
            assert _score_ok(ao.exact_score(refs[v].astype(np.float64), sub, got_o), best), (t, k, got_o)
            results.append((best, got_o))
        wk = ao.max_score_select(results, MOS)
        tied = [k for k in range(K) if _score_ok(results[k][0], results[wk][0])]
        assert bk[t] in tied and (bo[t], bs[t]) == (a_o[t * K + bk[t]], a_s[t * K + bk[t]]), (t, bk[t], tied)
