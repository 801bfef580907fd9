"""CPU suite for the host planners past 32-bit sample and byte indices (csrc/sync_plan.h through
tests/host_emul/plan_emul, csrc/ingest_plan.h through tests/host_emul/ingest_emul).

A library's PCM buffer passes element 2^31 after about 18 videos of two hours at 16 kHz, and byte 2^32 soon after;
one video of 12.4 h at 48 kHz is longer than 2^31 samples on its own.  Here:
  * a batch placed at pcm_off values just below and above 2^31, 2^32 and 2^33 plans exactly the batch at offset 0
    with every sample index shifted: chunk tables, segment items, staged ranges; sub-batch cuts, reference offsets,
    frame tables and energy floors unchanged;
  * one video longer than 2^31 samples (48 kHz, 44.1 kHz, 22.05 kHz's ragged 100 s calls, auditok's chunks) gets the
    chunk table and reference length of the reference's chunk loop, computed here in Python integers;
  * sampled segments whose first sample lies past 2^31 and 2^32 get the items of their detector calls;
  * an ingest stream whose byte, sample and window counters pass 2^31 and 2^32, with odd-byte pushes straddling each
    mark, is cut into the spans of the one-shot detector."""
import numpy as np
import pytest

from oracle import auditok_oracle as ad
from sync_plan import plan
from test_ingest_cpu import check_spans

M31, M32, M33 = 1 << 31, 1 << 32, 1 << 33
# placements of the batch's first sample: around element 2^31, byte 2^32 (element 2^31), element 2^32 (byte 2^33)
BASES = [M31 - 4321, M31 + 8, M32 - 1, M32 + 3, M33 - 16]
SHIFTED = ("ch_pcm", "det_end", "item_start", "item_end", "stage_lo", "stage_hi")


def _call(fr):
    """The reference's 100 s read in samples, and whether energy / ZCR restarts its window grid there."""
    call = (2 * fr // 100) * 5000
    return call, call % int(fr / 100 + 0.5) != 0


def _batch(fr, detector, base, seg=False):
    """A b2_sync_tracks(_seg) request of five videos starting at sample `base`: lengths around the window, the
    100 s read and sub-window; three tracks per video but the second; with seg, video 3 is a segment video."""
    fpw = fr // 100
    call, _ = _call(fr)
    n = [call + fpw + 1, 0, 3 * call - 7, fpw - 1, 95 * fr + fpw // 2]
    pcm_off = base + np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    per = [3, 0, 3, 3, 3]
    tv = np.repeat(np.arange(5), per).astype(np.int32)
    T = len(tv)
    st = np.tile([1.0, 5.0, 9.5, 40.0], T)
    req = dict(pcm_off=pcm_off, track_video=tv, cue_start=st, cue_end=st + 2.0, cue_off=np.arange(T + 1) * 4,
               ratios=[0.96, 1.0, 1.04], frame_rate=fr, energy_threshold=100000, detector=detector,
               chunk_samples=333 * fpw + 7 if detector else 0, subbatches="3", lane=1)
    if seg:
        total = n[2] / fr
        lo = [0, 120 * fr - 3, 2 * call]
        hi = [30 * fr, 150 * fr, n[2]]
        req.update(who="sync_tracks_seg", seg_video=[2], seg_total=[total], seg_off=[0, 3], seg_start=[0, 120, 200],
                   seg_lo=lo, seg_hi=hi)
    return req


def _ok(p):
    assert p["status"] == 0, p["err"]
    return p


@pytest.mark.parametrize("fr,detector", [(16000, 0), (48000, 0), (22050, 0), (44100, 0), (16000, 1), (48000, 1)])
@pytest.mark.parametrize("seg", [False, True])
def test_far_placement_plans_the_batch_at_offset_0_shifted(fr, detector, seg):
    near = _ok(plan(**_batch(fr, detector, 0, seg)))
    assert near["ch_pcm"].size or not (detector or _call(fr)[1])
    if seg:
        assert near["item_start"].size > 1
    for base in BASES:
        far = _ok(plan(**_batch(fr, detector, base, seg)))
        assert far.keys() == near.keys()
        for k, v in near.items():
            if k in SHIFTED:
                # item_start's spare last entry repeats the last start, shifted like the others
                assert np.array_equal(far[k], v + base), (k, base, far[k][:4], v[:4])
            elif k == "audio_samples" or not isinstance(v, np.ndarray):
                assert np.array_equal(far[k], v) if isinstance(v, np.ndarray) else far[k] == v, (k, base)
            else:
                assert np.array_equal(far[k], v), (k, base, far[k][:8], v[:8])


def _chunk_loop(n, fpw, step):
    """The reference's chunk loop over n samples in calls of step samples (0: one call): chunk ends and frame ends."""
    ends, frames, s, f = [], [], 0, 0
    while s < n:
        e = min(n, s + step) if step > 0 else n
        f += -(-(e - s) // fpw)
        ends.append(e)
        frames.append(f)
        s = e
    return ends, frames


@pytest.mark.parametrize("fr,detector,extra", [(48000, 0, 4321), (44100, 0, 1), (22050, 0, 333), (16000, 0, 7),
                                               (48000, 1, 4321), (44100, 1, 4410000 - 1)])
def test_one_video_past_2_31_samples(fr, detector, extra):
    """One video of 2^31 + extra samples, placed behind an empty video and then past 2^32: its chunk table, reference
    length and (auditok) the energy floor of its short last block."""
    n = M31 + extra
    fpw = int(fr / 100 + 0.5) if not detector else fr // 100
    call, ragged = _call(fr)
    step = (4800 * fpw + 13) if detector else (call if ragged else 0)
    for base in (0, M32 + 8):
        req = dict(pcm_off=[base, base, base + n], track_video=[1, 1], cue_start=[10.0, 40000.0],
                   cue_end=[12.0, 40002.0], cue_off=[0, 1, 2], ratios=[1.0], frame_rate=fr, energy_threshold=100000,
                   detector=detector, chunk_samples=step if detector else 0, lane=1)
        p = _ok(plan(**req))
        ends, frames = _chunk_loop(n, fpw, step)
        assert p["ref_off"].tolist() == [0, 0, frames[-1]]
        assert p["audio_samples"].tolist() == [n]
        if not p["ch_pcm"].size:   # energy / ZCR whose calls divide into windows: one launch entry per video
            assert not (detector or ragged)
            continue
        # the empty video has no chunk; the long video's follow
        assert p["ch_first"].tolist() == [0, 0, len(ends)]
        assert p["ch_pcm"].tolist() == [base] + [base + e for e in ends]
        assert p["ch_out"].tolist() == [0] + frames
        rem = [(e - s) % fpw for s, e in zip([0] + ends[:-1], ends)]
        if detector:
            assert p["ch_tail"].tolist() == [ad.energy_floor(r) if r else 0 for r in rem]
        else:   # energy / ZCR: a call's ragged last window never reaches its floor
            assert p["ch_tail"].tolist() == [(1 << 63) - 1 if r else 0 for r in rem]


@pytest.mark.parametrize("fr,detector", [(48000, 0), (22050, 0), (48000, 1)])
def test_segments_past_2_31_samples(fr, detector):
    """A video an hour longer than 2^31 samples whose sampled segments start past samples 2^31 and 2^32 of the call's
    buffer: the items of
    their detector calls, their frames, and the ranges a host call stages."""
    fpw = int(fr / 100 + 0.5) if not detector else fr // 100
    call, ragged = _call(fr)
    step = 4800 * fpw + 13 if detector else (call if ragged else 0)
    total_s = M31 // fr + 3600
    n = total_s * fr
    starts = [2 * 3600, M31 // fr - 1, M31 // fr + 60, total_s - 100]
    lo = [s * fr for s in starts]
    hi = [min(n, a + 200 * fr + 17) for a in lo]
    for base in (0, M31 + 8, M32 - 16):
        req = dict(who="sync_tracks_seg", pcm_off=[base, base + n], track_video=[0], cue_start=[10.0], cue_end=[12.0],
                   cue_off=[0, 1], ratios=[1.0], frame_rate=fr, energy_threshold=100000, detector=detector,
                   chunk_samples=step if detector else 0, seg_video=[0], seg_total=[float(total_s)],
                   seg_off=[0, len(starts)], seg_start=starts, seg_lo=lo, seg_hi=hi, lane=1)
        p = _ok(plan(**req))
        i_start, i_end, i_out, f = [], [], [0], 0
        for a, b in zip(lo, hi):
            ends, frames = _chunk_loop(b - a, fpw, step)
            i_start += [base + a + e0 for e0 in [0] + ends[:-1]]
            i_end += [base + a + e for e in ends]
            i_out += [f + x for x in frames]
            f += frames[-1]
        assert p["item_start"].tolist() == i_start + i_start[-1:]
        assert p["item_end"].tolist() == i_end
        assert p["item_out"].tolist() == i_out
        assert p["item_first"].tolist() == [0, len(i_end)]
        assert p["det_end"][0] == base                          # the segment video's main entry is empty
        merged = []                                             # the staged ranges: the segments' samples, merged
        for a0, b0 in sorted(zip(lo, hi)):
            if merged and a0 <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], b0)
            else:
                merged.append([a0, b0])
        assert p["stage_lo"].tolist() == [base + m[0] for m in merged]
        assert p["stage_hi"].tolist() == [base + m[1] for m in merged]


@pytest.mark.parametrize("auditok,fpw,chunk", [(False, 480, 0), (False, 441, 0), (False, 221, 2205000),
                                               (True, 480, 4800000), (True, 441, 4800 * 441 + 13)])
def test_ingest_counters_past_2_31_and_2_32(auditok, fpw, chunk):
    """Two streams pushed to beyond 2^33 bytes: odd-byte pushes end one byte short of, and straddle, bytes 2^32 and
    2^33 (samples 2^31 and 2^32), interleaved with the other stream, which passes the marks in window-sized steps."""
    ops, at = [], [0, 0]

    def push(v, to):
        ops.append(("p", v, to - at[v]))
        at[v] = to

    for mark in (M31, M32, M33):
        push(0, mark - 1)               # one byte short of the mark: the last sample is incomplete
        push(1, mark - 2 * fpw - 3)
        push(0, mark + 2)               # straddles it: the held byte joins the next sample
        push(1, mark + 2 * fpw + 1)
        push(0, mark + 2 * fpw * 3 + 1)
    push(0, M33 + M31 + 5)
    push(1, M33 + 2 * (chunk or 7 * fpw) + 3)
    ops += [("f", 0), ("f", 1)]
    check_spans(2, fpw, auditok, chunk, ops)
