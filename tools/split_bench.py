"""Cost of the per-segment offsets (b2_split_tracks) at the bench shape, alone and after the sync step it follows.

    python tools/split_bench.py [--pairs 256] [--ratios 5] [--penalty 20] [--repeats 10] [--warmup 2]
                                [--split-max-offset-seconds S] [--max-segments N] [--split-direction {-1,1}]
                                [--split-breaks D1,D2,..]

The workload is bench.py's (BASELINE configs[2]): 256 two-hour pairs (synth.make_pairs, about 1 200 cues each), K = 5,
+-60 s, PCM synthesised on the device.  Half the pairs get a planted 90 s cut in the middle: 9 000 windows of their
video are removed halfway and the end padded with silence, so their subtitles after the cut sit 90 s later than the
audio.  The sync step is BatchSynchronizer.sync_device with speech_video covering every video (the references the
split reads); the split is split_tracks over its results.  Timed with CUDA events on one stream, after warm-up, in
alternating repeats: the split alone over one sync step's results (including the read-back of best_k that forms the
ratio list), and sync + split.  Reports DP cells (units x window offsets, summed over the tracks) per second of the
split alone, the segment counts of the cut and uncut pairs at a few penalties, and the GPU's name, power limit and SM
clock read in the same run.  Needs an H100.

--split-max-offset-seconds (default: the sync window, +-60 s) sets the split's own window
(split_tracks(split_max_offset_seconds=...), b2_split_tracks_wide): the second half of a cut pair needs
true_offset - 9000 frames, which the +-60 s window cannot hold for any of the bench's seeds.  The run then also
reports the CTAs per track's cluster (ceil(window / 16 384)), and, per penalty, how many cut pairs come back as exactly
two segments at true_offset and true_offset - 9000 with the break in the middle cue, and how many uncut pairs stay
whole.

--max-segments N also times the capped split (split_tracks(max_segments=N), b2_split_tracks_capped) alternating with the
uncapped one in the same repeats, and reports under "capped": its median time, per penalty 0, 20, 200 and 2 000 the
cut pairs found as exactly two segments at true_offset and true_offset - 9000 and the uncut pairs that stay whole, and
at penalty 0 the quantiles of split_profile[:, 1] - split_profile[:, 0] over cut and over uncut pairs (N >= 2).

--split-direction D also times the directed split (split_tracks(split_direction=D), b2_split_tracks_directed) alternating
with the undirected one in the same repeats, and reports under "directed": its median time, and for both directions
(-1 fits the cut pairs: their later cues sit 90 s earlier) at penalties 0, 20, 200, 2 000 and 20 000 the cut pairs found
as exactly two segments at true_offset and true_offset - 9000, the uncut pairs that stay whole, and the median segment
count of each group.

--split-breaks D1,D2,.. (each +1 or -1, e.g. -1 or +1,+1,+1) also times the split along those breaks
(split_tracks(split_breaks=...), b2_split_tracks_breaks) alternating with the others in the same repeats, and, unless
they are given, the capped split at N = len(breaks) + 1 and the directed one in the first break's direction, for the
cost beside them.  It reports under "breaks": its median time and its ratio to the plain, capped and directed calls'
medians; per penalty 0, 20, 200, 2 000 and 20 000 the cut pairs found as exactly two segments at true_offset and
true_offset - 9000, the uncut pairs that stay whole, the median segment count of each group and the histogram of
segment counts; and, per penalty, the quantiles of split_profile[:, 1] - split_profile[:, 0] over cut and over uncut
pairs.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from tracks_bench import FPW, FRAME_RATE, SAMPLE_RATE, gpu_info  # noqa: E402

CUT = 9000   # windows of 10 ms: 90 s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=256)
    ap.add_argument("--ratios", type=int, default=5)
    ap.add_argument("--penalty", type=float, default=20.0)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--split-max-offset-seconds", type=float, default=None)
    ap.add_argument("--max-segments", type=int, default=None)
    ap.add_argument("--split-direction", type=int, choices=(-1, 1), default=None)
    ap.add_argument("--split-breaks", type=str, default=None)
    args = ap.parse_args()
    brk = None
    if args.split_breaks is not None:
        brk = tuple(int(x) for x in args.split_breaks.split(","))
        if args.max_segments is None:
            args.max_segments = len(brk) + 1
        if args.split_direction is None:
            args.split_direction = brk[0]

    import torch
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.synth import BENCH_RATIOS, make_pairs
    from oracle import aligner_oracle as ao
    from oracle import raster_oracle as ro

    if not torch.cuda.is_available():
        sys.exit("split_bench: no CUDA device (this measurement runs on the GPU only)")
    info = gpu_info()
    print(json.dumps(dict(info, event="gpu")), flush=True)
    dev = torch.device("cuda", 0)
    ratios = list(BENCH_RATIOS[: args.ratios])
    B = args.pairs
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    bs = BatchSynchronizer(ratios, FRAME_RATE, SAMPLE_RATE, 0.0, max_offset_seconds=60)
    bs.use_torch_stream()
    h = bs.handle
    pairs = make_pairs([13 + b for b in range(B)], 7200.0, ratios, handle=h)
    wc = pairs.window_class.copy()
    cut = np.zeros(B, bool)
    for b in range(0, B, 2):   # the planted cut: the middle 90 s of the video removed
        a, e = int(pairs.win_off[b]), int(pairs.win_off[b + 1])
        mid = a + (e - a) // 2
        wc[a:e] = np.concatenate([wc[a:mid], wc[mid + CUT:e], np.zeros(CUT, wc.dtype)])
        cut[b] = True
    n_win = int(pairs.win_off[-1])
    cls_d = torch.from_numpy(wc).to(dev)
    pcm = torch.empty(n_win * FPW, dtype=torch.int16, device=dev)
    h.synth_pcm(cls_d.data_ptr(), n_win, FPW, 1234, out=pcm.data_ptr(), memspace=_native.B2_DEVICE)
    del cls_d
    pcm_off = pairs.win_off * FPW
    cs, ce, co = pairs.cue_start, pairs.cue_end, pairs.cue_off
    tv = np.arange(B, dtype=np.int32)
    sv = np.arange(B)

    def sync():
        return bs.sync_device(pcm, pcm_off, cs, ce, co, speech_video=sv)

    def split(out, pen=args.penalty):
        return bs.split_tracks(out, tv, cs, ce, co, split_penalty=pen,
                               split_max_offset_seconds=args.split_max_offset_seconds)

    def split_capped(out, pen=args.penalty):
        return bs.split_tracks(out, tv, cs, ce, co, split_penalty=pen,
                               split_max_offset_seconds=args.split_max_offset_seconds, max_segments=args.max_segments)

    def split_directed(out, pen=args.penalty, d=args.split_direction):
        return bs.split_tracks(out, tv, cs, ce, co, split_penalty=pen,
                               split_max_offset_seconds=args.split_max_offset_seconds, split_direction=d)

    def split_breaks(out, pen=args.penalty):
        return bs.split_tracks(out, tv, cs, ce, co, split_penalty=pen,
                               split_max_offset_seconds=args.split_max_offset_seconds, split_breaks=brk)

    def timed(fn, n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(n):
            fn()
        e1.record(stream)
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n

    capped = args.max_segments is not None
    directed = args.split_direction is not None
    out = sync()
    for _ in range(args.warmup):
        split(out)
        split(sync())
        if capped:
            split_capped(out)
        if directed:
            split_directed(out)
        if brk is not None:
            split_breaks(out)
    torch.cuda.synchronize(dev)
    split_ms, both_ms, capped_ms, directed_ms, breaks_ms = [], [], [], [], []
    for _ in range(args.repeats):   # alternating
        split_ms.append(timed(lambda: split(out), 1))
        both_ms.append(timed(lambda: split(sync()), 1))
        if capped:
            capped_ms.append(timed(lambda: split_capped(out), 1))
        if directed:
            directed_ms.append(timed(lambda: split_directed(out), 1))
        if brk is not None:
            breaks_ms.append(timed(lambda: split_breaks(out), 1))
    res = split(out)
    torch.cuda.synchronize(dev)
    ns = res["n_segments"].cpu().numpy()
    # DP cells: units (runs of the mask at the track's ratio, at least 1) x window offsets
    ref_len = np.diff(out["speech_off"])
    mos = bs.max_offset_samples if args.split_max_offset_seconds is None else \
        abs(int(args.split_max_offset_seconds * SAMPLE_RATE))
    cells = 0
    ctas = set()
    for t in range(B):
        if np.isnan(res["ratio"][t]):
            continue
        mask = ro.rasterize(cs[co[t]:co[t + 1]], ce[co[t]:co[t + 1]], None, SAMPLE_RATE, 0.0, res["ratio"][t])[0] > 0
        o_lo, o_hi = ao.offset_range(int(ref_len[t]), len(mask), mos)
        cells += max(1, int(np.count_nonzero(np.diff(np.concatenate([[0], mask.astype(np.int8)])) == 1))) * \
            max(0, o_hi - o_lo + 1)
        ctas.add(-(-max(0, o_hi - o_lo + 1) // 16384))
    med_split, med_both = float(np.median(split_ms)), float(np.median(both_ms))
    # segments per pair at other penalties (the VAD reference is noisy: small penalties split on its noise too)
    # a cut pair is found when its cues take true_offset before the middle of the video and true_offset - CUT after
    # it (cues are rasterised at the pair's ratio; the cut sits at the middle window of the video)
    segs = {}
    for pen in (args.penalty, 200.0, 2000.0, 20000.0):
        r = split(out, pen)
        n_s, c_o = r["n_segments"].cpu().numpy(), r["cue_offset"].cpu().numpy()
        found = 0
        for b in np.flatnonzero(cut):
            if n_s[b] != 2 or np.isnan(r["ratio"][b]):
                continue
            o = c_o[co[b]:co[b + 1]]
            t0 = int(pairs.true_offset[b])
            before = np.flatnonzero(o == t0)
            after = np.flatnonzero(o == t0 - CUT)
            found += int(len(before) + len(after) == len(o) and len(before) and len(after)
                         and before.max() < after.min())
        segs[str(pen)] = dict(cut_median=float(np.median(n_s[cut])), uncut_median=float(np.median(n_s[~cut])),
                              cut_two=int(np.sum(n_s[cut] == 2)), uncut_one=int(np.sum(n_s[~cut] == 1)),
                              cut_two_at_true_offsets=found)
    extra = {}
    if capped:
        csegs = {}
        for pen in (0.0, 20.0, 200.0, 2000.0):
            r = split_capped(out, pen)
            n_s, c_o = r["n_segments"].cpu().numpy(), r["cue_offset"].cpu().numpy()
            found = 0
            for b in np.flatnonzero(cut):
                if n_s[b] != 2:
                    continue
                o = c_o[co[b]:co[b + 1]]
                t0 = int(pairs.true_offset[b])
                before, after = np.flatnonzero(o == t0), np.flatnonzero(o == t0 - CUT)
                found += int(len(before) + len(after) == len(o) and len(before) and len(after)
                             and before.max() < after.min())
            csegs[str(pen)] = dict(cut_two_at_true_offsets=found, uncut_one=int(np.sum(n_s[~cut] == 1)),
                                   cut_two=int(np.sum(n_s[cut] == 2)), segments_hist=np.bincount(
                                       np.maximum(n_s, 0), minlength=args.max_segments + 1).tolist())
            if pen == 0.0 and args.max_segments >= 2:
                prof = r["split_profile"].cpu().numpy()
                gain = prof[:, 1] - prof[:, 0]
                q = [0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0]
                ok = ~np.isnan(gain)
                gains = dict(quantiles=q, cut=np.quantile(gain[cut & ok], q).round(1).tolist(),
                             uncut=np.quantile(gain[~cut & ok], q).round(1).tolist())
        extra = dict(capped=dict(max_segments=args.max_segments, split_ms=round(float(np.median(capped_ms)), 3),
                                 split_ms_all=[round(x, 3) for x in capped_ms],
                                 ratio_to_uncapped=round(float(np.median(capped_ms)) / med_split, 2),
                                 segments_by_penalty=csegs, **({"profile_gain_at_penalty_0": gains}
                                                               if args.max_segments >= 2 else {})))
    if directed:
        dsegs = {}
        for d in (-1, 1):
            for pen in (0.0, 20.0, 200.0, 2000.0, 20000.0):
                r = split_directed(out, pen, d)
                n_s, c_o = r["n_segments"].cpu().numpy(), r["cue_offset"].cpu().numpy()
                found = 0
                for b in np.flatnonzero(cut):
                    if n_s[b] != 2:
                        continue
                    o = c_o[co[b]:co[b + 1]]
                    t0 = int(pairs.true_offset[b])
                    before, after = np.flatnonzero(o == t0), np.flatnonzero(o == t0 - CUT)
                    found += int(len(before) + len(after) == len(o) and len(before) and len(after)
                                 and before.max() < after.min())
                dsegs["%+d@%s" % (d, pen)] = dict(cut_two_at_true_offsets=found,
                                                  uncut_one=int(np.sum(n_s[~cut] == 1)),
                                                  cut_median=float(np.median(n_s[cut])),
                                                  uncut_median=float(np.median(n_s[~cut])))
        extra["directed"] = dict(split_direction=args.split_direction,
                                 split_ms=round(float(np.median(directed_ms)), 3),
                                 split_ms_all=[round(x, 3) for x in directed_ms],
                                 ratio_to_undirected=round(float(np.median(directed_ms)) / med_split, 2),
                                 segments_by_direction_and_penalty=dsegs)
    if brk is not None:
        bsegs, bgain = {}, {}
        q = [0.0, 0.05, 0.25, 0.5, 0.75, 0.95, 1.0]
        for pen in (0.0, 20.0, 200.0, 2000.0, 20000.0):
            r = split_breaks(out, pen)
            n_s, c_o = r["n_segments"].cpu().numpy(), r["cue_offset"].cpu().numpy()
            found = 0
            for b in np.flatnonzero(cut):
                if n_s[b] != 2:
                    continue
                o = c_o[co[b]:co[b + 1]]
                t0 = int(pairs.true_offset[b])
                before, after = np.flatnonzero(o == t0), np.flatnonzero(o == t0 - CUT)
                found += int(len(before) + len(after) == len(o) and len(before) and len(after)
                             and before.max() < after.min())
            bsegs[str(pen)] = dict(cut_two_at_true_offsets=found, uncut_one=int(np.sum(n_s[~cut] == 1)),
                                   cut_median=float(np.median(n_s[cut])), uncut_median=float(np.median(n_s[~cut])),
                                   segments_hist=np.bincount(np.maximum(n_s, 0), minlength=len(brk) + 2).tolist())
            prof = r["split_profile"].cpu().numpy()
            gain = prof[:, 1] - prof[:, 0]
            ok = np.isfinite(gain)
            bgain[str(pen)] = dict(cut=np.quantile(gain[cut & ok], q).round(1).tolist() if (cut & ok).any() else [],
                                   uncut=np.quantile(gain[~cut & ok], q).round(1).tolist() if (~cut & ok).any() else [],
                                   not_finite=int(np.sum(~ok)))
        med_b = float(np.median(breaks_ms))
        extra["breaks"] = dict(split_breaks=list(brk), split_ms=round(med_b, 3),
                               split_ms_all=[round(x, 3) for x in breaks_ms],
                               ratio_to_plain=round(med_b / med_split, 2),
                               ratio_to_capped=round(med_b / float(np.median(capped_ms)), 2),
                               ratio_to_directed=round(med_b / float(np.median(directed_ms)), 2),
                               segments_by_penalty=bsegs,
                               profile_gain_quantiles=q, profile_gain_by_penalty=bgain)
    print(json.dumps(dict(info, event="measure", pairs=B, K=len(ratios), penalty=args.penalty, cues=int(co[-1]),
                          split_max_offset_samples=mos, cluster_ctas=sorted(ctas),
                          split_ms=round(med_split, 3), split_ms_all=[round(x, 3) for x in split_ms],
                          sync_plus_split_ms=round(med_both, 3), sync_plus_split_ms_all=[round(x, 3) for x in both_ms],
                          dp_cells=int(cells), dp_cells_per_s=round(cells / (med_split * 1e-3), 1),
                          cut_pairs=int(cut.sum()), cut_pairs_with_two_segments=int(np.sum(ns[cut] == 2)),
                          uncut_pairs_with_one_segment=int(np.sum(ns[~cut] == 1)), segments_by_penalty=segs, **extra)),
          flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
