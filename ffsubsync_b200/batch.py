"""Batch front end of the hot path: many (video, subtitle) pairs per call.

``BatchSynchronizer.sync_device`` keeps everything resident in HBM (PCM in, per-pair
``(score, offset, ratio index)`` out) and launches on torch's current CUDA stream, so callers
can time it with torch.cuda.Event and chain it with NCCL collectives (ffsubsync_b200.distributed).
``sync_host`` is the same call with host buffers (numpy / pinned tensors): the C library copies
the PCM in, runs the identical kernels and copies the results out.

This is what ``ffs ref.mkv -i in.srt`` does per pair in the reference - VideoSpeechTransformer.fit
(ffsubsync/ffsubsync.py:637) followed by MaxScoreAligner over the ratio grid (:196-235) - for a
batch, with the subtitle scaling + rasterisation fused into one kernel.
"""
import contextlib
from typing import Optional, Sequence

import numpy as np

from . import _native
from .constants import (BATCH_VADS, DEFAULT_APPLY_OFFSET_SECONDS, DEFAULT_ENERGY_THRESHOLD,
                        DEFAULT_MAX_FRAMERATE_DEVIATION, DEFAULT_MAX_OFFSET_SECONDS, DEFAULT_MIN_SCORE,
                        DEFAULT_QUALITY_MAX_OFFSET_SECONDS, SAMPLE_RATE, detector_chunk_bytes)


def load_serialized_speech(paths, non_speech_label: float = 0.0, stored: bool = False):
    """Batch ingest of ``--serialize-speech`` / ``--make-test-case`` artefacts (``.npz`` with key
    "speech", or ``.npy``): each file goes through DeserializeSpeechTransformer
    (ffsubsync/speech_transformers.py:987-1009: values < 1 become ``non_speech_label``).
    Returns (signals float32 back to back, offsets int64[B+1]) ready for ``sync_signals``.
    stored=True: the stored values themselves as float64, back to back, without the rule (non_speech_label is not
    read), ready for the ``sig`` / ``sig_off`` arguments of the sync methods, which apply the rule at their own
    label."""
    from .speech_transformers import DeserializeSpeechTransformer, load_stored_speech
    if stored:
        sigs = [np.asarray(load_stored_speech(p), dtype=np.float64).ravel() for p in paths]
        off = np.concatenate([[0], np.cumsum([len(s) for s in sigs])]).astype(np.int64)
        return (np.concatenate(sigs) if sigs else np.zeros(0, np.float64)), off
    sigs = [np.asarray(DeserializeSpeechTransformer(non_speech_label).fit(p).transform(), dtype=np.float32)
            for p in paths]
    off = np.concatenate([[0], np.cumsum([len(s) for s in sigs])]).astype(np.int64)
    return (np.concatenate(sigs) if sigs else np.zeros(0, np.float32)), off


def save_serialized_speech(paths, speech, speech_off, speech_video=None, seg_video=None) -> None:
    """Write what ``--serialize-speech`` writes (ffsubsync/ffsubsync.py:639-644): ``np.savez_compressed(paths[i],
    speech=...)`` of listed video i's signal ``speech[speech_off[i]: speech_off[i+1]]`` (the ``speech`` /
    ``speech_off`` results of a sync method called with ``speech_video``), readable by ``load_stored_speech`` and
    ``load_serialized_speech``.  Choosing the names (the reference's ``_npy_savename``) is the caller's job.
    A CUDA ``speech`` is copied to the host after a synchronisation of its whole device, so the signals a device sync
    method enqueued on its handle's own stream are complete before they are read.
    ``seg_video``: the call's segment videos (``--multi-segment-sync``); ``speech_video``, the call's listed videos, is
    then required.  A listed segment video whose signal has no frame > 0 is refused with the reference's ValueError
    before anything is written, as MultiSegmentVideoSpeechTransformer.fit raises before the reference serializes.
    This is the rule behind the tracks' ``best_k == B2_BEST_K_NO_SPEECH``, so it also covers a call without tracks."""
    if hasattr(speech, "cpu"):
        import torch
        if speech.is_cuda:
            torch.cuda.synchronize(speech.device)
        speech = speech.cpu().numpy()
    speech = np.asarray(speech)
    speech_off = np.asarray(speech_off, dtype=np.int64)
    if len(paths) != len(speech_off) - 1:
        raise ValueError("%d paths for %d signals" % (len(paths), len(speech_off) - 1))
    if seg_video is not None:
        if speech_video is None:
            raise ValueError("seg_video needs speech_video, the videos the signals belong to")
        if len(speech_video) != len(paths):
            raise ValueError("speech_video has %d entries for %d paths" % (len(speech_video), len(paths)))
        seg = {int(v) for v in np.asarray(seg_video).ravel()}
        for i, v in enumerate(np.asarray(speech_video).ravel()):
            if int(v) in seg and not np.any(speech[speech_off[i]: speech_off[i + 1]] > 0):
                raise ValueError("video %d: %s" % (int(v), _NO_SPEECH_MESSAGE))
    for i, path in enumerate(paths):
        np.savez_compressed(path, speech=np.asarray(speech[speech_off[i]: speech_off[i + 1]], dtype=np.float64))


# keyword arguments of the sync methods that describe the embedded subtitle streams of a subs_then_ detector
_STREAM_ARGS = ("ref_cue_start", "ref_cue_end", "ref_cue_off", "ref_stream_video", "ref_cue_content", "ref_cue_keep")
# keyword arguments of the sync methods that describe the videos' PGS (bitmap subtitle) display intervals
_PGS_ARGS = ("pgs_start", "pgs_end", "pgs_off", "pgs_video")
# keyword arguments of the sync methods that give videos a serialized speech signal as reference
_SIG_ARGS = ("sig", "sig_off", "sig_video")
# keyword arguments of the sync methods that give videos sampled segments as reference (--multi-segment-sync)
_SEG_ARGS = ("seg_video", "seg_total", "seg_off", "seg_start", "seg_lo", "seg_hi")
# subtitle-file references (the reference's SUBTITLE_EXTENSIONS), which the batched calls do not take
_SUBTITLE_EXTENSIONS = ("srt", "ass", "ssa", "sub")
# sync_media: the segment field of a decoder job that probes a PGS stream instead of decoding audio
_PGS_JOB = "pgs"
_NO_SPEECH_MESSAGE = ("Unable to detect speech in any sampled segment. "
                      "Perhaps try specifying a different stream / track, or a different vad.")


def segment_table(pcm_off, frame_rate: int, videos=None, totals=None, segment_count: int = 8,
                  segment_duration: int = 60, skip_intro_outro: bool = False, piece_samples=None) -> dict:
    """The segment keyword arguments of the sync methods (``--multi-segment-sync``) for the videos ``videos`` (default:
    every video of pcm_off [V+1]), with the reference's knobs ``segment_count``, ``segment_duration`` and
    ``skip_intro_outro``.  Each video's starts are MultiSegmentVideoSpeechTransformer._segment_starts of its duration
    ``totals[i]`` (seconds, e.g. ffprobe's; default: its samples / frame_rate, as the transformer probes raw PCM).
    Two layouts of a video's PCM range:
    - ``piece_samples`` None: the range holds the video's whole decode; segment s is the slice lo = min(n, round(s *
      frame_rate)), hi = min(n, lo + round(segment_duration * frame_rate)).
    - ``piece_samples[i]``: the range holds only the sampled windows (``ffmpeg -ss s -t segment_duration``) back to
      back in start order, with these sample counts (one per start; a short last piece is fine).
    Returns dict(seg_video, seg_total, seg_off, seg_start, seg_lo, seg_hi)."""
    from .speech_transformers import MultiSegmentVideoSpeechTransformer
    pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
    V = len(pcm_off) - 1
    videos = np.arange(V) if videos is None else np.ascontiguousarray(videos, dtype=np.int64)
    t = MultiSegmentVideoSpeechTransformer(vad="energy", sample_rate=SAMPLE_RATE, frame_rate=frame_rate,
                                           non_speech_label=0.0, segment_count=segment_count,
                                           segment_duration=segment_duration, skip_intro_outro=skip_intro_outro)
    total_out, off, start, lo, hi = [], [0], [], [], []
    for i, v in enumerate(videos):
        n = int(pcm_off[v + 1] - pcm_off[v])
        total = float(totals[i]) if totals is not None else n / float(frame_rate)
        starts = t._segment_starts(total)
        if piece_samples is None:
            for s in starts:
                a = min(n, int(round(s * frame_rate)))
                lo.append(a)
                hi.append(min(n, a + int(round(segment_duration * frame_rate))))
        else:
            pieces = [int(x) for x in piece_samples[i]]
            if len(pieces) != len(starts) or sum(pieces) != n:
                raise ValueError("video %d: %d decoded pieces of %d samples for %d starts in a range of %d samples"
                                 % (int(v), len(pieces), sum(pieces), len(starts), n))
            at = 0
            for m in pieces:
                lo.append(at)
                hi.append(at + m)
                at += m
        start += [int(s) for s in starts]
        total_out.append(total)
        off.append(len(start))
    return dict(seg_video=np.asarray(videos, dtype=np.int32), seg_total=np.asarray(total_out, dtype=np.float64),
                seg_off=np.asarray(off, dtype=np.int64), seg_start=np.asarray(start, dtype=np.int64),
                seg_lo=np.asarray(lo, dtype=np.int64), seg_hi=np.asarray(hi, dtype=np.int64))


def _is_unsupported(e: Exception) -> bool:
    return isinstance(e, _native.NativeError) and e.status == -6   # B2_ERR_UNSUPPORTED


class BatchSynchronizer:
    """``ratios``: the framerate ratio grid in list order.  A trailing ``None`` adds the golden-section search
    over [0.9, 1.1] as one more candidate, last in list order, the way the reference's list carries ``--gss``
    (``constants.framerate_ratios_to_try(gss=True)``); results then gain ``gss_ratio`` and ``best_k == K``
    (K = the grid's length) means the search won.

    ``vad``: the detector that turns PCM into the reference signal.  ``"energy_zcr"`` (default) is this package's
    energy / zero-crossing detector; ``"auditok"`` is the reference's auditok detector (``--vad auditok``) with its
    default constants (50 dB, min 0.2 s, max 5 s, 0.25 s of continuous silence), run over the reference's chunk loop
    (one detector call per 100 s).  ``energy_threshold`` / ``z_lo`` / ``z_hi`` belong to the energy detector and must
    stay at their defaults with ``"auditok"``.

    ``"subs_then_energy_zcr"`` / ``"subs_then_auditok"`` are the reference's ``subs_then_`` detectors (its default
    ``--vad subs_then_webrtc``, and ``subs_then_auditok``): a video with an embedded text subtitle stream is synced
    against that stream instead of its audio (VideoSpeechTransformer.fit, ffsubsync/speech_transformers.py:609-619),
    the others against the detector after the prefix.  The sync methods then take the candidate streams as
    keyword arguments: S streams of cues ``ref_cue_start`` / ``ref_cue_end`` (seconds, as parsed),
    ``ref_cue_off`` [S+1], ``ref_stream_video`` [S] (the video of each stream, non-decreasing) and either
    ``ref_cue_content`` (the cue texts: keep flags by the reference's metadata filter) or ``ref_cue_keep``.  Each
    video uses its stream with the largest ``max_end - start_seconds`` (the first on a tie), rasterised at
    ``sample_rate`` with level 1.0; a video with a stream must have an empty PCM range (its audio is never read;
    ``pcm`` may be None when no video has any).  Extracting the streams from containers (ffprobe / ffmpeg) and
    ``--reference-stream`` remain the caller's job; bitmap (PGS) streams come as their own arguments (below).  Without streams the results are those of the
    detector alone.

    PGS references (``--pgs-ref-stream``, with every ``vad``): the sync methods also take the display intervals of
    P videos' PGS (Blu-ray bitmap) subtitle streams as keyword arguments ``pgs_start`` / ``pgs_end`` (seconds:
    ffprobe's ``pts_time`` and ``pts_time + duration_time``, e.g. from ``speech_transformers.pgs_timings_from_packets``),
    ``pgs_off`` [P+1] and ``pgs_video`` [P] (increasing: at most one interval list per video).  Such a video is synced
    against its intervals rasterised by PGSSpeechTransformer's rule (b2_rasterize_pgs) instead of its audio or text
    stream - the reference tries ``--pgs-ref-stream`` first - and must have an empty PCM range.  Running ffprobe
    stays the caller's job.

    Serialized speech signals (``ffs ref.npz -i in.srt``, with every ``vad``): the sync methods also take the stored
    values of P videos' ``--serialize-speech`` / ``--make-test-case`` signals as keyword arguments ``sig`` (the values
    back to back, e.g. ``load_serialized_speech(paths, stored=True)``: a numpy array for the host methods, a CUDA
    tensor for the device ones; other dtypes are converted to float64), ``sig_off`` [P+1] and ``sig_video`` [P]
    (increasing: one signal per video).  Such a video is synced against its signal by DeserializeSpeechTransformer's
    rule at this synchroniser's ``non_speech_label``, frame ``(float)(x < 1.0 ? non_speech_label : x)`` - no detector
    runs for it - and must have an empty PCM range and no text or PGS reference.  Every stored value must be < 1.0 or
    exactly 1.0: a video with a value > 1.0 or NaN gets ``best_k == -2`` (``_native.B2_BEST_K_BAD_SIGNAL``), NaN
    scores and offsets 0 on all its tracks from the device methods, and the host methods raise ValueError naming the
    video and its first such frame."""

    def __init__(self, ratios: Sequence[Optional[float]], frame_rate: int = 16000, sample_rate: int = SAMPLE_RATE,
                 non_speech_label: float = 0.0, energy_threshold: int = DEFAULT_ENERGY_THRESHOLD,
                 z_lo: int = -1, z_hi: int = -1, start_seconds: float = 0.0,
                 max_offset_seconds: Optional[float] = DEFAULT_MAX_OFFSET_SECONDS,
                 device: Optional[int] = None, vad: str = "energy_zcr") -> None:
        if vad not in BATCH_VADS:
            raise ValueError("vad must be one of %s, not %r" % (", ".join(BATCH_VADS), vad))
        self.subs_then = vad.startswith("subs_then_")
        self.detector = vad[len("subs_then_"):] if self.subs_then else vad
        if self.detector == "auditok" and (energy_threshold != DEFAULT_ENERGY_THRESHOLD or z_lo != -1 or z_hi != -1):
            raise ValueError("energy_threshold / z_lo / z_hi configure the energy_zcr detector; vad=%r "
                             "does not read them" % vad)
        self.vad = vad
        ratios = list(ratios)
        self.gss = bool(ratios) and ratios[-1] is None
        grid = ratios[:-1] if self.gss else ratios
        if any(r is None for r in grid):
            raise ValueError("None (the golden-section search) may only be the last entry of ratios")
        if self.gss and not grid:
            raise ValueError("the golden-section search (None) needs at least one grid ratio before it")
        self.ratios = np.ascontiguousarray(grid, dtype=np.float64)
        self.frame_rate = frame_rate
        self.sample_rate = sample_rate
        self.non_speech_label = non_speech_label
        self.energy_threshold = energy_threshold
        self.z_lo, self.z_hi = z_lo, z_hi
        self.start_seconds = start_seconds
        # MaxScoreAligner.__init__ (ffsubsync/aligners.py:98-101)
        self.max_offset_samples = None if max_offset_seconds is None else abs(int(max_offset_seconds * sample_rate))
        self.handle = _native.get_handle(device)
        # auditok: samples per detector call, as VideoSpeechTransformer._chunks reads them (energy / ZCR: the library
        # derives its calls from the rates, b2_vad_call_samples)
        self.chunk_samples = detector_chunk_bytes(frame_rate, sample_rate) // 2

    @property
    def auditok(self) -> bool:
        return self.detector == "auditok"

    def _references(self, V: int, streams: dict):
        """(refs, pgs) of the keyword arguments: refs from _subs_refs, pgs from _pgs_refs.  A video with both a PGS
        reference and text streams keeps the PGS one (make_reference_pipe's order), so its text stream is dropped."""
        pgs = self._pgs_refs(V, {k: streams.pop(k) for k in _PGS_ARGS if k in streams})
        refs = self._subs_refs(V, streams)
        if refs is None or pgs is None or not np.any(refs[0] & pgs[0]):
            return refs, pgs
        return self._drop_text(V, refs, pgs[0] != 0), pgs

    def _all_refs(self, V: int, streams: dict, on_device: bool, seg=None):
        """(refs, pgs, sig, seg) of the keyword arguments: refs and pgs from _references, sig from _sig_refs, seg from
        _seg_refs.  A video with a signal and a text or PGS reference is refused: the reference tool's reference is a
        single file.  So is a video with segments and a PGS or signal reference; its text streams are dropped, since
        sampling is audio-only (the reference drops a ``subs_then_`` prefix).  ``seg``: segment videos declared
        elsewhere (an ingest session's (seg_video, seg_total)) in place of the segment keyword arguments."""
        if seg is None:
            seg = self._seg_refs(V, {k: streams.pop(k) for k in _SEG_ARGS if k in streams})
        sig = self._sig_refs(V, {k: streams.pop(k) for k in _SIG_ARGS if k in streams}, on_device)
        refs, pgs = self._references(V, streams)
        if seg is not None:
            is_seg = np.zeros(V, dtype=bool)
            is_seg[seg[0]] = True
            for r, what in ((pgs, "a PGS reference"), (sig, "a serialized signal")):
                both = np.flatnonzero(is_seg & (r[0] != 0)) if r is not None else []
                if len(both):
                    raise ValueError("video %d has sampled segments and %s; a video has one reference"
                                     % (int(both[0]), what))
            if refs is not None and np.any(is_seg & (refs[0] != 0)):
                refs = self._drop_text(V, refs, is_seg)
        if sig is not None:
            other = np.zeros(V, dtype=bool)
            for r in (refs, pgs):
                if r is not None:
                    other |= r[0] != 0
            both = np.flatnonzero(other & (sig[0] != 0))
            if len(both):
                raise ValueError("video %d has a serialized signal and a text / PGS reference; a video has one "
                                 "reference" % int(both[0]))
        return refs, pgs, sig, seg

    @staticmethod
    def _drop_text(V: int, refs, drop):
        """refs (from _subs_refs) without the text streams of the videos where drop[v] is set."""
        is_subs, rs, re_, rk, roff = refs
        keep_v = (is_subs != 0) & ~drop
        pick = np.concatenate([np.arange(roff[v], roff[v + 1]) for v in range(V) if keep_v[v]]
                              + [np.zeros(0, np.int64)]).astype(np.int64)
        lens = np.where(keep_v, np.diff(roff), 0)
        return (keep_v.astype(np.uint8), rs[pick], re_[pick], None if rk is None else rk[pick],
                np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))

    @staticmethod
    def _seg_refs(V: int, args: dict):
        """The segment table, or None when none is given: (seg_video i32, seg_total f64, seg_off, seg_start, seg_lo,
        seg_hi int64) for b2_sync_tracks_seg (e.g. from segment_table)."""
        if all(args.get(k) is None for k in _SEG_ARGS):
            return None
        missing = [k for k in _SEG_ARGS if args.get(k) is None]
        if missing:
            raise ValueError("segment references need %s" % ", ".join(_SEG_ARGS))
        video = np.ascontiguousarray(args["seg_video"], dtype=np.int32)
        if len(video) and (np.any(np.diff(video) <= 0) or video[0] < 0 or video[-1] >= V):
            raise ValueError("seg_video must be increasing video indices in [0, %d) (one segment table per video)" % V)
        return (video, np.ascontiguousarray(args["seg_total"], dtype=np.float64)) + tuple(
            np.ascontiguousarray(args[k], dtype=np.int64) for k in ("seg_off", "seg_start", "seg_lo", "seg_hi"))

    @staticmethod
    def _no_speech_videos(seg, best_k, track_video):
        """The segment videos whose tracks got B2_BEST_K_NO_SPEECH, ascending."""
        if seg is None:
            return []
        bk = np.asarray(best_k)
        return sorted({int(track_video[t]) for t in np.flatnonzero(bk == _native.B2_BEST_K_NO_SPEECH)})

    def _raise_no_speech(self, seg, best_k, track_video) -> None:
        """The host methods' error for the sentinel best_k == B2_BEST_K_NO_SPEECH."""
        vids = self._no_speech_videos(seg, best_k, track_video)
        if vids:
            raise ValueError("video %d: %s" % (vids[0], _NO_SPEECH_MESSAGE))

    def _sig_refs(self, V: int, args: dict, on_device: bool):
        """Each video's stored signal, or None when none is given: returns (ref_is_sig u8[V], x float64, sig_off
        int64[V+1]) for b2_sync_tracks_sig, x a numpy array (on_device False) or a CUDA tensor on the handle's device,
        sig_off absolute into x."""
        if all(args.get(k) is None for k in _SIG_ARGS):
            return None
        missing = [k for k in _SIG_ARGS if args.get(k) is None]
        if missing:
            raise ValueError("signal references need %s" % ", ".join(_SIG_ARGS))
        off = np.ascontiguousarray(args["sig_off"], dtype=np.int64)
        video = np.ascontiguousarray(args["sig_video"], dtype=np.int64)
        P = len(off) - 1
        if len(video) != P:
            raise ValueError("sig_video has %d entries for %d signals" % (len(video), P))
        if P and (np.any(np.diff(video) <= 0) or video[0] < 0 or video[-1] >= V):
            raise ValueError("sig_video must be increasing video indices in [0, %d) (one signal per video)" % V)
        x = args["sig"]
        if on_device:
            import torch
            dev = torch.device("cuda", self.handle.device)
            x = torch.as_tensor(x).to(device=dev, dtype=torch.float64).contiguous()
        else:
            x = np.ascontiguousarray(x.cpu().numpy() if hasattr(x, "cpu") else x, dtype=np.float64)
        if x.ndim != 1:
            raise ValueError("sig must be one-dimensional (the signals back to back)")
        if np.any(np.diff(off) < 0) or (P and (off[0] < 0 or off[-1] > len(x))):
            raise ValueError("sig_off must be non-decreasing and within sig")
        is_sig = np.zeros(V, dtype=np.uint8)
        is_sig[video] = 1
        # video v's range in x: its signal's, or an empty one where the previous range ended
        voff = np.empty(V + 1, dtype=np.int64)
        pos, i = (int(off[0]) if P else 0), 0
        for v in range(V):
            voff[v] = pos
            if i < P and video[i] == v:
                voff[v], pos = off[i], off[i + 1]
                i += 1
        voff[V] = pos
        return is_sig, x, voff

    @staticmethod
    def _bad_signals(sig):
        """{video: first frame} of the signal videos with a stored value > 1.0 or NaN (sig from _sig_refs)."""
        is_sig, x, voff = sig
        x = x.cpu().numpy() if hasattr(x, "cpu") else x
        bad = {}
        for v in np.flatnonzero(is_sig):
            out = np.flatnonzero(~(x[voff[v]: voff[v + 1]] <= 1.0))
            if len(out):
                bad[int(v)] = int(out[0])
        return bad

    def _raise_bad_signals(self, sig, best_k) -> None:
        """The host methods' error for the sentinel best_k == B2_BEST_K_BAD_SIGNAL."""
        if sig is None or not np.any(np.asarray(best_k) == _native.B2_BEST_K_BAD_SIGNAL):
            return
        v, f = sorted(self._bad_signals(sig).items())[0]
        x = sig[1]
        raise ValueError("video %d: its serialized signal holds %r at frame %d; stored values must be < 1.0 or "
                         "exactly 1.0" % (v, float(x[int(sig[2][v]) + f]), f))

    def _pgs_refs(self, V: int, args: dict):
        """Each video's PGS interval list, or None when none is given: returns (ref_is_pgs u8[V], pgs_start,
        pgs_end, pgs_off [V+1]) for b2_sync_tracks_pgs."""
        if all(args.get(k) is None for k in _PGS_ARGS):
            return None
        missing = [k for k in _PGS_ARGS if args.get(k) is None]
        if missing:
            raise ValueError("PGS references need %s" % ", ".join(_PGS_ARGS))
        start = np.ascontiguousarray(args["pgs_start"], dtype=np.float64)
        end = np.ascontiguousarray(args["pgs_end"], dtype=np.float64)
        off = np.ascontiguousarray(args["pgs_off"], dtype=np.int64)
        video = np.ascontiguousarray(args["pgs_video"], dtype=np.int64)
        P = len(off) - 1
        if len(video) != P:
            raise ValueError("pgs_video has %d entries for %d interval lists" % (len(video), P))
        if P and (np.any(np.diff(video) <= 0) or video[0] < 0 or video[-1] >= V):
            raise ValueError("pgs_video must be increasing video indices in [0, %d) (one interval list per video)" % V)
        if np.any(np.diff(off) < 0) or (P and (off[0] < 0 or off[-1] > min(len(start), len(end)))):
            raise ValueError("pgs_off must be non-decreasing and within the interval arrays")
        is_pgs = np.zeros(V, dtype=np.uint8)
        is_pgs[video] = 1
        lens = np.zeros(V, dtype=np.int64)
        lens[video] = np.diff(off)
        pick = np.concatenate([np.arange(off[i], off[i + 1]) for i in range(P)] + [np.zeros(0, np.int64)])
        pick = pick.astype(np.int64)
        return is_pgs, start[pick], end[pick], np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)

    def _subs_refs(self, V: int, streams: dict):
        """Each video's reference stream by the reference's rule, or None when no stream is given: returns
        (ref_is_subs u8[V], ref_cue_start, ref_cue_end, ref_cue_keep, ref_cue_off [V+1]) for b2_sync_tracks_subs."""
        unknown = set(streams) - set(_STREAM_ARGS)
        if unknown:
            raise TypeError("unexpected keyword arguments %s" % ", ".join(sorted(unknown)))
        given = sorted(k for k, v in streams.items() if v is not None)
        if given and not self.subs_then:
            raise ValueError("%s describe embedded subtitle streams; vad=%r does not read them (use vad='subs_then_%s')"
                             % (", ".join(given), self.vad, self.detector))
        if streams.get("ref_cue_off") is None or len(streams["ref_cue_off"]) <= 1:
            return None
        if streams.get("ref_cue_content") is not None and streams.get("ref_cue_keep") is not None:
            raise ValueError("pass ref_cue_content or ref_cue_keep, not both")
        return select_reference_streams(V, streams["ref_cue_start"], streams["ref_cue_end"], streams["ref_cue_off"],
                                        streams["ref_stream_video"], self.start_seconds,
                                        content=streams.get("ref_cue_content"), keep=streams.get("ref_cue_keep"))

    def _dispatch(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, gss: bool, pgs=None,
                  sig=None, seg=None, **kw):
        """The batched call of this synchroniser's detector with the search on or off: b2_sync_tracks_pgs with PGS
        references (pgs, from _pgs_refs), else b2_sync_tracks_subs with subtitle references (refs, from _subs_refs), else b2_sync_tracks_auditok for auditok, else
        b2_sync_tracks_gss / b2_sync_tracks; b2_sync_tracks_sig with signal references (sig, from _sig_refs, with
        any of the others).  pcm: int16 numpy array, CUDA tensor or None; kw: the outputs (device
        pointers) or want_all, and memspace.  Returns (best_score, best_offset, best_k, all_score, all_offset), plus
        (gss_ratio, gss_evals) with gss."""
        h = self.handle
        p = pcm if pcm is None or isinstance(pcm, np.ndarray) else pcm.data_ptr()
        cues = (cue_start, cue_end, cue_keep, cue_off, self.ratios, self.start_seconds, self.max_offset_samples)
        if seg is not None:   # b2_sync_tracks_seg, with any of the other references
            det = _native.B2_DETECTOR_AUDITOK if self.auditok else _native.B2_DETECTOR_ENERGY_ZCR
            other = {} if refs is None else dict(zip(("ref_is_subs", "ref_cue_start_s", "ref_cue_end_s",
                                                      "ref_cue_keep", "ref_cue_off"), refs))
            if pgs is not None:
                other.update(zip(("ref_is_pgs", "pgs_start_s", "pgs_end_s", "pgs_off"), pgs))
            if sig is not None:
                is_sig, x, voff = sig
                other.update(ref_is_sig=is_sig, x=x if isinstance(x, np.ndarray) else (x.data_ptr() if x.numel()
                                                                                       else None), sig_off=voff)
            return h.sync_tracks_seg(p, pcm_off, track_video, self.frame_rate, self.sample_rate,
                                     self.non_speech_label, *seg, *cues, detector=det,
                                     energy_threshold=self.energy_threshold, z_lo=self.z_lo, z_hi=self.z_hi,
                                     chunk_samples=self.chunk_samples, gss=gss, **other, **kw)
        if sig is not None:
            det = _native.B2_DETECTOR_AUDITOK if self.auditok else _native.B2_DETECTOR_ENERGY_ZCR
            is_sig, x, voff = sig
            other = {} if refs is None else dict(zip(("ref_is_subs", "ref_cue_start_s", "ref_cue_end_s",
                                                      "ref_cue_keep", "ref_cue_off"), refs))
            if pgs is not None:
                other.update(zip(("ref_is_pgs", "pgs_start_s", "pgs_end_s", "pgs_off"), pgs))
            xp = x if isinstance(x, np.ndarray) else (x.data_ptr() if x.numel() else None)
            return h.sync_tracks_sig(p, pcm_off, track_video, self.frame_rate, self.sample_rate,
                                     self.non_speech_label, is_sig, xp, voff, *cues, detector=det,
                                     energy_threshold=self.energy_threshold, z_lo=self.z_lo, z_hi=self.z_hi,
                                     chunk_samples=self.chunk_samples, gss=gss, **other, **kw)
        if pgs is not None:
            det = _native.B2_DETECTOR_AUDITOK if self.auditok else _native.B2_DETECTOR_ENERGY_ZCR
            text = {} if refs is None else dict(zip(("ref_is_subs", "ref_cue_start_s", "ref_cue_end_s", "ref_cue_keep",
                                                     "ref_cue_off"), refs))
            return h.sync_tracks_pgs(p, pcm_off, track_video, self.frame_rate, self.sample_rate,
                                     self.non_speech_label, *pgs, *cues, detector=det,
                                     energy_threshold=self.energy_threshold, z_lo=self.z_lo, z_hi=self.z_hi,
                                     chunk_samples=self.chunk_samples, gss=gss, **text, **kw)
        if refs is not None:
            det = _native.B2_DETECTOR_AUDITOK if self.auditok else _native.B2_DETECTOR_ENERGY_ZCR
            return h.sync_tracks_subs(p, pcm_off, track_video, self.frame_rate, self.sample_rate,
                                      self.non_speech_label, *refs, *cues, detector=det,
                                      energy_threshold=self.energy_threshold, z_lo=self.z_lo, z_hi=self.z_hi,
                                      chunk_samples=self.chunk_samples, gss=gss, **kw)
        if self.auditok:
            return h.sync_tracks_auditok(p, pcm_off, track_video, self.frame_rate, self.sample_rate,
                                         self.non_speech_label, *cues, self.chunk_samples, gss=gss, **kw)
        energy = (self.frame_rate, self.sample_rate, self.non_speech_label, self.energy_threshold, self.z_lo, self.z_hi)
        return (h.sync_tracks_gss if gss else h.sync_tracks)(p, pcm_off, track_video, *energy, *cues, **kw)

    def _sync_or_compose(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, pgs=None,
                         sig=None, seg=None, speech=None, **kw):
        """_dispatch with this synchroniser's search.  Outside the envelope of the device-driven search
        (B2_ERR_UNSUPPORTED) the search is composed of public steps instead (_gss_compose).  Returns
        (best_score, best_offset, best_k, all_score, all_offset), plus gss_ratio with the search; composed results
        are numpy arrays (all_* None unless want_all or device outputs were given).  speech (from _speech_request):
        the call writes the listed videos' reference signals into it; the composed search fills it from the
        reference signals it builds."""
        try:
            with self._speech_output(speech):
                return self._dispatch(pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, self.gss,
                                      pgs=pgs, sig=sig, seg=seg, **kw)[:6]
        except _native.NativeError as e:
            if not (self.gss and _is_unsupported(e)):
                raise
        want_all = kw.get("want_all", False) or kw.get("all_score") is not None
        bs, bo, bk, ratio, a_s, a_o = self._gss_compose(pcm, pcm_off, track_video, cue_start, cue_end, cue_off,
                                                        cue_keep, want_all=want_all, refs=refs, pgs=pgs, sig=sig,
                                                        seg=seg, speech=speech)
        return bs, bo, bk, a_s, a_o, ratio

    def use_torch_stream(self) -> None:
        """Launch on torch's current stream (so torch events / NCCL ops order against our kernels)."""
        import torch
        self.handle.set_stream(torch.cuda.current_stream().cuda_stream)

    def _reference_lengths(self, pcm_off, refs=None, pgs=None, sig=None, seg=None) -> np.ndarray:
        """Each video's reference length [V] in the batched calls, from the library's length helpers: the detector's
        windows over the chunk loop (b2_vad_num_windows, or auditok_out_off), a text stream's b2_rasterize_lengths at
        ratio 1.0, a PGS list's b2_rasterize_pgs_lengths, a signal's stored length and a segment video's b2_segment_length."""
        h = self.handle
        pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
        if self.auditok:
            lens = np.diff(h.auditok_out_off(pcm_off, self.frame_rate, self.sample_rate, self.chunk_samples))
        else:
            lens = np.array([h.lib.b2_vad_num_windows(int(n), self.frame_rate, self.sample_rate)
                             for n in np.diff(pcm_off)], dtype=np.int64)
        if refs is not None:
            is_subs, _, re_, _, roff = refs
            sub = h.rasterize_lengths(re_, roff, [1.0], 1, False, self.sample_rate)
            lens = np.where(is_subs != 0, sub, lens)
        if pgs is not None:
            is_pgs, _, pe, poff = pgs
            vids = np.flatnonzero(is_pgs)
            lens[vids] = h.rasterize_pgs_lengths(pe, np.concatenate([[0], np.cumsum(np.diff(poff)[vids])]),
                                                 self.sample_rate)
        if sig is not None:
            is_sig, _, voff = sig
            lens = np.where(is_sig != 0, np.diff(voff), lens)
        if seg is not None:
            for v, total in zip(seg[0], seg[1]):
                lens[v] = h.segment_length(total, self.sample_rate)
        return lens.astype(np.int64)

    def _speech_request(self, speech_video, pcm_off, refs=None, pgs=None, sig=None, seg=None, on_device=True,
                        device=None):
        """The speech output of a sync call with speech_video (None: no output): dict(video, off (the call writes
        it), buf (float64, CUDA tensor or numpy array, sized from _reference_lengths), total, memspace)."""
        if speech_video is None:
            return None
        V = len(pcm_off) - 1
        video = np.ascontiguousarray(speech_video, dtype=np.int64)
        if video.ndim != 1 or (len(video) and (np.any(np.diff(video) <= 0) or video[0] < 0 or video[-1] >= V)):
            raise ValueError("speech_video must be increasing video indices in [0, %d)" % V)
        lens = self._reference_lengths(pcm_off, refs, pgs, sig, seg)[video]
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        total = int(off[-1])
        if on_device:
            import torch
            buf = torch.empty(max(total, 1), dtype=torch.float64,
                              device=device if device is not None else torch.device("cuda", self.handle.device))
        else:
            buf = np.empty(max(total, 1), dtype=np.float64)
        return dict(video=video, off=np.empty(len(video) + 1, dtype=np.int64), want_off=off, buf=buf, total=total,
                    memspace=_native.B2_DEVICE if on_device else _native.B2_HOST)

    @contextlib.contextmanager
    def _speech_output(self, speech):
        """The handle's speech output set to the request `speech` (from _speech_request) while the block runs."""
        if speech is None:
            yield
            return
        buf = speech["buf"]
        self.handle.speech_output(buf.data_ptr() if hasattr(buf, "data_ptr") else buf, speech["total"],
                                  speech["video"], speech["off"], speech["memspace"])
        try:
            yield
        finally:
            self.handle.speech_output(None, 0, None, None)

    @staticmethod
    def _speech_result(speech):
        """(speech, speech_off) of a finished request: the written frames and offsets."""
        return speech["buf"][: speech["total"]], speech["off"]

    def sync_device(self, pcm, pcm_off, cue_start, cue_end, cue_off, cue_keep=None, out=None, all_out=None,
                    inputs_resident: bool = False, speech_video=None, **streams):
        """pcm: int16 CUDA tensor with all pairs back to back; pcm_off: [B+1] sample offsets (host).
        out: optional dict of preallocated CUDA tensors best_score f64[B], best_offset i32[B],
        best_k i32[B].  Returns that dict; nothing is synchronised.
        inputs_resident=True (B2_DEVICE_RESIDENT): the caller promises that nothing queued on the handle's
        stream before this call still writes ``pcm`` (a corpus that sits in HBM).  Back-to-back calls then
        overlap: the VAD of this batch starts while the last correlation chain of the previous batch is
        still running.  Results are identical; outputs stay ordered on the stream.
        With a ``subs_then_`` detector the embedded subtitle streams come as keyword arguments, and with any detector
        the PGS references and the serialized signals (see the class); with inputs_resident the promise covers
        ``sig`` too.
        speech_video: increasing video indices whose reference signals the call also writes (``--serialize-speech``):
        out then gains ``speech`` (float64 CUDA tensor, the signals back to back) and ``speech_off`` (int64 numpy
        array [P+1]); see b2_speech_output."""
        import torch
        B = len(pcm_off) - 1
        K = len(self.ratios)
        if (self.gss or self.auditok or self.subs_then
                or any(streams.get(k) is not None for k in _PGS_ARGS + _SIG_ARGS + _SEG_ARGS)):   # the identity track map: pair b is track b of video b
            return self.sync_device_tracks(pcm, pcm_off, np.arange(B, dtype=np.int32), cue_start, cue_end, cue_off,
                                           cue_keep, out=out, all_out=all_out, inputs_resident=inputs_resident,
                                           speech_video=speech_video, **streams)
        self._references(B, streams)   # rejects streams and unknown keywords
        dev = pcm.device
        if out is None:
            out = {"best_score": torch.empty(B, dtype=torch.float64, device=dev),
                   "best_offset": torch.empty(B, dtype=torch.int32, device=dev),
                   "best_k": torch.empty(B, dtype=torch.int32, device=dev)}
        a_s = all_out["score"].data_ptr() if all_out else None
        a_o = all_out["offset"].data_ptr() if all_out else None
        speech = self._speech_request(speech_video, pcm_off, device=dev)
        with self._speech_output(speech):
            self.handle.sync_batch(
                pcm.data_ptr(), pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label,
                self.energy_threshold, self.z_lo, self.z_hi, cue_start, cue_end, cue_keep, cue_off, self.ratios,
                self.start_seconds, self.max_offset_samples, out["best_score"].data_ptr(),
                out["best_offset"].data_ptr(), out["best_k"].data_ptr(), a_s, a_o,
                memspace=_native.B2_DEVICE_RESIDENT if inputs_resident else _native.B2_DEVICE)
        if speech is not None:
            out["speech"], out["speech_off"] = self._speech_result(speech)
        assert K == len(self.ratios)
        return out

    def sync_device_tracks(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep=None, out=None,
                           all_out=None, inputs_resident: bool = False, speech_video=None, **streams):
        """sync_device for several subtitle tracks per video (``ffs movie.mkv -i en.srt de.srt ...``):
        pcm holds the V videos back to back, pcm_off: [V+1] sample offsets (host); track t (cue list
        cue_off[t] .. cue_off[t+1]) is synced against video track_video[t] (host, non-decreasing).  Each
        video's PCM is read and run through the VAD once, however many tracks it has.  out: optional dict
        of CUDA tensors best_score f64[T], best_offset i32[T], best_k i32[T]; all_out: optional
        {"score": f64[T*K], "offset": i32[T*K]}.  Returns out; nothing is synchronised.  inputs_resident
        as for sync_device (resident calls of both methods chain with each other).
        With the golden-section search (a trailing None in ratios) out also holds gss_ratio f64[T] and all_out
        is {"score": f64[T*(K+1)], "offset": i32[T*(K+1)]} with column K the search's candidate.
        streams: the embedded subtitle streams of a ``subs_then_`` detector (ref_cue_start, ... - see the class) and
        the PGS references (pgs_start, pgs_end, pgs_off, pgs_video) and the serialized signals (sig, sig_off,
        sig_video; a float64 CUDA tensor keeps the call asynchronous, other inputs are converted first).
        speech_video as for sync_device (out gains speech and speech_off); with no tracks the call runs only the
        detector step of those videos (the reference's serialize-only run)."""
        import torch
        T = len(track_video)
        sig_in = streams.get("sig")
        refs, pgs, sig, seg = self._all_refs(len(pcm_off) - 1, streams, on_device=True)
        dev = pcm.device if pcm is not None else torch.device("cuda", self.handle.device)
        speech = self._speech_request(speech_video, pcm_off, refs, pgs, sig, seg, device=dev)
        if out is None:
            out = {"best_score": torch.empty(T, dtype=torch.float64, device=dev),
                   "best_offset": torch.empty(T, dtype=torch.int32, device=dev),
                   "best_k": torch.empty(T, dtype=torch.int32, device=dev)}
        if self.gss and "gss_ratio" not in out:
            out["gss_ratio"] = torch.empty(T, dtype=torch.float64, device=dev)
        memspace = _native.B2_DEVICE_RESIDENT if inputs_resident else _native.B2_DEVICE
        keys = ("best_score", "best_offset", "best_k") + (("gss_ratio",) if self.gss else ())
        ptrs = {k: out[k].data_ptr() for k in keys}
        if all_out:
            ptrs.update(all_score=all_out["score"].data_ptr(), all_offset=all_out["offset"].data_ptr())
        if sig is not None and sig[1] is not sig_in:
            # a converted copy: ready before the handle's stream reads it, and kept until the call is done
            torch.cuda.current_stream(sig[1].device).synchronize()
        res = self._sync_or_compose(pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, pgs=pgs,
                                    sig=sig, seg=seg, speech=speech, memspace=memspace, **ptrs)
        if sig is not None and sig[1] is not sig_in:
            self.handle.synchronize()
        if isinstance(res[0], np.ndarray):   # composed on the host
            for k, v in zip(keys, res[:3] + res[5:]):
                out[k].copy_(torch.from_numpy(v))
            if all_out:
                all_out["score"].copy_(torch.from_numpy(res[3]))
                all_out["offset"].copy_(torch.from_numpy(res[4]))
        if speech is not None:
            out["speech"], out["speech_off"] = self._speech_result(speech)
        return out

    def sync_host_tracks(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep=None,
                         want_all=False, speech_video=None, **streams):
        """sync_device_tracks with host buffers (pcm: int16 numpy array of the V videos).  Blocks until
        results are on the host.  Returns (best_score, best_offset, best_k[, all_score, all_offset]) per
        track, and gss_ratio last with the golden-section search.  streams as for sync_device_tracks.
        speech_video as for sync_device_tracks: the tuple then ends with (speech float64 numpy array, speech_off)."""
        refs, pgs, sig, seg = self._all_refs(len(pcm_off) - 1, streams, on_device=False)
        speech = self._speech_request(speech_video, pcm_off, refs, pgs, sig, seg, on_device=False)
        res = self._sync_or_compose(pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, pgs=pgs,
                                    sig=sig, seg=seg, speech=speech, want_all=want_all, memspace=_native.B2_HOST)
        self._raise_bad_signals(sig, res[2])
        self._raise_no_speech(seg, res[2], track_video)
        res = res if want_all else res[:3] + res[5:]
        return res if speech is None else res + self._speech_result(speech)

    def sync_signals(self, ref, ref_off, cue_start, cue_end, cue_off, cue_keep=None, speech_video=None):
        """Same as sync_device but starting from reference speech SIGNALS (100 Hz float32, all pairs
        back to back; numpy array or CUDA tensor) instead of PCM - the replay path of the
        reference's test-case bundles: ``ref.npz{"speech"}`` + ``in.srt``
        (ffsubsync/ffsubsync.py:338-343,639-644; DeserializeSpeechTransformer).
        Returns (best_score f64[B], best_offset i32[B], best_k i32[B]) as numpy arrays, and gss_ratio f64[B]
        last with the golden-section search (gss_batch.gss_align_batch on the same signals, merged as
        candidate K by gss_batch.combine_gss).  speech_video is refused: the signals are the caller's already."""
        import torch
        if speech_video is not None:
            raise ValueError("sync_signals starts from the reference signals; it does not write them (speech_video)")
        h = self.handle
        ref_off = np.ascontiguousarray(ref_off, dtype=np.int64)
        B, K = len(ref_off) - 1, len(self.ratios)
        if isinstance(ref, np.ndarray):
            ref = torch.from_numpy(np.ascontiguousarray(ref, dtype=np.float32)).cuda()
        dev = ref.device
        lengths = h.rasterize_lengths(cue_end, cue_off, self.ratios, K, False, self.sample_rate)
        sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
        h.rasterize(cue_start, cue_end, cue_keep, cue_off, self.ratios, K, False, self.sample_rate,
                    self.start_seconds, out=sub.data_ptr(), out_off=sub_off, memspace=_native.B2_DEVICE)
        score = torch.empty(B * K, dtype=torch.float64, device=dev)
        offset = torch.empty(B * K, dtype=torch.int32, device=dev)
        status = torch.empty(B * K, dtype=torch.int32, device=dev)
        h.align_batch(ref.data_ptr(), ref_off, sub.data_ptr(), sub_off, B, K, self.max_offset_samples,
                      score=score.data_ptr(), offset=offset.data_ptr(), status=status.data_ptr(),
                      memspace=_native.B2_DEVICE)
        bs = torch.empty(B, dtype=torch.float64, device=dev)
        bo = torch.empty(B, dtype=torch.int32, device=dev)
        bk = torch.empty(B, dtype=torch.int32, device=dev)
        h.reduce_ratios(score.data_ptr(), offset.data_ptr(), status.data_ptr(), B, K, self.max_offset_samples,
                        best_score=bs.data_ptr(), best_offset=bo.data_ptr(), best_k=bk.data_ptr(),
                        memspace=_native.B2_DEVICE)
        h.synchronize()
        if not self.gss:
            return bs.cpu().numpy(), bo.cpu().numpy(), bk.cpu().numpy()
        from .gss_batch import combine_gss, gss_align_batch
        g = gss_align_batch(ref, ref_off, cue_start, cue_end, cue_off, cue_keep, self.max_offset_samples,
                            self.sample_rate, self.start_seconds, handle=h)
        bs, bo, bk, ratio, _, _ = combine_gss(bs.cpu().numpy(), bo.cpu().numpy(), bk.cpu().numpy(), g, K,
                                              self.max_offset_samples)
        return bs, bo, bk, ratio

    def sync_device_candidate_sharded(self, pcm, pcm_off, cue_start, cue_end, cue_off, cue_keep=None,
                                      rank: int = 0, world: int = 1, group=None, speech_video=None, **pgs_args):
        """Secondary multi-GPU mode (SURVEY.md section 8e, "B < G": a few pairs on many GPUs): the K
        ratio candidates of every pair are dealt round-robin over the ranks.  Every rank runs the
        VAD of the (replicated) reference PCM - 33 us per 2 h signal, cheaper than shipping the
        signal - rasterises and aligns only ITS candidates (b2_align_batch with K_local ratios),
        the per-candidate (score, offset, status) triples are all-gathered back into list order
        (NCCL, 24 B per candidate) and b2_reduce_ratios applies the |offset| filter and the
        first-in-list tie rule on every rank, so all ranks hold the same (score, offset, ratio index)
        as a single-GPU run.  pcm: int16 CUDA tensor, same on every rank.  Returns CUDA tensors
        (best_score f64[B], best_offset i32[B], best_k i32[B]).  Not available with the golden-section search:
        its 17 evaluations are sequential per pair, so they cannot be dealt over ranks like grid candidates."""
        import torch
        from . import distributed
        if speech_video is not None:
            raise ValueError("sync_device_candidate_sharded does not write reference signals (speech_video); a "
                             "multi-GPU run writes each rank's own videos with sync_device")
        if self.gss:
            raise ValueError("sync_device_candidate_sharded shards the ratio grid; it does not run the "
                             "golden-section search (None in ratios)")
        if self.subs_then:
            raise ValueError("sync_device_candidate_sharded runs the detector on every video; it does not take "
                             "embedded subtitle references (vad=%r)" % self.vad)
        unknown = set(pgs_args) - set(_PGS_ARGS + _SIG_ARGS + _SEG_ARGS)
        if unknown:
            raise TypeError("unexpected keyword arguments %s" % ", ".join(sorted(unknown)))
        given_seg = sorted(k for k in _SEG_ARGS if pgs_args.pop(k, None) is not None)
        if given_seg:
            raise ValueError("sync_device_candidate_sharded runs the detector on every video's whole audio; it does "
                             "not take sampled segment references (%s)" % ", ".join(given_seg))
        given_sig = sorted(k for k in _SIG_ARGS if pgs_args.get(k) is not None)
        if given_sig:
            raise ValueError("sync_device_candidate_sharded runs the detector on every video; it does not take "
                             "serialized signal references (%s)" % ", ".join(given_sig))
        if any(v is not None for v in pgs_args.values()):
            raise ValueError("sync_device_candidate_sharded runs the detector on every video; it does not take "
                             "PGS references (%s)" % ", ".join(sorted(pgs_args)))
        h = self.handle
        self.use_torch_stream()   # torch ops and NCCL below are ordered against our kernels by the stream
        pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
        B, K = len(pcm_off) - 1, len(self.ratios)
        dev = pcm.device
        mine = distributed.shard_candidates(K, rank, world)
        if self.auditok:   # b2_vad_auditok's float64 signal, rounded once to float32
            ref, ref_off = self._vad_auditok_device(pcm, pcm_off)
        else:   # over the chunk loop's detector calls, as the batched calls run it
            calls, first = h.energy_calls(pcm_off, self.frame_rate, self.sample_rate)
            fpw = h.frames_per_window(self.frame_rate, self.sample_rate)
            call_out = np.concatenate([[0], np.cumsum((np.diff(calls) + fpw - 1) // fpw)]).astype(np.int64)
            ref_off = call_out[first]
            ref = torch.empty(int(ref_off[-1]), dtype=torch.float32, device=dev)
            h.vad_energy_zcr(pcm.data_ptr(), calls, self.frame_rate, self.sample_rate, self.non_speech_label,
                             self.energy_threshold, self.z_lo, self.z_hi, out=ref.data_ptr(),
                             memspace=_native.B2_DEVICE)
        k_loc = len(mine)
        local = torch.zeros((B, max(k_loc, 1), 3), dtype=torch.float64, device=dev)
        if k_loc:
            my_ratios = self.ratios[mine]
            lengths = h.rasterize_lengths(cue_end, cue_off, my_ratios, k_loc, False, self.sample_rate)
            sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
            sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
            h.rasterize(cue_start, cue_end, cue_keep, cue_off, my_ratios, k_loc, False, self.sample_rate,
                        self.start_seconds, out=sub.data_ptr(), out_off=sub_off, memspace=_native.B2_DEVICE)
            score = torch.empty(B * k_loc, dtype=torch.float64, device=dev)
            offset = torch.empty(B * k_loc, dtype=torch.int32, device=dev)
            status = torch.empty(B * k_loc, dtype=torch.int32, device=dev)
            h.align_batch(ref.data_ptr(), ref_off, sub.data_ptr(), sub_off, B, k_loc, self.max_offset_samples,
                          score=score.data_ptr(), offset=offset.data_ptr(), status=status.data_ptr(),
                          memspace=_native.B2_DEVICE)
            local[:, :, 0] = score.view(B, k_loc)
            local[:, :, 1] = offset.view(B, k_loc).to(torch.float64)
            local[:, :, 2] = status.view(B, k_loc).to(torch.float64)
        full = distributed.allgather_candidate_results(local[:, :k_loc], K, rank, world, group=group)
        score_all = full[:, :, 0].contiguous().view(-1)
        offset_all = full[:, :, 1].to(torch.int32).contiguous().view(-1)
        status_all = full[:, :, 2].to(torch.int32).contiguous().view(-1)
        bs = torch.empty(B, dtype=torch.float64, device=dev)
        bo = torch.empty(B, dtype=torch.int32, device=dev)
        bk = torch.empty(B, dtype=torch.int32, device=dev)
        h.reduce_ratios(score_all.data_ptr(), offset_all.data_ptr(), status_all.data_ptr(), B, K,
                        self.max_offset_samples, best_score=bs.data_ptr(), best_offset=bo.data_ptr(),
                        best_k=bk.data_ptr(), memspace=_native.B2_DEVICE)
        return bs, bo, bk

    def sync_host(self, pcm, pcm_off, cue_start, cue_end, cue_off, cue_keep=None, want_all=False, speech_video=None,
                  **streams):
        """pcm: int16 numpy array (ideally backed by pinned memory).  Blocks until results are on
        the host.  Returns (best_score, best_offset, best_k[, all_score, all_offset]), and gss_ratio last
        with the golden-section search.  With a ``subs_then_`` detector the embedded subtitle streams come as
        keyword arguments, and with any detector the PGS references and the serialized signals (see the class).
        speech_video as for sync_host_tracks."""
        if (self.gss or self.auditok or self.subs_then
                or any(streams.get(k) is not None for k in _PGS_ARGS + _SIG_ARGS + _SEG_ARGS)):
            return self.sync_host_tracks(pcm, pcm_off, np.arange(len(pcm_off) - 1, dtype=np.int32), cue_start,
                                         cue_end, cue_off, cue_keep, want_all=want_all, speech_video=speech_video,
                                         **streams)
        self._references(len(pcm_off) - 1, streams)   # rejects streams and unknown keywords
        speech = self._speech_request(speech_video, pcm_off, on_device=False)
        with self._speech_output(speech):
            res = self.handle.sync_batch(
                pcm, pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label, self.energy_threshold,
                self.z_lo, self.z_hi, cue_start, cue_end, cue_keep, cue_off, self.ratios, self.start_seconds,
                self.max_offset_samples, want_all=want_all, memspace=_native.B2_HOST)
        res = res if want_all else res[:3]
        return res if speech is None else res + self._speech_result(speech)

    def _apply_sync_args(self, apply_offset_seconds, skip_sync_on_low_quality, min_score, quality_max_offset_seconds,
                         max_framerate_deviation, suppress_output_if_offset_less_than) -> dict:
        return dict(sample_rate=self.sample_rate, apply_offset_seconds=apply_offset_seconds,
                    gate=skip_sync_on_low_quality, min_score=min_score,
                    quality_max_offset_seconds=quality_max_offset_seconds,
                    max_framerate_deviation=max_framerate_deviation, suppress=suppress_output_if_offset_less_than)

    def apply_sync(self, out, cue_start, cue_end, cue_off, *, apply_offset_seconds: float = DEFAULT_APPLY_OFFSET_SECONDS,
                   skip_sync_on_low_quality: bool = False, min_score: float = DEFAULT_MIN_SCORE,
                   quality_max_offset_seconds: float = DEFAULT_QUALITY_MAX_OFFSET_SECONDS,
                   max_framerate_deviation: float = DEFAULT_MAX_FRAMERATE_DEVIATION,
                   suppress_output_if_offset_less_than: Optional[float] = None) -> dict:
        """try_sync's output step (ffsubsync/ffsubsync.py:236-299) over the results of a device sync call: ``out`` is
        the dict sync_device / sync_device_tracks returned (gss_ratio included with the search), cue_start /
        cue_end / cue_off the same host cue lists that call took.  Enqueues one kernel on the handle's stream behind
        that call, without synchronising, and keeps a chain of resident calls intact.  Returns CUDA tensors:
        ``synced_start_us`` / ``synced_end_us`` int64 per cue (microseconds, as the reference writes them:
        scaled and shifted, or the originals for a gated or failed track), ``offset_seconds`` / ``scale`` f64 per
        track (NaN when the alignment failed) and ``status`` i32 per track (sync_output's bits).  The keywords are
        the reference's options of the same names (``--apply-offset-seconds``, ``--skip-sync-on-low-quality``, ...)."""
        import torch
        dev = out["best_score"].device
        n, T = int(np.asarray(cue_off)[-1]), len(cue_off) - 1
        res = {"synced_start_us": torch.empty(n, dtype=torch.int64, device=dev),
               "synced_end_us": torch.empty(n, dtype=torch.int64, device=dev),
               "offset_seconds": torch.empty(T, dtype=torch.float64, device=dev),
               "scale": torch.empty(T, dtype=torch.float64, device=dev),
               "status": torch.empty(T, dtype=torch.int32, device=dev)}
        gss = out["gss_ratio"].data_ptr() if self.gss else None
        self.handle.apply_sync(
            out["best_score"].data_ptr(), out["best_offset"].data_ptr(), out["best_k"].data_ptr(), gss, cue_start,
            cue_end, cue_off, self.ratios,
            outs=[t.data_ptr() for t in res.values()], memspace=_native.B2_DEVICE,
            **self._apply_sync_args(apply_offset_seconds, skip_sync_on_low_quality, min_score,
                                    quality_max_offset_seconds, max_framerate_deviation,
                                    suppress_output_if_offset_less_than))
        return res

    def apply_sync_host(self, res, cue_start, cue_end, cue_off, *,
                        apply_offset_seconds: float = DEFAULT_APPLY_OFFSET_SECONDS,
                        skip_sync_on_low_quality: bool = False, min_score: float = DEFAULT_MIN_SCORE,
                        quality_max_offset_seconds: float = DEFAULT_QUALITY_MAX_OFFSET_SECONDS,
                        max_framerate_deviation: float = DEFAULT_MAX_FRAMERATE_DEVIATION,
                        suppress_output_if_offset_less_than: Optional[float] = None) -> dict:
        """apply_sync over the numpy results of a host sync call: ``res`` is the tuple sync_host /
        sync_host_tracks returned (best_score, best_offset, best_k first, gss_ratio last with the search).  Blocks;
        returns the same keys as apply_sync as numpy arrays."""
        gss = res[-1] if self.gss else None
        outs = self.handle.apply_sync(
            res[0], res[1], res[2], gss, cue_start, cue_end, cue_off, self.ratios, memspace=_native.B2_HOST,
            **self._apply_sync_args(apply_offset_seconds, skip_sync_on_low_quality, min_score,
                                    quality_max_offset_seconds, max_framerate_deviation,
                                    suppress_output_if_offset_less_than))
        return dict(zip(("synced_start_us", "synced_end_us", "offset_seconds", "scale", "status"), outs))

    # -- per-segment offsets with a split penalty (b2_split_tracks, b2_apply_split) ---------------------------------
    def split_ratios(self, best_k, gss_ratio=None) -> np.ndarray:
        """Each track's ratio from a sync call's best_k (host arrays): ratios[best_k], gss_ratio for best_k == K with
        the search, NaN (skipped) for a track without an alignment."""
        best_k = np.asarray(best_k, dtype=np.int64)
        K = len(self.ratios)
        r = np.full(len(best_k), np.nan)
        grid = (best_k >= 0) & (best_k < K)
        r[grid] = self.ratios[best_k[grid]]
        if self.gss and gss_ratio is not None:
            g = best_k == K
            r[g] = np.asarray(gss_ratio, dtype=np.float64)[g]
        return r

    @staticmethod
    def _split_refs(speech_off, track_video, speech_video):
        """The tracks' indices into the written signals: speech_video lists the videos the sync call wrote (None: video
        i is signal i).  ValueError for a track whose video has no signal."""
        track_video = np.asarray(track_video, dtype=np.int64)
        P = len(speech_off) - 1
        listed = np.arange(P) if speech_video is None else np.asarray(speech_video, dtype=np.int64)
        pos = {int(v): i for i, v in enumerate(listed)}
        missing = sorted({int(v) for v in track_video if int(v) not in pos})
        if missing:
            raise ValueError("split needs the reference signals of videos %s: call the sync with speech_video covering "
                             "them" % missing)
        return np.array([pos[int(v)] for v in track_video], dtype=np.int32)

    @staticmethod
    def _split_direction(max_segments, split_direction):
        """Refuses a split_direction other than None, +1 and -1, and one combined with max_segments (at most N
        segments in direction d are split_breaks=(d,) * (N - 1))."""
        if split_direction is None:
            return
        if isinstance(split_direction, bool) or split_direction not in (1, -1):
            raise ValueError("split_direction must be None, +1 (offsets only grow) or -1 (only shrink), not %r"
                             % (split_direction,))
        if max_segments is not None:
            raise ValueError("split_direction and max_segments cannot be combined")

    @staticmethod
    def _split_breaks(max_segments, split_direction, split_breaks):
        """split_breaks as a tuple of +-1 ints (None stays None).  Refuses an empty sequence, bools, entries other than
        +1 and -1, and split_breaks combined with max_segments or split_direction."""
        if split_breaks is None:
            return None
        if isinstance(split_breaks, (str, bytes)) or not hasattr(split_breaks, "__len__"):
            raise ValueError("split_breaks must be a sequence of +1 / -1, not %r" % (split_breaks,))
        out = []
        for d in split_breaks:
            if isinstance(d, (bool, np.bool_)) or not isinstance(d, (int, np.integer)) or d not in (1, -1):
                raise ValueError("split_breaks entries must be +1 (the offset grows) or -1 (it shrinks), not %r"
                                 % (d,))
            out.append(int(d))
        if not out:
            raise ValueError("split_breaks must state at least one break")
        if max_segments is not None or split_direction is not None:
            raise ValueError("split_breaks cannot be combined with max_segments or split_direction")
        return tuple(out)

    def _split_window(self, split_max_offset_seconds, max_segments=None, split_direction=None, split_breaks=None):
        """(Handle method, max_offset_samples, arguments after split_penalty) of a split: None keeps the sync window
        and b2_split_tracks; seconds convert as max_offset_seconds does and go through b2_split_tracks_wide.  An integer
        max_segments goes through b2_split_tracks_capped at either window, a split_direction of +-1 through
        b2_split_tracks_directed, a split_breaks tuple through b2_split_tracks_breaks."""
        mos = self.max_offset_samples if split_max_offset_seconds is None else \
            abs(int(split_max_offset_seconds * self.sample_rate))
        if split_breaks is not None:
            return self.handle.split_tracks_breaks, mos, (split_breaks,)
        if max_segments is not None:
            return self.handle.split_tracks_capped, mos, (int(max_segments),)
        if split_direction is not None:
            return self.handle.split_tracks_directed, mos, (int(split_direction),)
        if split_max_offset_seconds is None:
            return self.handle.split_tracks, mos, ()
        return self.handle.split_tracks_wide, mos, ()

    def split_tracks(self, out, track_video, cue_start, cue_end, cue_off, cue_keep=None, *, split_penalty: float,
                     speech_video=None, split_max_offset_seconds=None, max_segments=None,
                     split_direction=None, split_breaks=None) -> dict:
        """Per-segment offsets (b2_split_tracks) over the results of a device sync call made with ``speech_video``
        (``out`` carries ``speech`` / ``speech_off``; pass the same speech_video here, None when it listed videos
        0 .. P-1): each track's cue runs are cut into segments with their own offsets, a change of offset costing
        ``split_penalty`` (+inf: one offset per track, the sync call's).  The tracks, cues and ratio are the sync
        call's (ratio from best_k / gss_ratio).  Waits for the sync call to read best_k (and gss_ratio) back into the ratio
        list, then enqueues the split on the handle's stream without synchronising.  Returns CUDA tensors ``cue_offset`` i32 per cue,
        ``n_segments`` i32 and ``split_score`` f64 per track, and the host ``ratio`` (NaN: skipped track).
        Departures a caller should know: the wait for best_k above (b2_split_tracks takes the ratios as host metadata,
        so that a bad ratio is refused before anything runs); a video whose reference has a third level is not an
        error here (the device call cannot stop after its level scan without a synchronisation) but gives its tracks
        ``n_segments == -1``, NaN and offsets 0, which apply_split marks FAILED - split_tracks_host raises instead; and a
        track with more than 16 384 kept cues is refused even when its cues make fewer runs (each run holds one).
        ``split_max_offset_seconds`` (None: the synchroniser's own max_offset_seconds) sets the window the segments'
        offsets are searched in, up to about +-1 310 s at 100 Hz (b2_split_tracks_wide).  Every segment offset is
        absolute and all segments share the window, so it must cover the sync offset plus the breaks before the last
        segment: after a 5 min ad break the later cues need the sync offset plus 300 s.
        ``max_segments`` (None: no cap, the calls above) caps each track at that many segments (b2_split_tracks_capped,
        1 .. 16, at most 8 at +-150 s on an H100) and adds ``split_profile``, a (T, max_segments) f64 tensor: column k
        is the track's best penalised objective with at most k + 1 segments (NaN for a track n_segments <= 0 marks).
        ``split_direction`` (None: either way, the calls above) makes the offsets move one way only along the track
        (b2_split_tracks_directed, at either window; same results): +1 when the video has breaks the subtitles lack
        (ad breaks, an intermission: every break moves the later cues later), -1 when the subtitles have content the
        video lacks (a cut release, a recap pruned from the video: later cues move earlier).  It cannot be combined
        with ``max_segments`` (ValueError, as for any value other than None, +1 and -1); ``split_breaks`` says both.
        ``split_breaks`` (None: the calls above) states the breaks a user knows of, in track order: a sequence of 1 to
        15 entries of +1 / -1, e.g. ``(-1,)`` for one cut or ``(1, 1, 1)`` for up to three ad breaks
        (b2_split_tracks_breaks, at either window).  A track gets at most that many breaks, its i-th break moving the
        offset the i-th way, and the result gains ``split_profile``, a (T, len(split_breaks) + 1) f64 tensor: column m
        is the track's best penalised objective with exactly m breaks (-inf when none fits, NaN for a track
        n_segments <= 0 marks).  ValueError for an empty sequence, bools, other entries, and with ``max_segments`` or
        ``split_direction``."""
        import torch
        self._split_direction(max_segments, split_direction)
        split_breaks = self._split_breaks(max_segments, split_direction, split_breaks)
        if "speech" not in out:
            raise ValueError("split_tracks needs the sync call's reference signals: call it with speech_video")
        idx = self._split_refs(out["speech_off"], track_video, speech_video)
        self.handle.synchronize()   # best_k is written on the handle's stream, which need not be torch's
        ratio = self.split_ratios(out["best_k"].cpu().numpy(),
                                  out["gss_ratio"].cpu().numpy() if self.gss else None)
        dev = out["speech"].device
        n, T = int(np.asarray(cue_off)[-1]), len(cue_off) - 1
        res = {"cue_offset": torch.empty(max(n, 1), dtype=torch.int32, device=dev),
               "n_segments": torch.empty(max(T, 1), dtype=torch.int32, device=dev),
               "split_score": torch.empty(max(T, 1), dtype=torch.float64, device=dev)}
        if max_segments is not None:
            res["split_profile"] = torch.empty((max(T, 1), max(int(max_segments), 1)), dtype=torch.float64, device=dev)
        if split_breaks is not None:
            res["split_profile"] = torch.empty((max(T, 1), len(split_breaks) + 1), dtype=torch.float64, device=dev)
        split, mos, cap = self._split_window(split_max_offset_seconds, max_segments, split_direction, split_breaks)
        split(out["speech"].data_ptr(), True, out["speech_off"], idx, cue_start, cue_end, cue_keep, cue_off, ratio,
              self.sample_rate, self.start_seconds, mos, split_penalty, *cap,
              outs=[t.data_ptr() for t in res.values()], memspace=_native.B2_DEVICE)
        res = {"cue_offset": res["cue_offset"][:n], "n_segments": res["n_segments"][:T],
               "split_score": res["split_score"][:T], "ratio": ratio,
               **({} if "split_profile" not in res else {"split_profile": res["split_profile"][:T]})}
        return res

    def split_tracks_host(self, res, track_video, cue_start, cue_end, cue_off, cue_keep=None, *, split_penalty: float,
                          speech_video=None, split_max_offset_seconds=None, max_segments=None,
                          split_direction=None, split_breaks=None) -> dict:
        """split_tracks over the tuple of a host sync call made with speech_video (best_score, best_offset, best_k
        first, gss_ratio before the trailing (speech, speech_off) with the search).  Blocks; numpy results.  A reference
        with a third level raises (NativeError, B2_ERR_UNSUPPORTED, naming the video and frame); more than 16 384 kept
        cues in a track too.  ``split_max_offset_seconds`` as for split_tracks: an absolute window shared by all
        segments, which must cover the sync offset plus the breaks before the last segment.  ``max_segments`` as for
        split_tracks: the result gains ``split_profile``, a (T, max_segments) numpy array.  ``split_direction`` as for
        split_tracks: +1 for ad breaks or an intermission in the video, -1 for a cut video or a pruned recap.
        ``split_breaks`` as for split_tracks: the result gains ``split_profile``, a (T, len(split_breaks) + 1) numpy
        array."""
        self._split_direction(max_segments, split_direction)
        split_breaks = self._split_breaks(max_segments, split_direction, split_breaks)
        speech, speech_off = res[-2], res[-1]
        idx = self._split_refs(speech_off, track_video, speech_video)
        ratio = self.split_ratios(res[2], res[-3] if self.gss else None)
        split, mos, cap = self._split_window(split_max_offset_seconds, max_segments, split_direction, split_breaks)
        outs = split(speech, True, speech_off, idx, cue_start, cue_end, cue_keep, cue_off, ratio, self.sample_rate,
                     self.start_seconds, mos, split_penalty, *cap, memspace=_native.B2_HOST)
        return dict(zip(("cue_offset", "n_segments", "split_score", "split_profile"), outs), ratio=ratio)

    def apply_split(self, split, cue_start, cue_end, cue_off, *,
                    apply_offset_seconds: float = DEFAULT_APPLY_OFFSET_SECONDS) -> dict:
        """try_sync's output step with each cue's own offset (b2_apply_split) over the dict split_tracks returned.
        Enqueues one kernel without synchronising; returns CUDA tensors ``synced_start_us`` / ``synced_end_us`` int64
        per cue and ``status`` i32 per track (WRITTEN | APPLIED, or FAILED for a skipped track)."""
        import torch
        dev = split["n_segments"].device
        n, T = int(np.asarray(cue_off)[-1]), len(cue_off) - 1
        res = {"synced_start_us": torch.empty(max(n, 1), dtype=torch.int64, device=dev),
               "synced_end_us": torch.empty(max(n, 1), dtype=torch.int64, device=dev),
               "status": torch.empty(max(T, 1), dtype=torch.int32, device=dev)}
        self.handle.apply_split(split["ratio"], split["n_segments"].data_ptr(), split["cue_offset"].data_ptr(),
                                cue_start, cue_end, cue_off, self.sample_rate, apply_offset_seconds,
                                outs=[t.data_ptr() for t in res.values()], memspace=_native.B2_DEVICE)
        return {"synced_start_us": res["synced_start_us"][:n], "synced_end_us": res["synced_end_us"][:n],
                "status": res["status"][:T]}

    def apply_split_host(self, split, cue_start, cue_end, cue_off, *,
                         apply_offset_seconds: float = DEFAULT_APPLY_OFFSET_SECONDS) -> dict:
        """apply_split over the numpy dict split_tracks_host returned.  Blocks; numpy results."""
        outs = self.handle.apply_split(split["ratio"], split["n_segments"], split["cue_offset"], cue_start, cue_end,
                                       cue_off, self.sample_rate, apply_offset_seconds, memspace=_native.B2_HOST)
        return dict(zip(("synced_start_us", "synced_end_us", "status"), outs))

    def _gss_compose(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep=None, want_all=False,
                     refs=None, pgs=None, sig=None, seg=None, speech=None):
        """The golden-section search outside the envelope of the device-driven search, composed of public steps:
        the grid (this synchroniser's batched call with the search off), gss_align_batch on each track's reference
        signal (_reference_signals, with subtitle references refs from _subs_refs) and the reference's combine.
        pcm: int16 numpy array or CUDA tensor (or None without audio).  Returns numpy arrays (best_score,
        best_offset, best_k, gss_ratio, all_score, all_offset) (all_* None unless want_all).  With signal references
        (sig, from _sig_refs) the tracks of a video with an out-of-domain value get the batched calls' sentinel."""
        import torch
        from .gss_batch import combine_gss, gss_align_batch
        h = self.handle
        pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
        track_video = np.ascontiguousarray(track_video, dtype=np.int32)
        K = len(self.ratios)
        on_device = pcm is not None and not isinstance(pcm, np.ndarray)
        if on_device:
            h.synchronize()
            torch.cuda.synchronize(pcm.device)
            pcm_host = pcm.cpu().numpy()
        else:
            pcm_host = pcm
        if sig is not None and not isinstance(sig[1], np.ndarray):
            h.synchronize()
            torch.cuda.synchronize(sig[1].device)
            sig = (sig[0], sig[1].cpu().numpy(), sig[2])
        grid = self._dispatch(pcm_host, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, False,
                              pgs=pgs, sig=sig, seg=seg, want_all=True, memspace=_native.B2_HOST)
        ref, ref_off = self._reference_signals(pcm_host, pcm_off, refs, pgs, sig, seg)
        if speech is not None:   # the listed videos' reference signals, widened
            parts = [ref[ref_off[v]: ref_off[v + 1]] for v in speech["video"]]
            x = np.concatenate(parts + [np.zeros(0, np.float32)]).astype(np.float64)
            speech["off"][:] = np.concatenate([[0], np.cumsum([len(p) for p in parts])])
            if isinstance(speech["buf"], np.ndarray):
                speech["buf"][: len(x)] = x
            else:
                import torch
                speech["buf"][: len(x)].copy_(torch.from_numpy(x))
        # one copy of its video's reference signal per track
        parts = [ref[ref_off[v]: ref_off[v + 1]] for v in track_video]
        t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        t_ref = np.concatenate(parts).astype(np.float32) if parts else np.zeros(0, np.float32)
        g = gss_align_batch(t_ref, t_off, cue_start, cue_end, cue_off, cue_keep, self.max_offset_samples,
                            self.sample_rate, self.start_seconds, handle=h)
        bs, bo, bk, ratio, a_s, a_o = combine_gss(grid[0], grid[1], grid[2], g, K, self.max_offset_samples,
                                                  grid[3], grid[4])
        marked = []
        if sig is not None:
            marked.append((list(self._bad_signals(sig)), _native.B2_BEST_K_BAD_SIGNAL))
        if seg is not None:
            marked.append((self._no_speech_videos(seg, grid[2], track_video), _native.B2_BEST_K_NO_SPEECH))
        for vids, sentinel in marked:
            for t in np.flatnonzero(np.isin(track_video, vids)):
                bs[t], bo[t], bk[t], ratio[t] = np.nan, 0, sentinel, np.nan
                a_s[t * (K + 1): (t + 1) * (K + 1)] = np.nan
                a_o[t * (K + 1): (t + 1) * (K + 1)] = 0
        return (bs, bo, bk, ratio) + ((a_s, a_o) if want_all else (None, None))

    def _reference_signals(self, pcm_host, pcm_off, refs=None, pgs=None, sig=None, seg=None):
        """The per-video reference signals the batched calls sync against, composed of public calls: the detector
        (b2_vad_energy_zcr, or b2_vad_auditok rounded to float32) over the chunk loop's calls of the videos' PCM, with
        subtitle references (refs, from _subs_refs) for a video that has one b2_rasterize of its stream at ratio 1.0 and level 1.0, and
        with PGS references (pgs, from _pgs_refs) for a video that has one b2_rasterize_pgs of its intervals, and with
        signal references (sig, from _sig_refs, on the host) for a video that has one DeserializeSpeechTransformer's
        rule at this synchroniser's label, in float64, rounded once to float32, and with segment references (seg, from
        _seg_refs) for a video that has them the detector over each segment's samples as one signal (b2_vad_energy_zcr
        or b2_vad_auditok rounded to float32, over the chunk loop), placed by MultiSegmentVideoSpeechTransformer.fit's
        rule (segment_oracle.assemble's, in start order) into int(total * sample_rate) + 2 frames of 0.0.
        Returns (float32 signals back to back, ref_off int64[V+1])."""
        h = self.handle
        V = len(pcm_off) - 1
        if pcm_host is None:   # no video has samples: every detector signal is empty
            det, det_off = np.zeros(0, np.float32), np.zeros(V + 1, np.int64)
        elif self.auditok:
            det, det_off = h.vad_auditok(pcm_host, pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label,
                                         chunk_samples=self.chunk_samples)
        else:
            det, det_off = self._vad_energy_host(pcm_host, pcm_off)
        if refs is None and pgs is None and sig is None and seg is None:
            return det.astype(np.float32), det_off
        parts = [det[det_off[v]: det_off[v + 1]].astype(np.float32) for v in range(V)]
        if refs is not None:
            is_subs, rs, re_, rk, roff = refs
            sub, sub_off = h.rasterize(rs, re_, rk, roff, [1.0], 1, False, self.sample_rate, self.start_seconds,
                                       levels=[1.0])
            for v in np.flatnonzero(is_subs):
                parts[v] = sub[sub_off[v]: sub_off[v + 1]]
        stored = sig
        if pgs is not None:
            is_pgs, ps, pe, poff = pgs
            vids = np.flatnonzero(is_pgs)
            sig, sig_off = h.rasterize_pgs(ps, pe, np.concatenate([[0], np.cumsum(np.diff(poff)[vids])]),
                                           self.sample_rate, self.start_seconds)
            for i, v in enumerate(vids):
                parts[v] = sig[sig_off[i]: sig_off[i + 1]]
        if stored is not None:
            is_sig, x, voff = stored
            for v in np.flatnonzero(is_sig):
                xv = x[voff[v]: voff[v + 1]]
                parts[v] = np.where(xv < 1.0, np.float64(self.non_speech_label), xv).astype(np.float32)
        if seg is not None:
            video, total, s_off, s_start, s_lo, s_hi = seg
            for i, v in enumerate(video):
                js = range(int(s_off[i]), int(s_off[i + 1]))
                pieces = [pcm_host[pcm_off[v] + s_lo[j]: pcm_off[v] + s_hi[j]] for j in js]
                p_off = np.concatenate([[0], np.cumsum([len(q) for q in pieces])]).astype(np.int64)
                flat = np.concatenate(pieces + [np.zeros(0, np.int16)]).astype(np.int16)
                if self.auditok:
                    d, d_off = h.vad_auditok(flat, p_off, self.frame_rate, self.sample_rate, self.non_speech_label,
                                             chunk_samples=self.chunk_samples)
                else:
                    d, d_off = self._vad_energy_host(flat, p_off)
                L = int(float(total[i]) * self.sample_rate) + 2
                x = np.zeros(L, dtype=np.float32)
                for k, j in enumerate(js):
                    b = int(s_start[j]) * self.sample_rate
                    e = min(b + int(d_off[k + 1] - d_off[k]), L)
                    if e > b:
                        x[b:e] = d[d_off[k]: d_off[k] + (e - b)].astype(np.float32)
                parts[v] = x
        off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        return (np.concatenate(parts) if parts else np.zeros(0, np.float32)), off

    def _vad_energy_host(self, pcm_host, pcm_off):
        """b2_vad_energy_zcr over the reference's chunk loop (each signal cut into its detector calls, as the batched
        calls cut it).  Returns (float32 frames back to back, out_off int64[B+1])."""
        h = self.handle
        calls, first = h.energy_calls(pcm_off, self.frame_rate, self.sample_rate)
        det, det_off = h.vad_energy_zcr(pcm_host, calls, self.frame_rate, self.sample_rate, self.non_speech_label,
                                        self.energy_threshold, self.z_lo, self.z_hi)
        return det, det_off[first]

    def _vad_auditok_device(self, pcm, pcm_off):
        """b2_vad_auditok over the videos of the CUDA tensor pcm (chunked as the batched calls chunk them), rounded
        once to float32.  Returns (float32 CUDA tensor, ref_off int64[V+1])."""
        import torch
        h = self.handle
        pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
        ref_off = h.auditok_out_off(pcm_off, self.frame_rate, self.sample_rate, self.chunk_samples)
        ref64 = torch.empty(int(ref_off[-1]), dtype=torch.float64, device=pcm.device)
        h.vad_auditok(pcm.data_ptr(), pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label,
                      chunk_samples=self.chunk_samples, out=ref64.data_ptr(), memspace=_native.B2_DEVICE)
        return ref64.to(torch.float32), ref_off

    def ingest(self, V: int, expect_samples=None, segments=None) -> "IngestSession":
        """A batched ingest session for V videos (b2_ingest_*): their PCM arrives in pushes of any size and the
        detector runs on the device as it comes, so only the reference signals are ever held - not the videos'
        whole decodes.  The results equal the whole-PCM sync methods' over the same bytes.  expect_samples [V]: a
        sizing hint (e.g. ffprobe's duration times frame_rate); a longer video still fits.  The audio detector is
        this synchroniser's (the one after ``subs_then_``).
        segments (``--multi-segment-sync``): dict(seg_video, seg_total, seg_off, seg_start), e.g. from
        ``ingest_segment_table``; those videos take their sampled segments' PCM (``push_segment``) and are synced
        against the sparse reference, as the sync methods with ``segment_table(..., piece_samples=...)`` over the
        pieces pushed.  A segment video's expect_samples entry is the hint for each of its segments.
        Videos whose reference needs no audio - an embedded text stream with a ``subs_then_`` detector, PGS intervals,
        a stored signal - take no pushes: their references are given to ``IngestSession.sync_tracks`` as the sync
        methods' keyword arguments."""
        return IngestSession(self, V, expect_samples, segments)


class IngestSession:
    """A batched ingest session (``BatchSynchronizer.ingest``).  ``push`` / ``push_many`` append s16le mono PCM to
    videos in any sizes and interleaving (bytes, uint8 or int16 arrays; copied before they return, detected on the
    device without a host synchronisation), ``windows`` reports the reference frames fixed so far, and
    ``sync_tracks`` runs the sync chain over the references and closes the session.  The handle is shared with the
    synchroniser and is not thread-safe: push from one thread."""

    def __init__(self, sync: BatchSynchronizer, V: int, expect_samples=None, segments=None) -> None:
        self.sync = sync
        self.V = int(V)
        self._bytes = np.zeros(self.V, dtype=np.int64)
        self._seg = None
        det = _native.B2_DETECTOR_AUDITOK if sync.auditok else _native.B2_DETECTOR_ENERGY_ZCR
        sync.handle.ingest_begin(self.V, sync.frame_rate, sync.sample_rate, sync.non_speech_label, detector=det,
                                 energy_threshold=sync.energy_threshold, z_lo=sync.z_lo, z_hi=sync.z_hi,
                                 chunk_samples=sync.chunk_samples, expect_samples=expect_samples)
        if segments is not None:
            try:
                sync.handle.ingest_segments(*(segments[k] for k in ("seg_video", "seg_total", "seg_off", "seg_start")))
            except BaseException:
                self.abort()
                raise
            # (seg_video, seg_total): what _reference_lengths and the no-speech rule read of a segment table
            self._seg = (np.asarray(segments["seg_video"], dtype=np.int32),
                         np.asarray(segments["seg_total"], dtype=np.float64))

    def push(self, video: int, chunk) -> None:
        self.push_many([video], [chunk])

    def push_segment(self, video: int, segment: int, chunk) -> None:
        """chunk to segment ``segment`` (counted within the video's segments) of segment video ``video``."""
        self.push_many([video], [chunk], segments=[segment])

    def push_many(self, videos, chunks, segments=None) -> None:
        """chunks[i] to video videos[i], in order (one b2_ingest_push), or with ``segments`` to its segment segments[i]
        (one b2_ingest_push_segments)."""
        self.sync.handle.ingest_push(videos, chunks, segments)
        if segments is None:
            for v, c in zip(videos, chunks):
                self._bytes[int(v)] += memoryview(c).nbytes

    def drop_segment(self, video: int, segment: int) -> None:
        """Discard a segment (the reference's "failed to extract segment"): what was pushed to it takes no part in the
        reference, and a later push to it is refused."""
        self.sync.handle.ingest_drop_segment(video, segment)

    def windows(self) -> np.ndarray:
        return self.sync.handle.ingest_windows()

    def abort(self) -> None:
        self.sync.handle.ingest_abort()

    def sync_tracks(self, track_video, cue_start, cue_end, cue_off, cue_keep=None, speech_video=None, out=None,
                    all_out=None, want_all: bool = False, **streams):
        """Sync track t (cue list cue_off[t] .. cue_off[t+1]) against video track_video[t] (non-decreasing) and close
        the session.  Without ``out``: what ``sync_host_tracks`` returns over the videos' PCM back to back.  With
        ``out`` (CUDA tensors best_score f64[T], best_offset i32[T], best_k i32[T], gss_ratio f64[T] with the search;
        ``all_out`` as for sync_device_tracks): what ``sync_device_tracks`` returns, with nothing synchronised.
        ``speech_video`` as there.  The golden-section search runs on the device only: outside its envelope the call
        raises (there is no PCM left to compose it from).  A segment video without a frame > 0 raises the reference's
        ValueError on the host and gets ``best_k == B2_BEST_K_NO_SPEECH`` on the device, as the sync methods do.
        streams: the references of videos that took no pushes, as the sync methods take them - the embedded text
        streams of a ``subs_then_`` detector (ref_cue_start, ref_cue_end, ref_cue_off, ref_stream_video and
        ref_cue_content or ref_cue_keep), PGS intervals (pgs_start, pgs_end, pgs_off, pgs_video) and stored signals
        (sig, sig_off, sig_video: a numpy array without ``out``, a CUDA tensor with it), combined by the same rules.
        Segments are declared at ``ingest``, not here.  A video given such a reference that received pushed bytes is
        refused (b2_ingest_sync_refs)."""
        s = self.sync
        h = s.handle
        pcm_off = np.concatenate([[0], np.cumsum(self._bytes // 2)]).astype(np.int64)
        on_device = out is not None
        sig_in = streams.get("sig")
        try:
            if any(streams.get(k) is not None for k in _SEG_ARGS):
                raise ValueError("a session declares its segments at ingest(segments=...), not at sync_tracks")
            refs, pgs, sig, _ = s._all_refs(self.V, streams, on_device, seg=self._seg)
            speech = s._speech_request(speech_video, pcm_off, refs, pgs, sig, seg=self._seg, on_device=on_device)
        except Exception:
            self.abort()
            raise
        tables = {}
        if refs is not None:
            tables.update(zip(("ref_is_subs", "ref_cue_start_s", "ref_cue_end_s", "ref_cue_keep", "ref_cue_off"), refs))
        if pgs is not None:
            tables.update(zip(("ref_is_pgs", "pgs_start_s", "pgs_end_s", "pgs_off"), pgs))
        if sig is not None:
            is_sig, x, voff = sig
            tables.update(ref_is_sig=is_sig, x=x if isinstance(x, np.ndarray) else (x.data_ptr() if x.numel() else None),
                          sig_off=voff)
            if on_device and x is not sig_in:
                # a converted copy: ready before the handle's stream reads it, and kept until the call is done
                import torch
                torch.cuda.current_stream(x.device).synchronize()
        cues = (track_video, cue_start, cue_end, cue_keep, cue_off, s.ratios, s.start_seconds, s.max_offset_samples)
        with s._speech_output(speech):
            if on_device:
                ptrs = {k: out[k].data_ptr() for k in ("best_score", "best_offset", "best_k")}
                if s.gss:
                    ptrs["gss_ratio"] = out["gss_ratio"].data_ptr()
                if all_out:
                    ptrs.update(all_score=all_out["score"].data_ptr(), all_offset=all_out["offset"].data_ptr())
                h.ingest_sync_tracks(*cues, gss=s.gss, memspace=_native.B2_DEVICE, **ptrs, **tables)
            else:
                res = h.ingest_sync_tracks(*cues, gss=s.gss, want_all=want_all, memspace=_native.B2_HOST, **tables)
        if on_device:
            if sig is not None and sig[1] is not sig_in:
                h.synchronize()
            if speech is not None:
                out["speech"], out["speech_off"] = s._speech_result(speech)
            return out
        s._raise_bad_signals(sig, res[2])
        s._raise_no_speech(self._seg, res[2], track_video)
        res = res[:6] if want_all else res[:3] + res[5:6]
        return res if speech is None else res + s._speech_result(speech)


def ingest_segment_table(totals, videos, segment_count: int = 8, segment_duration: int = 60,
                         skip_intro_outro: bool = False) -> dict:
    """The ``segments`` of ``BatchSynchronizer.ingest`` for the videos ``videos`` (increasing) of probed durations
    ``totals`` (seconds): MultiSegmentVideoSpeechTransformer._segment_starts with the reference's knobs, as
    ``segment_table`` without seg_lo / seg_hi (a session's pushes supply the samples)."""
    videos = np.ascontiguousarray(videos, dtype=np.int64)
    pcm_off = np.zeros(int(videos.max()) + 2 if len(videos) else 1, dtype=np.int64)
    t = segment_table(pcm_off, SAMPLE_RATE, videos, totals, segment_count, segment_duration, skip_intro_outro)
    return {k: t[k] for k in ("seg_video", "seg_total", "seg_off", "seg_start")}


def sync_media(paths, sync: BatchSynchronizer, track_video, cue_start, cue_end, cue_off, cue_keep=None,
               max_decoders: int = 4, ffmpeg_path: Optional[str] = None, max_duration_seconds: Optional[float] = None,
               ref_stream: Optional[str] = None, expect_samples=None, speech_video=None, want_all: bool = False,
               multi_segment=False, segment_count: int = 8, segment_duration: int = 60,
               skip_intro_outro: bool = False, pgs_ref_stream=None, **streams):
    """``ffs movie.mkv -i a.srt ...`` for a library: decodes paths[v] with up to ``max_decoders`` ffmpeg processes at
    a time (VideoSpeechTransformer._build_ffmpeg_args: ``-ss`` from the synchroniser's start_seconds, ``-t`` from
    max_duration_seconds, ffmpeg_path, ref_stream), reads each pipe in the reference's 100 s ``read()`` calls on a
    thread per decoder, pushes the chunks into one ingest session from this thread, and syncs the tracks as
    ``IngestSession.sync_tracks`` does on the host.  No video's whole decode is ever held.
    ``multi_segment`` (``--multi-segment-sync``): True for every video, or a list of video indices.  Such a video's
    duration is probed with ffprobe (MultiSegmentVideoSpeechTransformer._probe_duration; a failure raises its
    ValueError), and only its ``segment_count`` windows of ``segment_duration`` seconds (``_segment_starts``, with
    ``skip_intro_outro``) are decoded, each by its own ``ffmpeg -ss start -t segment_duration`` in the same pool.  A
    segment decoder that fails or cannot start is logged as the reference's "failed to extract segment" warning and
    the segment is dropped; a failing full-audio decoder aborts, as without segments.  The synchroniser's
    start_seconds applies to the subtitle tracks only there.
    References that are not a video's audio (make_reference_pipe's order): such a video gets no decoder job.
    - A path ending in ``npz`` / ``npy`` (the reference's ``_ref_format``) is a stored signal (``--serialize-speech``):
      it is loaded with ``load_stored_speech`` and passed as ``sig``.  A subtitle file (``srt``, ``ass``, ``ssa``,
      ``sub``) is refused with ValueError before anything starts: the batched calls have no subtitle-file references.
    - ``pgs_ref_stream`` (``--pgs-ref-stream``): None, ``"auto"`` (the first PGS stream), one specifier (``"s:N"`` /
      ``"0:s:N"``) for every video that is not a stored signal, or a list of V such entries (None: not PGS).  Each PGS
      video's display intervals are probed with ffprobe (PGSSpeechTransformer._probe_intervals) as jobs of the same
      pool; a failed probe, a stream without timings or intervals PGSSpeechTransformer.fit refuses (checked by fit's
      own rasterisation before the sync) raise the reference's ValueError, with no fallback to audio.
    - ``streams``: the embedded text streams of a ``subs_then_`` synchroniser, as the sync methods take them (their
      extraction stays the caller's job); any other keyword is refused with TypeError before anything starts.  A video
      that select_reference_streams gives a stream, and that is not a PGS or segment video, is not decoded.
    The combinations follow the sync methods: PGS wins over text; a signal video with a PGS or text reference, and a
    segment video with a PGS or signal reference, are refused; a segment video's text stream is dropped.  Returns what
    ``sync_host_tracks`` returns over the decoded audio videos' PCM and the same references."""
    import queue
    import shutil
    import subprocess
    import threading

    from .constants import detector_chunk_bytes
    from .speech_transformers import MultiSegmentVideoSpeechTransformer, VideoSpeechTransformer, logger
    V = len(paths)
    if multi_segment is True:
        seg_videos = list(range(V))
    elif multi_segment is False or multi_segment is None:
        seg_videos = []
    else:
        seg_videos = sorted({int(v) for v in multi_segment})
        if seg_videos and (seg_videos[0] < 0 or seg_videos[-1] >= V):
            raise ValueError("multi_segment lists video indices in [0, %d), not %r" % (V, list(multi_segment)))
    if seg_videos and max_duration_seconds is not None:
        raise ValueError("max_duration_seconds limits a full decode; multi_segment decodes sampled segments of "
                         "segment_duration seconds instead")
    from .speech_transformers import PGSSpeechTransformer, load_stored_speech
    # PGS and signal references come from pgs_ref_stream and the paths, segments from multi_segment: streams holds the
    # text streams alone, refused otherwise before any decoder starts
    other = sorted(k for k in streams if k not in _STREAM_ARGS)
    if other:
        raise TypeError("sync_media takes embedded text streams as keyword arguments (%s), not %s; PGS references "
                        "come from pgs_ref_stream, stored signals from .npz / .npy paths and segments from "
                        "multi_segment" % (", ".join(_STREAM_ARGS), ", ".join(other)))
    # the reference's choice by file type (make_reference_pipe: _ref_format is the name's last three characters)
    for p in paths:
        if str(p)[-3:] in _SUBTITLE_EXTENSIONS:
            raise ValueError("%r is a subtitle file; the batched calls take no subtitle-file references" % str(p))
    sig_videos = [v for v in range(V) if str(paths[v])[-3:] in ("npz", "npy")]
    if pgs_ref_stream is None or isinstance(pgs_ref_stream, str):
        pgs_spec = [None if v in sig_videos else pgs_ref_stream for v in range(V)]
    else:
        pgs_spec = list(pgs_ref_stream)
        if len(pgs_spec) != V:
            raise ValueError("pgs_ref_stream has %d entries for %d paths" % (len(pgs_spec), V))
    pgs_videos = [v for v in range(V) if pgs_spec[v] is not None]
    sigs = [np.asarray(load_stored_speech(paths[v]), dtype=np.float64).ravel() for v in sig_videos]
    sig_kw = {}
    if sig_videos:
        sig_kw = dict(sig=np.concatenate(sigs), sig_video=np.array(sig_videos, np.int64),
                      sig_off=np.concatenate([[0], np.cumsum([len(x) for x in sigs])]).astype(np.int64))
    # the combinations, checked before anything starts (PGS intervals stand empty here): the text videos that stay
    empty = np.zeros(0)
    pgs_stand = dict(pgs_start=empty, pgs_end=empty, pgs_off=np.zeros(len(pgs_videos) + 1, np.int64),
                     pgs_video=np.array(pgs_videos, np.int64)) if pgs_videos else {}
    refs, _, _, _ = sync._all_refs(V, dict(streams, **pgs_stand, **sig_kw), on_device=False,
                                   seg=(np.array(seg_videos, np.int32),) if seg_videos else None)
    text_videos = [] if refs is None else [int(v) for v in np.flatnonzero(refs[0])]
    no_audio = set(sig_videos) | set(pgs_videos) | set(text_videos)

    def ffmpeg_args(path, start_seconds, duration):
        return VideoSpeechTransformer(vad=sync.detector, sample_rate=sync.sample_rate, frame_rate=sync.frame_rate,
                                      non_speech_label=sync.non_speech_label, start_seconds=start_seconds,
                                      ffmpeg_path=ffmpeg_path, ref_stream=ref_stream,
                                      max_duration_seconds=duration)._build_ffmpeg_args(path)

    # the decoder jobs: (video, segment or None, ffmpeg arguments); a segment video has one job per segment, a PGS video
    # one probe job (video, _PGS_JOB, its PGSSpeechTransformer)
    is_seg = set(seg_videos)
    jobs = [(v, None, ffmpeg_args(paths[v], sync.start_seconds, max_duration_seconds)) for v in range(V)
            if v not in is_seg and v not in no_audio]
    for v in pgs_videos:
        spec = None if pgs_spec[v] == "auto" else pgs_spec[v]
        jobs.append((v, _PGS_JOB, PGSSpeechTransformer(sample_rate=sync.sample_rate, start_seconds=sync.start_seconds,
                                                       ffmpeg_path=ffmpeg_path, ref_stream=spec)))
    pgs_intervals = {}
    segments = None
    if seg_videos:
        mst = MultiSegmentVideoSpeechTransformer(vad=sync.detector, sample_rate=sync.sample_rate,
                                                 frame_rate=sync.frame_rate, non_speech_label=sync.non_speech_label,
                                                 segment_count=segment_count, segment_duration=segment_duration,
                                                 skip_intro_outro=skip_intro_outro, ffmpeg_path=ffmpeg_path,
                                                 ref_stream=ref_stream)
        segments = ingest_segment_table([mst._probe_duration(paths[v]) for v in seg_videos], seg_videos,
                                        segment_count, segment_duration, skip_intro_outro)
        for i, v in enumerate(seg_videos):
            for j in range(int(segments["seg_off"][i]), int(segments["seg_off"][i + 1])):
                start = int(segments["seg_start"][j])
                jobs.append((v, j - int(segments["seg_off"][i]), ffmpeg_args(paths[v], start, segment_duration)))
        expect = np.zeros(V, dtype=np.int64) if expect_samples is None else np.array(expect_samples, dtype=np.int64)
        expect[seg_videos] = int(round(segment_duration * sync.frame_rate))   # the hint of each segment
        expect_samples = expect
    decoders = [j for j in jobs if j[1] is not _PGS_JOB]
    if decoders and shutil.which(decoders[0][2][0]) is None:
        raise ValueError("cannot decode media: no ffmpeg binary found at %r" % decoders[0][2][0])
    n_read = detector_chunk_bytes(sync.frame_rate, sync.sample_rate)
    n_workers = max(1, min(int(max_decoders), len(jobs)))
    chunks: "queue.Queue" = queue.Queue(maxsize=2 * n_workers)
    todo: "queue.Queue" = queue.Queue()
    for job in range(len(jobs)):
        todo.put(job)
    stop = threading.Event()

    def probe(job: int):
        """A PGS video's display intervals (PGSSpeechTransformer.fit before its raster) into pgs_intervals."""
        v, _, t = jobs[job]
        intervals = t._probe_intervals(paths[v])
        if not intervals:
            given = t._given_stream()
            raise ValueError("No subtitle timings found in PGS stream {}.".format(given) if given is not None
                             else "No subtitle timings found in the PGS intervals given.")
        pgs_intervals[v] = intervals

    def decode(job: int):
        """Pushes job's 100 s reads to `chunks` (a PGS job: probes its intervals); returns why it failed (None: it
        did not)."""
        if jobs[job][1] is _PGS_JOB:   # a failed probe is the reference's ValueError, handed back as it is
            try:
                probe(job)
            except ValueError as e:
                return e
            return None
        proc = subprocess.Popen(jobs[job][2], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
        try:
            while not stop.is_set():
                data = proc.stdout.read(n_read)
                if not data:
                    break
                chunks.put((job, data, None))
        finally:
            if stop.is_set():
                proc.kill()
            proc.stdout.close()
            status = proc.wait()
        return "ffmpeg exited with status %d" % status if status and not stop.is_set() else None

    def worker() -> None:
        # every job taken ends with exactly one (job, None, error) sentinel, whatever happens while decoding it
        while not stop.is_set():
            try:
                job = todo.get_nowait()
            except queue.Empty:
                return
            try:
                err = decode(job)
            except Exception as e:   # Popen or the pipe failed (missing binary, EMFILE, ...)
                err = "%s: %s" % (type(e).__name__, e)
            chunks.put((job, None, err))

    session = sync.ingest(V, expect_samples, segments)
    threads = [threading.Thread(target=worker, daemon=True) for _ in range(n_workers)]
    for t in threads:
        t.start()
    try:
        left = len(jobs)
        while left:
            job, data, err = chunks.get()
            v, seg, _ = jobs[job]
            if data is not None:
                if seg is None:
                    session.push(v, data)
                else:
                    session.push_segment(v, seg, data)
                continue
            left -= 1
            if isinstance(err, Exception):
                raise err
            if err and seg is not None:   # one bad window must not sink the sync (speech_transformers.py:878-882)
                start = int(segments["seg_start"][int(segments["seg_off"][seg_videos.index(v)]) + seg])
                logger.warning("failed to extract segment at %ds: %s", start, err)
                session.drop_segment(v, seg)
            elif err:
                raise RuntimeError("decoding %r failed: %s" % (paths[v], err))
    except BaseException:
        stop.set()
        session.abort()
        while any(t.is_alive() for t in threads):   # drain so that no decoder blocks on a full queue
            try:
                chunks.get(timeout=0.05)
            except queue.Empty:
                pass
        raise
    for t in threads:
        t.join()
    pgs_kw = {}
    if pgs_videos:
        # a list the probe returns can still be one PGSSpeechTransformer.fit refuses (a non-finite or too large time):
        # fit's own rasterisation raises the reference's ValueError for it, before the sync
        try:
            for v, seg, t in jobs:
                if seg is _PGS_JOB:
                    t.fit(pgs_intervals[v])
        except BaseException:
            session.abort()
            raise
        iv = [np.asarray(pgs_intervals[v], dtype=np.float64).reshape(-1, 2) for v in pgs_videos]
        pgs_kw = dict(pgs_start=np.concatenate([x[:, 0] for x in iv]), pgs_end=np.concatenate([x[:, 1] for x in iv]),
                      pgs_off=np.concatenate([[0], np.cumsum([len(x) for x in iv])]).astype(np.int64),
                      pgs_video=np.array(pgs_videos, np.int64))
    return session.sync_tracks(track_video, cue_start, cue_end, cue_off, cue_keep, speech_video=speech_video,
                               want_all=want_all, **streams, **pgs_kw, **sig_kw)


def select_reference_streams(V: int, cue_start, cue_end, cue_off, stream_video, start_seconds: float = 0.0,
                             content=None, keep=None):
    """VideoSpeechTransformer.try_fit_using_embedded_subs' choice among a video's subtitle streams
    (ffsubsync/speech_transformers.py:505-523): every stream goes through SubtitleSpeechTransformer, whose
    ``max_time_`` is ``max(0, largest scaled cue end) - start_seconds`` (:958-961, metadata cues included), and the
    stream with the largest ``max_time_`` wins, the first on a tie (np.argmax).  A stream without cues counts
    (``max_time_ = -start_seconds``).  S streams: cue_off [S+1] (absolute into cue_start / cue_end),
    stream_video [S] (non-decreasing video index).  Keep flags: ``not _is_metadata(text, first or last cue of its
    stream)`` (:966) when ``content`` (the cue texts) is given, else ``keep`` (None = keep every cue).  Returns
    (ref_is_subs u8[V], ref_cue_start, ref_cue_end, ref_cue_keep, ref_cue_off int64[V+1]) - the chosen stream of
    each video - for b2_sync_tracks_subs.  A video without a stream gets ``ref_is_subs = 0`` and no cues."""
    from datetime import timedelta

    from .speech_transformers import _is_metadata
    cue_start = np.ascontiguousarray(cue_start, dtype=np.float64)
    cue_end = np.ascontiguousarray(cue_end, dtype=np.float64)
    cue_off = np.ascontiguousarray(cue_off, dtype=np.int64)
    stream_video = np.ascontiguousarray(stream_video, dtype=np.int64)
    S = len(cue_off) - 1
    if len(stream_video) != S:
        raise ValueError("ref_stream_video has %d entries for %d streams" % (len(stream_video), S))
    if S and (np.any(np.diff(stream_video) < 0) or stream_video[0] < 0 or stream_video[-1] >= V):
        raise ValueError("ref_stream_video must be non-decreasing video indices in [0, %d)" % V)
    if np.any(np.diff(cue_off) < 0) or (S and (cue_off[0] < 0 or cue_off[-1] > min(len(cue_start), len(cue_end)))):
        raise ValueError("ref_cue_off must be non-decreasing and within the cue arrays")
    if content is not None:
        if len(content) < int(cue_off[-1]):
            raise ValueError("ref_cue_content has %d entries for %d cues" % (len(content), int(cue_off[-1])))
        keep = np.ones(len(cue_start), dtype=np.uint8)
        for s in range(S):
            c0, c1 = int(cue_off[s]), int(cue_off[s + 1])
            for i in range(c0, c1):
                keep[i] = not _is_metadata(content[i], i == c0 or i + 1 == c1)
    elif keep is not None:
        keep = np.ascontiguousarray(keep, dtype=np.uint8)
    best = np.full(V, -1, dtype=np.int64)
    best_time = [0.0] * V
    for s in range(S):
        c0, c1 = int(cue_off[s]), int(cue_off[s + 1])
        max_time = 0
        if c1 > c0:
            e = float(np.max(cue_end[c0:c1]))
            # the largest scaled end is the scaled largest end (timedelta's rounding is monotone); a non-finite
            # time is left for b2_sync_tracks_subs to reject with its index
            max_time = max(max_time, timedelta(seconds=e).total_seconds() if np.isfinite(e) else e)
        t = max_time - start_seconds
        v = int(stream_video[s])
        if best[v] < 0 or t > best_time[v]:
            best[v], best_time[v] = s, t
    is_subs = (best >= 0).astype(np.uint8)
    lens = [int(cue_off[best[v] + 1] - cue_off[best[v]]) if best[v] >= 0 else 0 for v in range(V)]
    ref_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    pick = np.concatenate([np.arange(cue_off[best[v]], cue_off[best[v] + 1]) for v in range(V) if best[v] >= 0]
                          + [np.zeros(0, np.int64)]).astype(np.int64)
    return is_subs, cue_start[pick], cue_end[pick], (None if keep is None else keep[pick]), ref_off
