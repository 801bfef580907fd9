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
from typing import Optional, Sequence

import numpy as np

from . import _native
from .constants import (BATCH_VADS, DEFAULT_ENERGY_THRESHOLD, DEFAULT_MAX_OFFSET_SECONDS, SAMPLE_RATE,
                        detector_chunk_bytes)


def load_serialized_speech(paths, non_speech_label: float = 0.0):
    """Batch ingest of ``--serialize-speech`` / ``--make-test-case`` artefacts (``.npz`` with key
    "speech", or ``.npy``): each file goes through DeserializeSpeechTransformer
    (ffsubsync/speech_transformers.py:987-1009: values < 1 become ``non_speech_label``).
    Returns (signals float32 back to back, offsets int64[B+1]) ready for ``sync_signals``."""
    from .speech_transformers import DeserializeSpeechTransformer
    sigs = [np.asarray(DeserializeSpeechTransformer(non_speech_label).fit(p).transform(), dtype=np.float32)
            for p in paths]
    off = np.concatenate([[0], np.cumsum([len(s) for s in sigs])]).astype(np.int64)
    return (np.concatenate(sigs) if sigs else np.zeros(0, np.float32)), off


# keyword arguments of the sync methods that describe the embedded subtitle streams of a subs_then_ detector
_STREAM_ARGS = ("ref_cue_start", "ref_cue_end", "ref_cue_off", "ref_stream_video", "ref_cue_content", "ref_cue_keep")


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
    ``pcm`` may be None when no video has any).  Extracting the streams from containers (ffprobe / ffmpeg), bitmap
    (PGS) streams and ``--reference-stream`` remain the caller's job.  Without streams the results are those of the
    detector alone."""

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
        # auditok: samples per detector call, as VideoSpeechTransformer._chunks reads them
        self.chunk_samples = detector_chunk_bytes(frame_rate, sample_rate) // 2

    @property
    def auditok(self) -> bool:
        return self.detector == "auditok"

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

    def _dispatch(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, gss: bool, **kw):
        """The batched call of this synchroniser's detector with the search on or off: b2_sync_tracks_subs with
        subtitle references (refs, from _subs_refs), else b2_sync_tracks_auditok for auditok, else
        b2_sync_tracks_gss / b2_sync_tracks.  pcm: int16 numpy array, CUDA tensor or None; kw: the outputs (device
        pointers) or want_all, and memspace.  Returns (best_score, best_offset, best_k, all_score, all_offset), plus
        (gss_ratio, gss_evals) with gss."""
        h = self.handle
        p = pcm if pcm is None or isinstance(pcm, np.ndarray) else pcm.data_ptr()
        cues = (cue_start, cue_end, cue_keep, cue_off, self.ratios, self.start_seconds, self.max_offset_samples)
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

    def _sync_or_compose(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, **kw):
        """_dispatch with this synchroniser's search.  Outside the envelope of the device-driven search
        (B2_ERR_UNSUPPORTED) the search is composed of public steps instead (_gss_compose).  Returns
        (best_score, best_offset, best_k, all_score, all_offset), plus gss_ratio with the search; composed results
        are numpy arrays (all_* None unless want_all or device outputs were given)."""
        try:
            return self._dispatch(pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, self.gss,
                                  **kw)[:6]
        except _native.NativeError as e:
            if not (self.gss and _is_unsupported(e)):
                raise
        want_all = kw.get("want_all", False) or kw.get("all_score") is not None
        bs, bo, bk, ratio, a_s, a_o = self._gss_compose(pcm, pcm_off, track_video, cue_start, cue_end, cue_off,
                                                        cue_keep, want_all=want_all, refs=refs)
        return bs, bo, bk, a_s, a_o, ratio

    def use_torch_stream(self) -> None:
        """Launch on torch's current stream (so torch events / NCCL ops order against our kernels)."""
        import torch
        self.handle.set_stream(torch.cuda.current_stream().cuda_stream)

    def sync_device(self, pcm, pcm_off, cue_start, cue_end, cue_off, cue_keep=None, out=None, all_out=None,
                    inputs_resident: bool = False, **streams):
        """pcm: int16 CUDA tensor with all pairs back to back; pcm_off: [B+1] sample offsets (host).
        out: optional dict of preallocated CUDA tensors best_score f64[B], best_offset i32[B],
        best_k i32[B].  Returns that dict; nothing is synchronised.
        inputs_resident=True (B2_DEVICE_RESIDENT): the caller promises that nothing queued on the handle's
        stream before this call still writes ``pcm`` (a corpus that sits in HBM).  Back-to-back calls then
        overlap: the VAD of this batch starts while the last correlation chain of the previous batch is
        still running.  Results are identical; outputs stay ordered on the stream.
        With a ``subs_then_`` detector the embedded subtitle streams come as keyword arguments (see the class)."""
        import torch
        B = len(pcm_off) - 1
        K = len(self.ratios)
        if self.gss or self.auditok or self.subs_then:   # the identity track map: pair b is track b of video b
            return self.sync_device_tracks(pcm, pcm_off, np.arange(B, dtype=np.int32), cue_start, cue_end, cue_off,
                                           cue_keep, out=out, all_out=all_out, inputs_resident=inputs_resident,
                                           **streams)
        self._subs_refs(B, streams)   # rejects streams and unknown keywords
        dev = pcm.device
        if out is None:
            out = {"best_score": torch.empty(B, dtype=torch.float64, device=dev),
                   "best_offset": torch.empty(B, dtype=torch.int32, device=dev),
                   "best_k": torch.empty(B, dtype=torch.int32, device=dev)}
        a_s = all_out["score"].data_ptr() if all_out else None
        a_o = all_out["offset"].data_ptr() if all_out else None
        self.handle.sync_batch(
            pcm.data_ptr(), pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label,
            self.energy_threshold, self.z_lo, self.z_hi, cue_start, cue_end, cue_keep, cue_off, self.ratios,
            self.start_seconds, self.max_offset_samples, out["best_score"].data_ptr(),
            out["best_offset"].data_ptr(), out["best_k"].data_ptr(), a_s, a_o,
            memspace=_native.B2_DEVICE_RESIDENT if inputs_resident else _native.B2_DEVICE)
        assert K == len(self.ratios)
        return out

    def sync_device_tracks(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep=None, out=None,
                           all_out=None, inputs_resident: bool = False, **streams):
        """sync_device for several subtitle tracks per video (``ffs movie.mkv -i en.srt de.srt ...``):
        pcm holds the V videos back to back, pcm_off: [V+1] sample offsets (host); track t (cue list
        cue_off[t] .. cue_off[t+1]) is synced against video track_video[t] (host, non-decreasing).  Each
        video's PCM is read and run through the VAD once, however many tracks it has.  out: optional dict
        of CUDA tensors best_score f64[T], best_offset i32[T], best_k i32[T]; all_out: optional
        {"score": f64[T*K], "offset": i32[T*K]}.  Returns out; nothing is synchronised.  inputs_resident
        as for sync_device (resident calls of both methods chain with each other).
        With the golden-section search (a trailing None in ratios) out also holds gss_ratio f64[T] and all_out
        is {"score": f64[T*(K+1)], "offset": i32[T*(K+1)]} with column K the search's candidate.
        streams: the embedded subtitle streams of a ``subs_then_`` detector (ref_cue_start, ... - see the class)."""
        import torch
        T = len(track_video)
        refs = self._subs_refs(len(pcm_off) - 1, streams)
        dev = pcm.device if pcm is not None else torch.device("cuda", self.handle.device)
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
        res = self._sync_or_compose(pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs,
                                    memspace=memspace, **ptrs)
        if isinstance(res[0], np.ndarray):   # composed on the host
            for k, v in zip(keys, res[:3] + res[5:]):
                out[k].copy_(torch.from_numpy(v))
            if all_out:
                all_out["score"].copy_(torch.from_numpy(res[3]))
                all_out["offset"].copy_(torch.from_numpy(res[4]))
        return out

    def sync_host_tracks(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep=None,
                         want_all=False, **streams):
        """sync_device_tracks with host buffers (pcm: int16 numpy array of the V videos).  Blocks until
        results are on the host.  Returns (best_score, best_offset, best_k[, all_score, all_offset]) per
        track, and gss_ratio last with the golden-section search.  streams as for sync_device_tracks."""
        refs = self._subs_refs(len(pcm_off) - 1, streams)
        res = self._sync_or_compose(pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs,
                                    want_all=want_all, memspace=_native.B2_HOST)
        return res if want_all else res[:3] + res[5:]

    def sync_signals(self, ref, ref_off, cue_start, cue_end, cue_off, cue_keep=None):
        """Same as sync_device but starting from reference speech SIGNALS (100 Hz float32, all pairs
        back to back; numpy array or CUDA tensor) instead of PCM - the replay path of the
        reference's test-case bundles: ``ref.npz{"speech"}`` + ``in.srt``
        (ffsubsync/ffsubsync.py:338-343,639-644; DeserializeSpeechTransformer).
        Returns (best_score f64[B], best_offset i32[B], best_k i32[B]) as numpy arrays, and gss_ratio f64[B]
        last with the golden-section search (gss_batch.gss_align_batch on the same signals, merged as
        candidate K by gss_batch.combine_gss)."""
        import torch
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
                                      rank: int = 0, world: int = 1, group=None):
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
        if self.gss:
            raise ValueError("sync_device_candidate_sharded shards the ratio grid; it does not run the "
                             "golden-section search (None in ratios)")
        if self.subs_then:
            raise ValueError("sync_device_candidate_sharded runs the detector on every video; it does not take "
                             "embedded subtitle references (vad=%r)" % self.vad)
        h = self.handle
        self.use_torch_stream()   # torch ops and NCCL below are ordered against our kernels by the stream
        pcm_off = np.ascontiguousarray(pcm_off, dtype=np.int64)
        B, K = len(pcm_off) - 1, len(self.ratios)
        dev = pcm.device
        mine = distributed.shard_candidates(K, rank, world)
        if self.auditok:   # b2_vad_auditok's float64 signal, rounded once to float32
            ref, ref_off = self._vad_auditok_device(pcm, pcm_off)
        else:
            fpw = h.frames_per_window(self.frame_rate, self.sample_rate)
            ref_off = np.concatenate([[0], np.cumsum((np.diff(pcm_off) + fpw - 1) // fpw)]).astype(np.int64)
            ref = torch.empty(int(ref_off[-1]), dtype=torch.float32, device=dev)
            h.vad_energy_zcr(pcm.data_ptr(), pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label,
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

    def sync_host(self, pcm, pcm_off, cue_start, cue_end, cue_off, cue_keep=None, want_all=False, **streams):
        """pcm: int16 numpy array (ideally backed by pinned memory).  Blocks until results are on
        the host.  Returns (best_score, best_offset, best_k[, all_score, all_offset]), and gss_ratio last
        with the golden-section search.  With a ``subs_then_`` detector the embedded subtitle streams come as
        keyword arguments (see the class)."""
        if self.gss or self.auditok or self.subs_then:
            return self.sync_host_tracks(pcm, pcm_off, np.arange(len(pcm_off) - 1, dtype=np.int32), cue_start,
                                         cue_end, cue_off, cue_keep, want_all=want_all, **streams)
        self._subs_refs(len(pcm_off) - 1, streams)   # rejects streams and unknown keywords
        res = self.handle.sync_batch(
            pcm, pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label, self.energy_threshold,
            self.z_lo, self.z_hi, cue_start, cue_end, cue_keep, cue_off, self.ratios, self.start_seconds,
            self.max_offset_samples, want_all=want_all, memspace=_native.B2_HOST)
        return res if want_all else res[:3]

    def _gss_compose(self, pcm, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep=None, want_all=False,
                     refs=None):
        """The golden-section search outside the envelope of the device-driven search, composed of public steps:
        the grid (this synchroniser's batched call with the search off), gss_align_batch on each track's reference
        signal (_reference_signals, with subtitle references refs from _subs_refs) and the reference's combine.
        pcm: int16 numpy array or CUDA tensor (or None without audio).  Returns numpy arrays (best_score,
        best_offset, best_k, gss_ratio, all_score, all_offset) (all_* None unless want_all)."""
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
        grid = self._dispatch(pcm_host, pcm_off, track_video, cue_start, cue_end, cue_off, cue_keep, refs, False,
                              want_all=True, memspace=_native.B2_HOST)
        ref, ref_off = self._reference_signals(pcm_host, pcm_off, refs)
        # one copy of its video's reference signal per track
        parts = [ref[ref_off[v]: ref_off[v + 1]] for v in track_video]
        t_off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        t_ref = np.concatenate(parts).astype(np.float32) if parts else np.zeros(0, np.float32)
        g = gss_align_batch(t_ref, t_off, cue_start, cue_end, cue_off, cue_keep, self.max_offset_samples,
                            self.sample_rate, self.start_seconds, handle=h)
        bs, bo, bk, ratio, a_s, a_o = combine_gss(grid[0], grid[1], grid[2], g, K, self.max_offset_samples,
                                                  grid[3], grid[4])
        return (bs, bo, bk, ratio) + ((a_s, a_o) if want_all else (None, None))

    def _reference_signals(self, pcm_host, pcm_off, refs=None):
        """The per-video reference signals the batched calls sync against, composed of public calls: the detector
        (b2_vad_energy_zcr, or b2_vad_auditok rounded to float32) over the videos' PCM, and with subtitle references
        (refs, from _subs_refs) for a video that has one b2_rasterize of its stream at ratio 1.0 and level 1.0.
        Returns (float32 signals back to back, ref_off int64[V+1])."""
        h = self.handle
        V = len(pcm_off) - 1
        if pcm_host is None:   # no video has samples: every detector signal is empty
            det, det_off = np.zeros(0, np.float32), np.zeros(V + 1, np.int64)
        elif self.auditok:
            det, det_off = h.vad_auditok(pcm_host, pcm_off, self.frame_rate, self.sample_rate, self.non_speech_label,
                                         chunk_samples=self.chunk_samples)
        else:
            det, det_off = h.vad_energy_zcr(pcm_host, pcm_off, self.frame_rate, self.sample_rate,
                                            self.non_speech_label, self.energy_threshold, self.z_lo, self.z_hi)
        if refs is None:
            return det.astype(np.float32), det_off
        is_subs, rs, re_, rk, roff = refs
        sub, sub_off = h.rasterize(rs, re_, rk, roff, [1.0], 1, False, self.sample_rate, self.start_seconds,
                                   levels=[1.0])
        parts = [sub[sub_off[v]: sub_off[v + 1]] if is_subs[v] else det[det_off[v]: det_off[v + 1]].astype(np.float32)
                 for v in range(V)]
        off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
        return (np.concatenate(parts) if parts else np.zeros(0, np.float32)), off

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
