"""ctypes binding of the C ABI in include/ffsubsync_b200.h.

There is deliberately NO CPU fallback: if the CUDA library is missing or no H100 is visible,
every compute entry point raises.  Build the library with ``python __graft_entry__.py``.
"""
import contextlib
import ctypes
import os
import threading
from typing import Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_lib", "libffsubsync_b200.so")

B2_HOST, B2_DEVICE = 0, 1
B2_DEVICE_RESIDENT = 2   # b2_sync_batch only: device inputs that nothing queued before the call still writes
B2_MAX_OFFSET_NONE = -(1 << 63)   # INT64_MIN: FFTAligner(max_offset_samples=None)
ALIGN_OK, ALIGN_EMPTY, ALIGN_ALL_MASKED, ALIGN_CAND_OVERFLOW = 0, 1, 2, 4
STATUS_NAMES = {0: "B2_OK", -1: "B2_ERR_BAD_ARG", -2: "B2_ERR_CUDA", -3: "B2_ERR_EMPTY_INPUT",
                -4: "B2_ERR_NO_ALIGNMENT", -5: "B2_ERR_NOMEM", -6: "B2_ERR_UNSUPPORTED"}

# every symbol declared in include/ffsubsync_b200.h (tests check the header against this list)
EXPORTS = [
    "b2_version", "b2_create", "b2_destroy", "b2_set_stream", "b2_synchronize", "b2_last_error",
    "b2_launch_count", "b2_vad_frames_per_window", "b2_vad_call_samples", "b2_vad_num_windows",
    "b2_vad_energy_zcr", "b2_rasterize_lengths", "b2_rasterize", "b2_blend_signals", "b2_first_last_nonzero",
    "b2_align_batch", "b2_reduce_ratios", "b2_sync_batch", "b2_synth_pcm", "b2_vad_stream_begin", "b2_vad_stream_push",
    "b2_vad_stream_windows", "b2_vad_stream_end", "b2_auditok_block_size", "b2_auditok_energy_floor",
    "b2_vad_auditok", "b2_capture_nominations", "b2_sync_tracks", "b2_sync_tracks_gss",
    "b2_sync_tracks_auditok", "b2_sync_tracks_subs", "b2_rasterize_pgs_lengths", "b2_rasterize_pgs",
    "b2_sync_tracks_pgs", "b2_capture_reference", "b2_sync_tracks_sig", "b2_apply_sync",
    "b2_sync_tracks_seg", "b2_speech_output", "b2_segment_length", "b2_ingest_begin", "b2_ingest_push",
    "b2_ingest_windows", "b2_ingest_sync_tracks", "b2_ingest_abort", "b2_ingest_segments", "b2_ingest_push_segments",
    "b2_ingest_drop_segment", "b2_ingest_sync_refs", "b2_split_tracks", "b2_split_tracks_wide", "b2_split_tracks_capped",
    "b2_split_tracks_directed", "b2_split_tracks_breaks", "b2_apply_split",
]
B2_DETECTOR_ENERGY_ZCR, B2_DETECTOR_AUDITOK = 0, 1   # b2_sync_tracks_subs: the detector of the audio videos
B2_BEST_K_BAD_SIGNAL = -2   # best_k of the tracks of a video whose stored signal leaves its domain (b2_sync_tracks_sig)
B2_BEST_K_NO_SPEECH = -3    # best_k of the tracks of a video whose sampled segments hold no speech (b2_sync_tracks_seg)
GSS_EVALS = 17   # evaluations of the golden-section search over [0.9, 1.1] with tolerance 1e-4


class NativeError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        self.status = status
        super().__init__("%s failed with %s%s" % (where, STATUS_NAMES.get(status, status),
                                                  (": " + detail) if detail else ""))


_lib = None
_lib_lock = threading.Lock()
_tls = threading.local()

_vp, _i32, _i64, _f32, _f64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_double


def load() -> ctypes.CDLL:
    """Load the shared library (no CUDA initialisation happens here)."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "ffsubsync_b200: CUDA library %s not found - build it with "
                "`python __graft_entry__.py` (there is no CPU fallback)" % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        lib.b2_version.restype = ctypes.c_int
        lib.b2_create.argtypes = [ctypes.c_int, ctypes.POINTER(_vp)]
        lib.b2_destroy.argtypes = [_vp]
        lib.b2_set_stream.argtypes = [_vp, _vp]
        lib.b2_synchronize.argtypes = [_vp]
        lib.b2_last_error.argtypes = [_vp]
        lib.b2_last_error.restype = ctypes.c_char_p
        lib.b2_launch_count.argtypes = [_vp]
        lib.b2_launch_count.restype = _i64
        lib.b2_vad_frames_per_window.argtypes = [ctypes.c_int, ctypes.c_int]
        lib.b2_vad_call_samples.argtypes = [ctypes.c_int, ctypes.c_int]
        lib.b2_vad_call_samples.restype = _i64
        lib.b2_vad_num_windows.argtypes = [_i64, ctypes.c_int, ctypes.c_int]
        lib.b2_vad_num_windows.restype = _i64
        lib.b2_vad_energy_zcr.argtypes = [_vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                          _f32, _i64, ctypes.c_int, ctypes.c_int, _vp, _vp, ctypes.c_int]
        lib.b2_rasterize_lengths.argtypes = [_vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int,
                                             ctypes.c_int, _vp]
        lib.b2_rasterize.argtypes = [_vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int,
                                     ctypes.c_int, _vp, ctypes.c_int, _f64, _vp, _vp, ctypes.c_int]
        lib.b2_first_last_nonzero.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, _vp, ctypes.c_int]
        lib.b2_blend_signals.argtypes = [_vp, _vp, _vp, _i64, ctypes.c_int, _f64, _f64, _vp, ctypes.c_int]
        lib.b2_align_batch.argtypes = [_vp, _vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, _i64,
                                       _vp, _vp, _vp, ctypes.c_int]
        lib.b2_reduce_ratios.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, _i64,
                                         _vp, _vp, _vp, ctypes.c_int]
        lib.b2_sync_batch.argtypes = [_vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _f32,
                                      _i64, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp, _vp,
                                      ctypes.c_int, _f64, _i64, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]
        lib.b2_sync_tracks.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                       _f32, _i64, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp, _vp,
                                       ctypes.c_int, _f64, _i64, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]
        lib.b2_sync_tracks_gss.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, _f32, _i64, ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp,
                                           _vp, ctypes.c_int, _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                           ctypes.c_int]
        lib.b2_sync_tracks_auditok.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_int, _f64, _f64, _f64, _i64, _f64, _i64, _vp, _vp, _vp,
                                               _vp, _vp, ctypes.c_int, _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp,
                                               _vp, ctypes.c_int]
        lib.b2_sync_tracks_subs.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_int, _f64, _i64, ctypes.c_int, ctypes.c_int, _f64, _f64, _i64,
                                            _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int,
                                            _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]
        lib.b2_rasterize_pgs_lengths.argtypes = [_vp, _vp, ctypes.c_int, ctypes.c_int, _vp]
        lib.b2_rasterize_pgs.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, _f64, _vp, _vp, ctypes.c_int]
        lib.b2_sync_tracks_pgs.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, _f64, _i64, ctypes.c_int, ctypes.c_int, _f64, _f64, _i64,
                                           _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                           _vp, ctypes.c_int, _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                           ctypes.c_int]
        lib.b2_sync_tracks_sig.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_int, _f64, _i64, ctypes.c_int, ctypes.c_int, _f64, _f64, _i64,
                                           _f64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                           _vp, _vp, _vp, _vp, ctypes.c_int, _f64, _i64, _vp, _vp, _vp, _vp, _vp,
                                           _vp, _vp, ctypes.c_int]
        lib.b2_sync_tracks_seg.argtypes = (lib.b2_sync_tracks_sig.argtypes[:30] + [ctypes.c_int] + [_vp] * 6
                                           + lib.b2_sync_tracks_sig.argtypes[30:])
        lib.b2_synth_pcm.argtypes = [_vp, _vp, _i64, ctypes.c_int, ctypes.c_uint32, _vp, ctypes.c_int]
        lib.b2_vad_stream_begin.argtypes = [_vp, ctypes.c_int, ctypes.c_int, _f32, _i64, ctypes.c_int,
                                            ctypes.c_int]
        lib.b2_vad_stream_push.argtypes = [_vp, _vp, _i64]
        lib.b2_vad_stream_windows.argtypes = [_vp]
        lib.b2_vad_stream_windows.restype = _i64
        lib.b2_vad_stream_end.argtypes = [_vp, _vp, _i64, ctypes.POINTER(_i64)]
        lib.b2_auditok_block_size.argtypes = [ctypes.c_int, ctypes.c_int]
        lib.b2_auditok_energy_floor.argtypes = [ctypes.c_int, _f64]
        lib.b2_auditok_energy_floor.restype = _i64
        lib.b2_vad_auditok.argtypes = [_vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _f64, _f64,
                                       _f64, _i64, _f64, _i64, _vp, _vp, ctypes.c_int]
        lib.b2_capture_nominations.argtypes = [_vp, _vp, _i64, _vp, _vp, _vp]
        lib.b2_capture_reference.argtypes = [_vp, _vp, _i64, _vp, _vp, _i64]
        lib.b2_speech_output.argtypes = [_vp, _vp, _i64, _vp, ctypes.c_int, _vp, ctypes.c_int]
        lib.b2_segment_length.argtypes = [_f64, ctypes.c_int]
        lib.b2_segment_length.restype = _i64
        lib.b2_apply_sync.argtypes = [_vp, _vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_int,
                                      ctypes.c_int, _f64, ctypes.c_int, _f64, _f64, _f64, ctypes.c_int, _f64,
                                      _vp, _vp, _vp, _vp, _vp, ctypes.c_int]
        lib.b2_ingest_begin.argtypes = [_vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, _f64, _i64,
                                        ctypes.c_int, ctypes.c_int, _f64, _f64, _i64, _f64, _i64, _vp]
        lib.b2_ingest_push.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp]
        lib.b2_ingest_windows.argtypes = [_vp, _vp]
        lib.b2_ingest_sync_tracks.argtypes = [_vp, _vp, ctypes.c_int, _vp, _vp, _vp, _vp, _vp, ctypes.c_int, _f64, _i64,
                                              _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]
        lib.b2_ingest_sync_refs.argtypes = [_vp] + [_vp] * 12 + lib.b2_ingest_sync_tracks.argtypes[1:]
        lib.b2_ingest_abort.argtypes = [_vp]
        lib.b2_ingest_segments.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp, _vp]
        lib.b2_ingest_push_segments.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp, _vp]
        lib.b2_ingest_drop_segment.argtypes = [_vp, ctypes.c_int, _i64]
        lib.b2_split_tracks.argtypes = [_vp, _vp, ctypes.c_int, _vp, ctypes.c_int, _vp, ctypes.c_int, _vp, _vp, _vp, _vp,
                                        _vp, ctypes.c_int, _f64, _i64, _f64, _vp, _vp, _vp, ctypes.c_int]
        lib.b2_split_tracks_wide.argtypes = lib.b2_split_tracks.argtypes
        lib.b2_split_tracks_capped.argtypes = (lib.b2_split_tracks.argtypes[:16] + [ctypes.c_int, _vp, _vp, _vp, _vp,
                                                                                    ctypes.c_int])
        lib.b2_split_tracks_directed.argtypes = (lib.b2_split_tracks.argtypes[:16] + [ctypes.c_int] +
                                                 lib.b2_split_tracks.argtypes[16:])
        lib.b2_split_tracks_breaks.argtypes = (lib.b2_split_tracks.argtypes[:16] + [_vp, ctypes.c_int, _vp, _vp, _vp,
                                                                                    _vp, ctypes.c_int])
        lib.b2_apply_split.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_int, _vp, _vp, _vp, ctypes.c_int, _f64, _vp, _vp,
                                       _vp, ctypes.c_int]
        _lib = lib
        return lib


def _ptr(a) -> Optional[int]:
    """Pointer of a numpy array (kept alive by the caller), an int device pointer, or None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    return a.ctypes.data


def _mask_width(max_offset_samples) -> int:
    """None -> B2_MAX_OFFSET_NONE; any Python int -> an int64 the library feeds to the reference's
    slice arithmetic (aligners.py:31-43).  Widths beyond +-2^62 behave like every width larger
    than the padded length, so clamping them keeps the result and avoids ctypes wrap-around."""
    if max_offset_samples is None:
        return B2_MAX_OFFSET_NONE
    lim = 1 << 62
    return max(-lim, min(lim, int(max_offset_samples)))


def _auditok_tokenizer(sample_rate: int, min_length=None, max_length=None, max_continuous_silence=None):
    """(min_length, max_length, max_continuous_silence) of the auditok tokenizer in blocks, None taking the
    reference's defaults (speech_transformers.py:126-131): 0.2 s, 5 s, 0.25 s."""
    return (float(0.2 * sample_rate if min_length is None else min_length),
            int(int(5 * sample_rate) if max_length is None else max_length),
            float(0.25 * sample_rate if max_continuous_silence is None else max_continuous_silence))


def _i64a(x) -> np.ndarray:
    return np.ascontiguousarray(x, dtype=np.int64)


class Handle:
    """One library handle = one CUDA stream + workspace.  Not thread-safe; see get_handle()."""

    def __init__(self, device: int = 0):
        self.lib = load()
        h = _vp()
        st = self.lib.b2_create(int(device), ctypes.byref(h))
        if st != 0:
            raise NativeError(st, "b2_create(device=%d)" % device,
                              "no usable sm_90 (H100) CUDA device; this package has no CPU path")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.b2_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, st: int, where: str):
        if st != 0:
            raise NativeError(st, where, self.lib.b2_last_error(self.h).decode("utf-8", "replace"))

    # -- plumbing ---------------------------------------------------------------------------
    def set_stream(self, cuda_stream: Optional[int]):
        """cuda_stream: a cudaStream_t handle as int (e.g. torch.cuda.Stream().cuda_stream);
        0 means the legacy default stream (torch's default), None gives the handle its own stream."""
        if cuda_stream is not None and int(cuda_stream) == 0:
            cuda_stream = 1  # cudaStreamLegacy: NULL would mean "own stream" in the C ABI
        self._check(self.lib.b2_set_stream(self.h, cuda_stream), "b2_set_stream")

    def synchronize(self):
        self._check(self.lib.b2_synchronize(self.h), "b2_synchronize")

    @property
    def launch_count(self) -> int:
        return int(self.lib.b2_launch_count(self.h))

    # -- VAD ----------------------------------------------------------------------------------
    def frames_per_window(self, frame_rate: int, sample_rate: int) -> int:
        return int(self.lib.b2_vad_frames_per_window(frame_rate, sample_rate))

    def energy_calls(self, pcm_off, frame_rate: int, sample_rate: int):
        """The energy / ZCR detector calls of the reference's chunk loop over B signals (b2_vad_call_samples samples
        each from every signal's start; one per signal where that is 0): (call_off [C+1], first [B+1]), signal b's
        calls first[b] .. first[b+1]-1.  b2_vad_energy_zcr over call_off writes each signal's frames back to back,
        signal b's from out_off[first[b]] on."""
        pcm_off = _i64a(pcm_off)
        call = int(self.lib.b2_vad_call_samples(frame_rate, sample_rate))
        if call <= 0:
            return pcm_off, np.arange(len(pcm_off), dtype=np.int64)
        parts = [np.arange(a, b, call, dtype=np.int64) for a, b in zip(pcm_off[:-1], pcm_off[1:])]
        first = np.concatenate([[0], np.cumsum([len(q) for q in parts])]).astype(np.int64)
        return np.concatenate(parts + [pcm_off[-1:]]).astype(np.int64), first

    def vad_energy_zcr(self, pcm, pcm_off, frame_rate: int, sample_rate: int, non_speech_label: float,
                       energy_threshold: int, z_lo: int = -1, z_hi: int = -1, out=None,
                       memspace: int = B2_HOST):
        """pcm: int16 numpy array (host) or device pointer; pcm_off: [B+1] sample offsets."""
        pcm_off = _i64a(pcm_off)
        B = len(pcm_off) - 1
        fpw = self.frames_per_window(frame_rate, sample_rate)
        if fpw <= 0:
            raise ValueError("bad frame_rate / sample_rate")
        nwin = (np.diff(pcm_off) + fpw - 1) // fpw
        out_off = np.concatenate([[0], np.cumsum(nwin)]).astype(np.int64)
        if memspace == B2_HOST:
            pcm = np.ascontiguousarray(pcm, dtype=np.int16)
            out = np.empty(int(out_off[-1]), dtype=np.float32)
        st = self.lib.b2_vad_energy_zcr(self.h, _ptr(pcm), _ptr(pcm_off), B, frame_rate, sample_rate,
                                        float(non_speech_label), int(energy_threshold), int(z_lo),
                                        int(z_hi), _ptr(out), _ptr(out_off), memspace)
        self._check(st, "b2_vad_energy_zcr")
        return out, out_off

    def vad_auditok(self, pcm, pcm_off, frame_rate: int, sample_rate: int, non_speech_label: float,
                    energy_threshold_db: float = 50.0, min_length: Optional[float] = None,
                    max_length: Optional[int] = None, max_continuous_silence: Optional[float] = None,
                    chunk_samples: int = 0, out=None, memspace: int = B2_HOST):
        """auditok detector over B signals (b2_vad_auditok); tokenizer defaults are the reference's
        (speech_transformers.py:126-131).  Returns (float64 per block, out_off[B+1])."""
        pcm_off = _i64a(pcm_off)
        B = len(pcm_off) - 1
        min_length, max_length, max_continuous_silence = _auditok_tokenizer(sample_rate, min_length, max_length,
                                                                            max_continuous_silence)
        out_off = self.auditok_out_off(pcm_off, frame_rate, sample_rate, chunk_samples)
        if memspace == B2_HOST:
            pcm = np.ascontiguousarray(pcm, dtype=np.int16)
            out = np.empty(int(out_off[-1]), dtype=np.float64)
        st = self.lib.b2_vad_auditok(self.h, _ptr(pcm), _ptr(pcm_off), B, frame_rate, sample_rate,
                                     float(non_speech_label), float(energy_threshold_db), float(min_length),
                                     int(max_length), float(max_continuous_silence), int(chunk_samples),
                                     _ptr(out), _ptr(out_off), memspace)
        self._check(st, "b2_vad_auditok")
        return out, out_off

    def auditok_out_off(self, pcm_off, frame_rate: int, sample_rate: int, chunk_samples: int) -> np.ndarray:
        """out_off [B+1] of the auditok detector over B signals cut into detector calls of chunk_samples samples
        (0: one call each): a signal has the sum over its chunks of ceil(chunk / block) blocks."""
        fpw = int(self.lib.b2_auditok_block_size(frame_rate, sample_rate))
        if fpw <= 0:
            raise ValueError("auditok detector: unsupported frame_rate=%r / sample_rate=%r" % (frame_rate, sample_rate))
        n = np.diff(_i64a(pcm_off))
        if chunk_samples > 0:
            nwin = n // chunk_samples * ((chunk_samples + fpw - 1) // fpw) + (n % chunk_samples + fpw - 1) // fpw
        else:
            nwin = (n + fpw - 1) // fpw
        return np.concatenate([[0], np.cumsum(nwin)]).astype(np.int64)

    # streaming detector (b2_vad_stream_*): push() returns before the chunk is processed
    def vad_stream_begin(self, frame_rate: int, sample_rate: int, non_speech_label: float,
                         energy_threshold: int, z_lo: int = -1, z_hi: int = -1) -> None:
        self._check(self.lib.b2_vad_stream_begin(self.h, frame_rate, sample_rate, float(non_speech_label),
                                                 int(energy_threshold), int(z_lo), int(z_hi)),
                    "b2_vad_stream_begin")

    def vad_stream_push(self, chunk) -> None:
        """chunk: bytes-like or uint8/int16 array (host); copied before the call returns."""
        if isinstance(chunk, np.ndarray):
            buf = np.ascontiguousarray(chunk)
            ptr, n = buf.ctypes.data, buf.nbytes
        else:
            buf = np.frombuffer(chunk, dtype=np.uint8)
            ptr, n = (buf.ctypes.data if len(buf) else None), len(buf)
        self._check(self.lib.b2_vad_stream_push(self.h, ptr, n), "b2_vad_stream_push")

    def vad_stream_end(self) -> np.ndarray:
        n = int(self.lib.b2_vad_stream_windows(self.h))
        out = np.empty(max(n, 0), dtype=np.float32)
        got = _i64(0)
        self._check(self.lib.b2_vad_stream_end(self.h, _ptr(out) if n > 0 else None, max(n, 0),
                                               ctypes.byref(got)), "b2_vad_stream_end")
        return out[: got.value]

    def synth_pcm(self, window_class, n_windows: int, fpw: int, seed: int, out=None,
                  memspace: int = B2_HOST):
        if memspace == B2_HOST:
            window_class = np.ascontiguousarray(window_class, dtype=np.uint8)
            n_windows = len(window_class)
            out = np.empty(n_windows * fpw, dtype=np.int16)
        st = self.lib.b2_synth_pcm(self.h, _ptr(window_class), int(n_windows), int(fpw),
                                   int(seed) & 0xFFFFFFFF, _ptr(out), memspace)
        self._check(st, "b2_synth_pcm")
        return out

    # -- subtitle side ------------------------------------------------------------------------
    def rasterize_lengths(self, cue_end_s, cue_off, ratios, K: int, per_pair: bool, sample_rate: int):
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        cue_off = _i64a(cue_off)
        ratios = np.ascontiguousarray(ratios, dtype=np.float64)
        B = len(cue_off) - 1
        lengths = np.empty(B * K, dtype=np.int64)
        st = self.lib.b2_rasterize_lengths(_ptr(cue_end_s), _ptr(cue_off), B, _ptr(ratios), K,
                                           int(per_pair), sample_rate, _ptr(lengths))
        if st != 0:
            raise NativeError(st, "b2_rasterize_lengths")
        return lengths

    def rasterize(self, cue_start_s, cue_end_s, cue_keep, cue_off, ratios, K: int, per_pair: bool,
                  sample_rate: int, start_seconds: float, levels=None, out=None, out_off=None,
                  memspace: int = B2_HOST):
        cue_start_s = np.ascontiguousarray(cue_start_s, dtype=np.float64)
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        cue_keep = None if cue_keep is None else np.ascontiguousarray(cue_keep, dtype=np.uint8)
        cue_off = _i64a(cue_off)
        ratios = np.ascontiguousarray(ratios, dtype=np.float64)
        levels = None if levels is None else np.ascontiguousarray(levels, dtype=np.float64)
        B = len(cue_off) - 1
        if out_off is None:
            lengths = self.rasterize_lengths(cue_end_s, cue_off, ratios, K, per_pair, sample_rate)
            out_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        out_off = _i64a(out_off)
        if memspace == B2_HOST:
            out = np.empty(int(out_off[-1]), dtype=np.float32)
        st = self.lib.b2_rasterize(self.h, _ptr(cue_start_s), _ptr(cue_end_s), _ptr(cue_keep),
                                   _ptr(cue_off), B, _ptr(ratios), K, int(per_pair), _ptr(levels),
                                   sample_rate, float(start_seconds), _ptr(out), _ptr(out_off), memspace)
        self._check(st, "b2_rasterize")
        return out, out_off

    def rasterize_pgs_lengths(self, end_s, off, sample_rate: int) -> np.ndarray:
        """Signal lengths int(max_end * sample_rate) + 2 of B PGS interval lists (b2_rasterize_pgs_lengths)."""
        end_s = np.ascontiguousarray(end_s, dtype=np.float64)
        off = _i64a(off)
        B = len(off) - 1
        lengths = np.empty(B, dtype=np.int64)
        st = self.lib.b2_rasterize_pgs_lengths(_ptr(end_s), _ptr(off), B, int(sample_rate), _ptr(lengths))
        if st != 0:
            raise NativeError(st, "b2_rasterize_pgs_lengths")
        return lengths

    def rasterize_pgs(self, start_s, end_s, off, sample_rate: int, start_seconds: float, out=None, out_off=None,
                      memspace: int = B2_HOST):
        """PGSSpeechTransformer.fit's signal of B interval lists (b2_rasterize_pgs): list b is
        start_s / end_s[off[b] .. off[b+1]].  Returns (float32 signals back to back, out_off int64[B+1])."""
        start_s = np.ascontiguousarray(start_s, dtype=np.float64)
        end_s = np.ascontiguousarray(end_s, dtype=np.float64)
        off = _i64a(off)
        B = len(off) - 1
        if out_off is None:
            out_off = np.concatenate([[0], np.cumsum(self.rasterize_pgs_lengths(end_s, off, sample_rate))])
        out_off = _i64a(out_off)
        if memspace == B2_HOST:
            out = np.empty(int(out_off[-1]), dtype=np.float32)
        st = self.lib.b2_rasterize_pgs(self.h, _ptr(start_s), _ptr(end_s), _ptr(off), B, int(sample_rate),
                                       float(start_seconds), _ptr(out), _ptr(out_off), memspace)
        self._check(st, "b2_rasterize_pgs")
        return out, out_off

    def blend_signals(self, a, b, mode: int, wa: float = 0.6, wb: float = 0.4, out=None, n=None,
                      memspace: int = B2_HOST):
        """mode 0 = min, 1 = max, 2 = wa*a + wb*b; host arrays are clipped to their common length."""
        if memspace == B2_HOST:
            n = min(len(a), len(b))
            a = np.ascontiguousarray(a[:n], dtype=np.float32)
            b = np.ascontiguousarray(b[:n], dtype=np.float32)
            out = np.empty(n, dtype=np.float32)
        st = self.lib.b2_blend_signals(self.h, _ptr(a), _ptr(b), int(n), int(mode), float(wa), float(wb),
                                       _ptr(out), memspace)
        self._check(st, "b2_blend_signals")
        return out

    def first_last_nonzero(self, sig, sig_off, memspace: int = B2_HOST, first=None, last=None):
        sig_off = _i64a(sig_off)
        n = len(sig_off) - 1
        if memspace == B2_HOST:
            sig = np.ascontiguousarray(sig, dtype=np.float32)
            first = np.empty(n, dtype=np.int64)
            last = np.empty(n, dtype=np.int64)
        st = self.lib.b2_first_last_nonzero(self.h, _ptr(sig), _ptr(sig_off), n, _ptr(first),
                                            _ptr(last), memspace)
        self._check(st, "b2_first_last_nonzero")
        return first, last

    # -- aligner ------------------------------------------------------------------------------
    def align_batch(self, ref, ref_off, sub, sub_off, B: int, K: int, max_offset_samples: Optional[int],
                    score=None, offset=None, status=None, memspace: int = B2_HOST):
        ref_off, sub_off = _i64a(ref_off), _i64a(sub_off)
        mos = _mask_width(max_offset_samples)
        if memspace == B2_HOST:
            ref = np.ascontiguousarray(ref, dtype=np.float32)
            sub = np.ascontiguousarray(sub, dtype=np.float32)
            score = np.empty(B * K, dtype=np.float64)
            offset = np.empty(B * K, dtype=np.int32)
            status = np.empty(B * K, dtype=np.int32)
        st = self.lib.b2_align_batch(self.h, _ptr(ref), _ptr(ref_off), _ptr(sub), _ptr(sub_off), B, K,
                                     mos, _ptr(score), _ptr(offset), _ptr(status), memspace)
        self._check(st, "b2_align_batch")
        return score, offset, status

    def reduce_ratios(self, score, offset, status, B: int, K: int, max_offset_samples: Optional[int],
                      best_score=None, best_offset=None, best_k=None, memspace: int = B2_HOST):
        mos = _mask_width(max_offset_samples)
        if memspace == B2_HOST:
            score = np.ascontiguousarray(score, dtype=np.float64)
            offset = np.ascontiguousarray(offset, dtype=np.int32)
            status = None if status is None else np.ascontiguousarray(status, dtype=np.int32)
            best_score = np.empty(B, dtype=np.float64)
            best_offset = np.empty(B, dtype=np.int32)
            best_k = np.empty(B, dtype=np.int32)
        st = self.lib.b2_reduce_ratios(self.h, _ptr(score), _ptr(offset), _ptr(status), B, K, mos,
                                       _ptr(best_score), _ptr(best_offset), _ptr(best_k), memspace)
        self._check(st, "b2_reduce_ratios")
        return best_score, best_offset, best_k

    def _sync(self, entry, pcm, pcm_off, track_video, detector_args, cue_start_s, cue_end_s, cue_keep, cue_off,
              ratios, start_seconds, max_offset_samples, outs, want_all, memspace, gss=None, want_evals=False):
        """The call of one b2_sync_* entry point: coerces the arrays, checks cue_off's length, allocates the host
        outputs (all_* with K + 1 columns with the search) and passes the arguments in the ABI's order.
        track_video None: b2_sync_batch (video b against track b).  detector_args: the entry point's arguments
        between sample_rate and the track cues.  outs: (best_score, best_offset, best_k, all_score, all_offset,
        gss_ratio, gss_evals).  gss: None for the entry points without the search's arguments, else whether it runs.
        Returns (best_score, best_offset, best_k, all_score, all_offset), plus (gss_ratio, gss_evals) with gss."""
        pcm_off, cue_off = _i64a(pcm_off), _i64a(cue_off)
        V = len(pcm_off) - 1
        videos = [V]
        if track_video is not None:
            track_video = np.ascontiguousarray(track_video, dtype=np.int32)
            T = len(track_video)
            if len(cue_off) != T + 1:
                raise NativeError(-1, entry, "cue_off has %d entries for %d tracks" % (len(cue_off), T))
            videos += [_ptr(track_video), T]
        else:
            T = V
        ratios = np.ascontiguousarray(ratios, dtype=np.float64)
        K = len(ratios)
        cue_start_s = np.ascontiguousarray(cue_start_s, dtype=np.float64)
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        cue_keep = None if cue_keep is None else np.ascontiguousarray(cue_keep, dtype=np.uint8)
        best_score, best_offset, best_k, all_score, all_offset, gss_ratio, gss_evals = outs
        if memspace == B2_HOST:
            pcm = None if pcm is None else np.ascontiguousarray(pcm, dtype=np.int16)
            best_score = np.empty(T, dtype=np.float64)
            best_offset = np.empty(T, dtype=np.int32)
            best_k = np.empty(T, dtype=np.int32)
            gss_ratio = np.empty(T, dtype=np.float64) if gss else None
            if want_all:
                cols = K + 1 if gss else K
                all_score = np.empty(T * cols, dtype=np.float64)
                all_offset = np.empty(T * cols, dtype=np.int32)
            gss_evals = np.empty(T * GSS_EVALS, dtype=np.float64) if gss and want_evals else None
        elif gss and gss_ratio is None:
            raise ValueError("%s with the search on device memory needs gss_ratio" % entry)
        search = [] if gss is None else [_ptr(gss_ratio) if gss else None, _ptr(gss_evals) if gss else None]
        st = getattr(self.lib, entry)(
            self.h, _ptr(pcm), _ptr(pcm_off), *videos, *detector_args, _ptr(cue_start_s), _ptr(cue_end_s),
            _ptr(cue_keep), _ptr(cue_off), _ptr(ratios), K, float(start_seconds), _mask_width(max_offset_samples),
            _ptr(best_score), _ptr(best_offset), _ptr(best_k), _ptr(all_score), _ptr(all_offset), *search, memspace)
        self._check(st, entry)
        res = (best_score, best_offset, best_k, all_score, all_offset)
        return res + (gss_ratio, gss_evals) if gss else res

    def sync_batch(self, pcm, pcm_off, frame_rate: int, sample_rate: int, non_speech_label: float,
                   energy_threshold: int, z_lo: int, z_hi: int, cue_start_s, cue_end_s, cue_keep,
                   cue_off, ratios, start_seconds: float, max_offset_samples: Optional[int],
                   best_score=None, best_offset=None, best_k=None, all_score=None, all_offset=None,
                   want_all: bool = False, memspace: int = B2_HOST):
        return self._sync("b2_sync_batch", pcm, pcm_off, None,
                          (frame_rate, sample_rate, float(non_speech_label), int(energy_threshold), int(z_lo),
                           int(z_hi)), cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds,
                          max_offset_samples, (best_score, best_offset, best_k, all_score, all_offset, None, None),
                          want_all, memspace)

    def sync_tracks(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int, non_speech_label: float,
                    energy_threshold: int, z_lo: int, z_hi: int, cue_start_s, cue_end_s, cue_keep,
                    cue_off, ratios, start_seconds: float, max_offset_samples: Optional[int],
                    best_score=None, best_offset=None, best_k=None, all_score=None, all_offset=None,
                    want_all: bool = False, memspace: int = B2_HOST):
        """sync_batch for T subtitle tracks over V videos (b2_sync_tracks): pcm_off [V+1] sample offsets,
        track_video [T] (non-decreasing video index of each track), cue_off [T+1].  Outputs per track:
        best_* [T], all_* [T*K]."""
        return self._sync("b2_sync_tracks", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, float(non_speech_label), int(energy_threshold), int(z_lo),
                           int(z_hi)), cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds,
                          max_offset_samples, (best_score, best_offset, best_k, all_score, all_offset, None, None),
                          want_all, memspace)

    def sync_tracks_gss(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int, non_speech_label: float,
                        energy_threshold: int, z_lo: int, z_hi: int, cue_start_s, cue_end_s, cue_keep,
                        cue_off, ratios, start_seconds: float, max_offset_samples: Optional[int],
                        best_score=None, best_offset=None, best_k=None, all_score=None, all_offset=None,
                        gss_ratio=None, gss_evals=None, want_all: bool = False, want_evals: bool = False,
                        memspace: int = B2_HOST):
        """sync_tracks with the golden-section search as candidate K (b2_sync_tracks_gss).  Outputs per track:
        best_* [T] (best_k == K: the search won), all_* [T*(K+1)] (column K: the search's candidate),
        gss_ratio [T] (NaN for an empty reference), gss_evals [T*17].  Raises NativeError with status
        B2_ERR_UNSUPPORTED (-6) outside the envelope of the device-driven rounds."""
        return self._sync("b2_sync_tracks_gss", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, float(non_speech_label), int(energy_threshold), int(z_lo),
                           int(z_hi)), cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds,
                          max_offset_samples, (best_score, best_offset, best_k, all_score, all_offset, gss_ratio,
                                               gss_evals), want_all, memspace, gss=True, want_evals=want_evals)

    def sync_tracks_auditok(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int,
                            non_speech_label: float, cue_start_s, cue_end_s, cue_keep, cue_off, ratios,
                            start_seconds: float, max_offset_samples: Optional[int], chunk_samples: int,
                            energy_threshold_db: float = 50.0, min_length: Optional[float] = None,
                            max_length: Optional[int] = None, max_continuous_silence: Optional[float] = None,
                            gss: bool = False, best_score=None, best_offset=None, best_k=None, all_score=None,
                            all_offset=None, gss_ratio=None, gss_evals=None, want_all: bool = False,
                            want_evals: bool = False, memspace: int = B2_HOST):
        """sync_tracks / sync_tracks_gss with the reference's auditok detector (b2_sync_tracks_auditok): each video
        is cut into detector calls of chunk_samples samples (0: one call).  Detector defaults as for vad_auditok.
        Returns (best_score, best_offset, best_k, all_score, all_offset), plus (gss_ratio, gss_evals) with
        gss=True (all_* then [T*(K+1)])."""
        tok = _auditok_tokenizer(sample_rate, min_length, max_length, max_continuous_silence)
        return self._sync("b2_sync_tracks_auditok", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, float(non_speech_label), float(energy_threshold_db), tok[0],
                           tok[1], tok[2], int(chunk_samples)), cue_start_s, cue_end_s, cue_keep, cue_off, ratios,
                          start_seconds, max_offset_samples,
                          (best_score, best_offset, best_k, all_score, all_offset, gss_ratio, gss_evals), want_all,
                          memspace, gss=bool(gss), want_evals=want_evals)

    def sync_tracks_subs(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int, non_speech_label: float,
                         ref_is_subs, ref_cue_start_s, ref_cue_end_s, ref_cue_keep, ref_cue_off, cue_start_s,
                         cue_end_s, cue_keep, cue_off, ratios, start_seconds: float,
                         max_offset_samples: Optional[int], detector: int = B2_DETECTOR_ENERGY_ZCR,
                         energy_threshold: int = 0, z_lo: int = -1, z_hi: int = -1, chunk_samples: int = 0,
                         energy_threshold_db: float = 50.0, min_length: Optional[float] = None,
                         max_length: Optional[int] = None, max_continuous_silence: Optional[float] = None,
                         gss: bool = False, best_score=None, best_offset=None, best_k=None, all_score=None,
                         all_offset=None, gss_ratio=None, gss_evals=None, want_all: bool = False,
                         want_evals: bool = False, memspace: int = B2_HOST):
        """sync_tracks / sync_tracks_auditok where the videos with ref_is_subs[v] != 0 take their subtitle stream
        (reference cues ref_cue_off[v] .. ref_cue_off[v+1], host arrays) as reference signal instead of the
        detector's output (b2_sync_tracks_subs).  pcm may be None when no video has samples.  detector:
        B2_DETECTOR_ENERGY_ZCR (energy_threshold, z_lo, z_hi) or B2_DETECTOR_AUDITOK (chunk_samples and the
        tokenizer arguments, defaults as for vad_auditok).  Returns (best_score, best_offset, best_k, all_score,
        all_offset), plus (gss_ratio, gss_evals) with gss=True (all_* then [T*(K+1)])."""
        V, T = len(pcm_off) - 1, len(track_video)
        ref_cue_off = _i64a(ref_cue_off)
        if len(cue_off) != T + 1 or len(ref_cue_off) != V + 1:
            raise NativeError(-1, "b2_sync_tracks_subs", "cue_off / ref_cue_off have %d / %d entries for %d tracks / "
                              "%d videos" % (len(cue_off), len(ref_cue_off), T, V))
        ref_is_subs = None if ref_is_subs is None else np.ascontiguousarray(ref_is_subs, dtype=np.uint8)
        if ref_is_subs is not None and len(ref_is_subs) != V:
            raise NativeError(-1, "b2_sync_tracks_subs", "ref_is_subs has %d entries for %d videos"
                              % (len(ref_is_subs), V))
        ref_cue_start_s = np.ascontiguousarray(ref_cue_start_s, dtype=np.float64)
        ref_cue_end_s = np.ascontiguousarray(ref_cue_end_s, dtype=np.float64)
        ref_cue_keep = None if ref_cue_keep is None else np.ascontiguousarray(ref_cue_keep, dtype=np.uint8)
        tok = _auditok_tokenizer(sample_rate, min_length, max_length, max_continuous_silence)
        return self._sync("b2_sync_tracks_subs", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, int(detector), float(non_speech_label), int(energy_threshold),
                           int(z_lo), int(z_hi), float(energy_threshold_db), tok[0], tok[1], tok[2], int(chunk_samples),
                           _ptr(ref_is_subs), _ptr(ref_cue_start_s), _ptr(ref_cue_end_s), _ptr(ref_cue_keep),
                           _ptr(ref_cue_off)), cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds,
                          max_offset_samples,
                          (best_score, best_offset, best_k, all_score, all_offset, gss_ratio, gss_evals), want_all,
                          memspace, gss=bool(gss), want_evals=want_evals)

    def sync_tracks_pgs(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int, non_speech_label: float,
                        ref_is_pgs, pgs_start_s, pgs_end_s, pgs_off, cue_start_s, cue_end_s, cue_keep, cue_off, ratios,
                        start_seconds: float, max_offset_samples: Optional[int], ref_is_subs=None,
                        ref_cue_start_s=None, ref_cue_end_s=None, ref_cue_keep=None, ref_cue_off=None,
                        detector: int = B2_DETECTOR_ENERGY_ZCR, energy_threshold: int = 0, z_lo: int = -1,
                        z_hi: int = -1, chunk_samples: int = 0, energy_threshold_db: float = 50.0,
                        min_length: Optional[float] = None, max_length: Optional[int] = None,
                        max_continuous_silence: Optional[float] = None, gss: bool = False, best_score=None,
                        best_offset=None, best_k=None, all_score=None, all_offset=None, gss_ratio=None, gss_evals=None,
                        want_all: bool = False, want_evals: bool = False, memspace: int = B2_HOST):
        """sync_tracks_subs where the videos with ref_is_pgs[v] != 0 take their PGS display intervals (pgs_off[v] ..
        pgs_off[v+1], host arrays) rasterised by PGSSpeechTransformer's rule as reference signal
        (b2_sync_tracks_pgs).  The text references (ref_is_subs, ref_cue_*) are optional.  Returns as
        sync_tracks_subs."""
        V, T = len(pcm_off) - 1, len(track_video)
        pgs_off = _i64a(pgs_off)
        if len(cue_off) != T + 1 or len(pgs_off) != V + 1:
            raise NativeError(-1, "b2_sync_tracks_pgs", "cue_off / pgs_off have %d / %d entries for %d tracks / "
                              "%d videos" % (len(cue_off), len(pgs_off), T, V))
        ref_is_pgs = None if ref_is_pgs is None else np.ascontiguousarray(ref_is_pgs, dtype=np.uint8)
        ref_is_subs = None if ref_is_subs is None else np.ascontiguousarray(ref_is_subs, dtype=np.uint8)
        for name, a in (("ref_is_pgs", ref_is_pgs), ("ref_is_subs", ref_is_subs)):
            if a is not None and len(a) != V:
                raise NativeError(-1, "b2_sync_tracks_pgs", "%s has %d entries for %d videos" % (name, len(a), V))
        if ref_cue_off is not None:
            ref_cue_off = _i64a(ref_cue_off)
            if len(ref_cue_off) != V + 1:
                raise NativeError(-1, "b2_sync_tracks_pgs", "ref_cue_off has %d entries for %d videos"
                                  % (len(ref_cue_off), V))
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
        pgs_start_s, pgs_end_s = f64(pgs_start_s), f64(pgs_end_s)
        ref_cue_start_s, ref_cue_end_s = f64(ref_cue_start_s), f64(ref_cue_end_s)
        ref_cue_keep = None if ref_cue_keep is None else np.ascontiguousarray(ref_cue_keep, dtype=np.uint8)
        tok = _auditok_tokenizer(sample_rate, min_length, max_length, max_continuous_silence)
        return self._sync("b2_sync_tracks_pgs", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, int(detector), float(non_speech_label), int(energy_threshold),
                           int(z_lo), int(z_hi), float(energy_threshold_db), tok[0], tok[1], tok[2], int(chunk_samples),
                           _ptr(ref_is_subs), _ptr(ref_cue_start_s), _ptr(ref_cue_end_s), _ptr(ref_cue_keep),
                           _ptr(ref_cue_off), _ptr(ref_is_pgs), _ptr(pgs_start_s), _ptr(pgs_end_s), _ptr(pgs_off)),
                          cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds, max_offset_samples,
                          (best_score, best_offset, best_k, all_score, all_offset, gss_ratio, gss_evals), want_all,
                          memspace, gss=bool(gss), want_evals=want_evals)

    def sync_tracks_sig(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int, non_speech_label: float,
                        ref_is_sig, x, sig_off, cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds: float,
                        max_offset_samples: Optional[int], ref_is_subs=None, ref_cue_start_s=None, ref_cue_end_s=None,
                        ref_cue_keep=None, ref_cue_off=None, ref_is_pgs=None, pgs_start_s=None, pgs_end_s=None,
                        pgs_off=None, detector: int = B2_DETECTOR_ENERGY_ZCR, energy_threshold: int = 0,
                        z_lo: int = -1, z_hi: int = -1, chunk_samples: int = 0, energy_threshold_db: float = 50.0,
                        min_length: Optional[float] = None, max_length: Optional[int] = None,
                        max_continuous_silence: Optional[float] = None, gss: bool = False, best_score=None,
                        best_offset=None, best_k=None, all_score=None, all_offset=None, gss_ratio=None, gss_evals=None,
                        want_all: bool = False, want_evals: bool = False, memspace: int = B2_HOST):
        """sync_tracks_pgs where the videos with ref_is_sig[v] != 0 take their serialized speech signal (the float64
        values x[sig_off[v] .. sig_off[v+1]), frame (float)(x < 1.0 ? non_speech_label : x)) as reference signal
        (b2_sync_tracks_sig).  x: a float64 numpy array under B2_HOST, a device pointer otherwise; sig_off: host.
        The text and PGS references are optional.  A video whose signal holds a value > 1.0 or NaN gets best_k =
        B2_BEST_K_BAD_SIGNAL on every track.  Returns as sync_tracks_subs."""
        V, T = len(pcm_off) - 1, len(track_video)
        sig_off = _i64a(sig_off)
        if len(cue_off) != T + 1 or len(sig_off) != V + 1:
            raise NativeError(-1, "b2_sync_tracks_sig", "cue_off / sig_off have %d / %d entries for %d tracks / "
                              "%d videos" % (len(cue_off), len(sig_off), T, V))
        u8 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint8)   # noqa: E731
        ref_is_sig, ref_is_pgs, ref_is_subs = u8(ref_is_sig), u8(ref_is_pgs), u8(ref_is_subs)
        for name, a in (("ref_is_sig", ref_is_sig), ("ref_is_pgs", ref_is_pgs), ("ref_is_subs", ref_is_subs)):
            if a is not None and len(a) != V:
                raise NativeError(-1, "b2_sync_tracks_sig", "%s has %d entries for %d videos" % (name, len(a), V))
        for name, off in (("ref_cue_off", ref_cue_off), ("pgs_off", pgs_off)):
            if off is not None and len(off) != V + 1:
                raise NativeError(-1, "b2_sync_tracks_sig", "%s has %d entries for %d videos" % (name, len(off), V))
        ref_cue_off = None if ref_cue_off is None else _i64a(ref_cue_off)
        pgs_off = None if pgs_off is None else _i64a(pgs_off)
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
        if x is not None and not isinstance(x, int):
            x = f64(x)
        pgs_start_s, pgs_end_s = f64(pgs_start_s), f64(pgs_end_s)
        ref_cue_start_s, ref_cue_end_s = f64(ref_cue_start_s), f64(ref_cue_end_s)
        ref_cue_keep = u8(ref_cue_keep)
        tok = _auditok_tokenizer(sample_rate, min_length, max_length, max_continuous_silence)
        return self._sync("b2_sync_tracks_sig", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, int(detector), float(non_speech_label), int(energy_threshold),
                           int(z_lo), int(z_hi), float(energy_threshold_db), tok[0], tok[1], tok[2], int(chunk_samples),
                           _ptr(ref_is_subs), _ptr(ref_cue_start_s), _ptr(ref_cue_end_s), _ptr(ref_cue_keep),
                           _ptr(ref_cue_off), _ptr(ref_is_pgs), _ptr(pgs_start_s), _ptr(pgs_end_s), _ptr(pgs_off),
                           _ptr(ref_is_sig), _ptr(x), _ptr(sig_off)),
                          cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds, max_offset_samples,
                          (best_score, best_offset, best_k, all_score, all_offset, gss_ratio, gss_evals), want_all,
                          memspace, gss=bool(gss), want_evals=want_evals)

    def sync_tracks_seg(self, pcm, pcm_off, track_video, frame_rate: int, sample_rate: int, non_speech_label: float,
                        seg_video, seg_total, seg_off, seg_start, seg_lo, seg_hi, cue_start_s, cue_end_s, cue_keep,
                        cue_off, ratios, start_seconds: float, max_offset_samples: Optional[int], ref_is_sig=None, x=None,
                        sig_off=None, ref_is_subs=None, ref_cue_start_s=None, ref_cue_end_s=None, ref_cue_keep=None,
                        ref_cue_off=None, ref_is_pgs=None, pgs_start_s=None, pgs_end_s=None, pgs_off=None,
                        detector: int = B2_DETECTOR_ENERGY_ZCR, energy_threshold: int = 0, z_lo: int = -1,
                        z_hi: int = -1, chunk_samples: int = 0, energy_threshold_db: float = 50.0,
                        min_length: Optional[float] = None, max_length: Optional[int] = None,
                        max_continuous_silence: Optional[float] = None, gss: bool = False, best_score=None,
                        best_offset=None, best_k=None, all_score=None, all_offset=None, gss_ratio=None, gss_evals=None,
                        want_all: bool = False, want_evals: bool = False, memspace: int = B2_HOST):
        """sync_tracks_sig where the P videos seg_video [P] (increasing) take MultiSegmentVideoSpeechTransformer.fit's
        sparse reference of their sampled segments (b2_sync_tracks_seg): video seg_video[i] has the probed duration
        seg_total[i] seconds and the segments seg_off[i] .. seg_off[i+1]-1, segment j starting at seg_start[j] whole
        seconds with the samples pcm_off[v] + seg_lo[j] .. pcm_off[v] + seg_hi[j] (host arrays).  The signal, text and
        PGS references are optional.  A video without speech in its segments gets best_k = B2_BEST_K_NO_SPEECH on
        every track.  Returns as sync_tracks_subs."""
        V, T = len(pcm_off) - 1, len(track_video)
        seg_video = np.ascontiguousarray(seg_video, dtype=np.int32)
        seg_total = np.ascontiguousarray(seg_total, dtype=np.float64)
        seg_off = _i64a(seg_off)
        P = len(seg_video)
        if len(cue_off) != T + 1 or len(seg_off) != P + 1 or len(seg_total) != P:
            raise NativeError(-1, "b2_sync_tracks_seg", "cue_off / seg_off / seg_total have %d / %d / %d entries for "
                              "%d tracks / %d segment videos" % (len(cue_off), len(seg_off), len(seg_total), T, P))
        seg_start, seg_lo, seg_hi = (_i64a(a) for a in (seg_start, seg_lo, seg_hi))
        if not (len(seg_start) == len(seg_lo) == len(seg_hi) >= (seg_off[-1] if P else 0)):
            raise NativeError(-1, "b2_sync_tracks_seg", "seg_start / seg_lo / seg_hi have %d / %d / %d entries for %d "
                              "segments" % (len(seg_start), len(seg_lo), len(seg_hi), int(seg_off[-1]) if P else 0))
        u8 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint8)   # noqa: E731
        ref_is_sig, ref_is_pgs, ref_is_subs = u8(ref_is_sig), u8(ref_is_pgs), u8(ref_is_subs)
        for name, a in (("ref_is_sig", ref_is_sig), ("ref_is_pgs", ref_is_pgs), ("ref_is_subs", ref_is_subs)):
            if a is not None and len(a) != V:
                raise NativeError(-1, "b2_sync_tracks_seg", "%s has %d entries for %d videos" % (name, len(a), V))
        for name, off in (("ref_cue_off", ref_cue_off), ("pgs_off", pgs_off), ("sig_off", sig_off)):
            if off is not None and len(off) != V + 1:
                raise NativeError(-1, "b2_sync_tracks_seg", "%s has %d entries for %d videos" % (name, len(off), V))
        ref_cue_off, pgs_off, sig_off = (None if a is None else _i64a(a) for a in (ref_cue_off, pgs_off, sig_off))
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
        if x is not None and not isinstance(x, int):
            x = f64(x)
        pgs_start_s, pgs_end_s = f64(pgs_start_s), f64(pgs_end_s)
        ref_cue_start_s, ref_cue_end_s = f64(ref_cue_start_s), f64(ref_cue_end_s)
        ref_cue_keep = u8(ref_cue_keep)
        tok = _auditok_tokenizer(sample_rate, min_length, max_length, max_continuous_silence)
        return self._sync("b2_sync_tracks_seg", pcm, pcm_off, track_video,
                          (frame_rate, sample_rate, int(detector), float(non_speech_label), int(energy_threshold),
                           int(z_lo), int(z_hi), float(energy_threshold_db), tok[0], tok[1], tok[2], int(chunk_samples),
                           _ptr(ref_is_subs), _ptr(ref_cue_start_s), _ptr(ref_cue_end_s), _ptr(ref_cue_keep),
                           _ptr(ref_cue_off), _ptr(ref_is_pgs), _ptr(pgs_start_s), _ptr(pgs_end_s), _ptr(pgs_off),
                           _ptr(ref_is_sig), _ptr(x), _ptr(sig_off), P, _ptr(seg_video), _ptr(seg_total),
                           _ptr(seg_off), _ptr(seg_start), _ptr(seg_lo), _ptr(seg_hi)),
                          cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds, max_offset_samples,
                          (best_score, best_offset, best_k, all_score, all_offset, gss_ratio, gss_evals), want_all,
                          memspace, gss=bool(gss), want_evals=want_evals)

    # batched ingest session (b2_ingest_*): push() returns before the chunks are processed
    def ingest_begin(self, V: int, frame_rate: int, sample_rate: int, non_speech_label: float,
                     detector: int = B2_DETECTOR_ENERGY_ZCR, energy_threshold: int = 0, z_lo: int = -1, z_hi: int = -1,
                     chunk_samples: int = 0, energy_threshold_db: float = 50.0, min_length: Optional[float] = None,
                     max_length: Optional[int] = None, max_continuous_silence: Optional[float] = None,
                     expect_samples=None) -> None:
        """Open a session for V videos (b2_ingest_begin); detector arguments as for sync_tracks_subs, expect_samples
        [V] a sizing hint (or None)."""
        tok = _auditok_tokenizer(sample_rate, min_length, max_length, max_continuous_silence)
        expect = None if expect_samples is None else _i64a(expect_samples)
        if expect is not None and len(expect) != V:
            raise NativeError(-1, "b2_ingest_begin", "expect_samples has %d entries for %d videos" % (len(expect), V))
        self._check(self.lib.b2_ingest_begin(self.h, int(V), frame_rate, sample_rate, int(detector),
                                             float(non_speech_label), int(energy_threshold), int(z_lo), int(z_hi),
                                             float(energy_threshold_db), tok[0], tok[1], tok[2], int(chunk_samples),
                                             _ptr(expect)), "b2_ingest_begin")
        self._ingest_V = int(V)

    def ingest_segments(self, seg_video, seg_total, seg_off, seg_start) -> None:
        """Declare the session's segment videos (b2_ingest_segments): segment_table's arrays without seg_lo / seg_hi."""
        video = np.ascontiguousarray(seg_video, dtype=np.int32)
        total = np.ascontiguousarray(seg_total, dtype=np.float64)
        off = _i64a(seg_off)
        start = _i64a(seg_start)
        if len(total) != len(video) or len(off) != len(video) + 1:
            raise NativeError(-1, "b2_ingest_segments", "%d totals and %d offsets for %d segment videos"
                              % (len(total), len(off), len(video)))
        self._check(self.lib.b2_ingest_segments(self.h, len(video), _ptr(video), _ptr(total), _ptr(off), _ptr(start)),
                    "b2_ingest_segments")

    def ingest_drop_segment(self, video: int, segment: int) -> None:
        self._check(self.lib.b2_ingest_drop_segment(self.h, int(video), int(segment)), "b2_ingest_drop_segment")

    def ingest_push(self, videos, chunks, segments=None) -> None:
        """Append chunks[i] (bytes-like, uint8 or int16 array) to video videos[i], in order (b2_ingest_push), or with
        ``segments`` to its segment segments[i] (b2_ingest_push_segments).  The library has copied them when this
        returns."""
        bufs = []
        for c in chunks:
            if isinstance(c, np.ndarray):
                bufs.append(np.ascontiguousarray(c).view(np.uint8).reshape(-1))
            else:
                bufs.append(np.frombuffer(c, dtype=np.uint8))
        n = len(bufs)
        video = np.ascontiguousarray(videos, dtype=np.int32)
        if len(video) != n:
            raise NativeError(-1, "b2_ingest_push", "%d videos for %d chunks" % (len(video), n))
        ptrs = (ctypes.c_void_p * max(n, 1))(*[b.ctypes.data if len(b) else None for b in bufs])
        sizes = np.array([len(b) for b in bufs], dtype=np.int64)
        if segments is None:
            self._check(self.lib.b2_ingest_push(self.h, n, _ptr(video), ptrs, _ptr(sizes)), "b2_ingest_push")
            return
        seg = _i64a(segments)
        if len(seg) != n:
            raise NativeError(-1, "b2_ingest_push_segments", "%d segments for %d chunks" % (len(seg), n))
        self._check(self.lib.b2_ingest_push_segments(self.h, n, _ptr(video), _ptr(seg), ptrs, _ptr(sizes)),
                    "b2_ingest_push_segments")

    def ingest_windows(self) -> np.ndarray:
        out = np.zeros(max(getattr(self, "_ingest_V", 0), 1), dtype=np.int64)
        self._check(self.lib.b2_ingest_windows(self.h, _ptr(out)), "b2_ingest_windows")
        return out[: getattr(self, "_ingest_V", 0)]

    def ingest_abort(self) -> None:
        self._check(self.lib.b2_ingest_abort(self.h), "b2_ingest_abort")

    def ingest_sync_tracks(self, track_video, cue_start_s, cue_end_s, cue_keep, cue_off, ratios, start_seconds: float,
                           max_offset_samples: Optional[int], gss: bool = False, best_score=None, best_offset=None,
                           best_k=None, all_score=None, all_offset=None, gss_ratio=None, gss_evals=None,
                           want_all: bool = False, want_evals: bool = False, memspace: int = B2_HOST,
                           ref_is_subs=None, ref_cue_start_s=None, ref_cue_end_s=None, ref_cue_keep=None,
                           ref_cue_off=None, ref_is_pgs=None, pgs_start_s=None, pgs_end_s=None, pgs_off=None,
                           ref_is_sig=None, x=None, sig_off=None):
        """Flush, sync the tracks against the session's references and close it (b2_ingest_sync_tracks).  Outputs as
        for sync_tracks / sync_tracks_gss (memspace B2_HOST allocates them; B2_DEVICE takes device pointers).
        The reference tables of sync_tracks_sig (text streams, PGS intervals, stored signals; x a float64 numpy array
        under B2_HOST, a device pointer otherwise) give videos without pushes their references
        (b2_ingest_sync_refs, called when any table is given).
        Returns (best_score, best_offset, best_k, all_score, all_offset), plus (gss_ratio, gss_evals) with gss."""
        track_video = np.ascontiguousarray(track_video, dtype=np.int32)
        cue_off = _i64a(cue_off)
        T = len(track_video)
        V = getattr(self, "_ingest_V", 0)
        tables = any(a is not None for a in (ref_is_subs, ref_cue_off, ref_is_pgs, pgs_off, ref_is_sig, sig_off))
        name = "b2_ingest_sync_refs" if tables else "b2_ingest_sync_tracks"
        if len(cue_off) != T + 1:
            self.ingest_abort()
            raise NativeError(-1, name, "cue_off has %d entries for %d tracks" % (len(cue_off), T))
        u8 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.uint8)   # noqa: E731
        f64 = lambda a: None if a is None else np.ascontiguousarray(a, dtype=np.float64)   # noqa: E731
        ref_is_subs, ref_is_pgs, ref_is_sig = u8(ref_is_subs), u8(ref_is_pgs), u8(ref_is_sig)
        ref_cue_off, pgs_off, sig_off = (None if a is None else _i64a(a) for a in (ref_cue_off, pgs_off, sig_off))
        for what, a, n in (("ref_is_subs", ref_is_subs, V), ("ref_is_pgs", ref_is_pgs, V), ("ref_is_sig", ref_is_sig, V),
                           ("ref_cue_off", ref_cue_off, V + 1), ("pgs_off", pgs_off, V + 1), ("sig_off", sig_off, V + 1)):
            if a is not None and len(a) != n:
                self.ingest_abort()
                raise NativeError(-1, name, "%s has %d entries for %d videos" % (what, len(a), V))
        ref_cue_start_s, ref_cue_end_s, pgs_start_s, pgs_end_s = (f64(a) for a in (ref_cue_start_s, ref_cue_end_s,
                                                                                   pgs_start_s, pgs_end_s))
        ref_cue_keep = u8(ref_cue_keep)
        if x is not None and not isinstance(x, int):
            x = f64(x)
        ratios = np.ascontiguousarray(ratios, dtype=np.float64)
        K = len(ratios)
        cue_start_s = np.ascontiguousarray(cue_start_s, dtype=np.float64)
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        cue_keep = None if cue_keep is None else np.ascontiguousarray(cue_keep, dtype=np.uint8)
        if memspace == B2_HOST:
            best_score = np.empty(T, dtype=np.float64)
            best_offset = np.empty(T, dtype=np.int32)
            best_k = np.empty(T, dtype=np.int32)
            gss_ratio = np.empty(T, dtype=np.float64) if gss else None
            if want_all:
                cols = K + 1 if gss else K
                all_score = np.empty(T * cols, dtype=np.float64)
                all_offset = np.empty(T * cols, dtype=np.int32)
            gss_evals = np.empty(T * GSS_EVALS, dtype=np.float64) if gss and want_evals else None
        elif gss and gss_ratio is None:
            self.ingest_abort()
            raise ValueError("%s with the search on device memory needs gss_ratio" % name)
        args = (_ptr(track_video), T, _ptr(cue_start_s), _ptr(cue_end_s), _ptr(cue_keep), _ptr(cue_off), _ptr(ratios),
                K, float(start_seconds), _mask_width(max_offset_samples), _ptr(best_score), _ptr(best_offset),
                _ptr(best_k), _ptr(all_score), _ptr(all_offset), _ptr(gss_ratio) if gss else None,
                _ptr(gss_evals) if gss else None, memspace)
        if tables:
            st = self.lib.b2_ingest_sync_refs(
                self.h, _ptr(ref_is_subs), _ptr(ref_cue_start_s), _ptr(ref_cue_end_s), _ptr(ref_cue_keep),
                _ptr(ref_cue_off), _ptr(ref_is_pgs), _ptr(pgs_start_s), _ptr(pgs_end_s), _ptr(pgs_off),
                _ptr(ref_is_sig), _ptr(x), _ptr(sig_off), *args)
        else:
            st = self.lib.b2_ingest_sync_tracks(self.h, *args)
        self._check(st, name)
        res = (best_score, best_offset, best_k, all_score, all_offset)
        return res + (gss_ratio, gss_evals) if gss else res

    def segment_length(self, total_seconds: float, sample_rate: int) -> int:
        """The reference length int(total_seconds * sample_rate) + 2 of a segment video (b2_segment_length); raises
        ValueError where the batched calls refuse the duration."""
        n = int(self.lib.b2_segment_length(float(total_seconds), int(sample_rate)))
        if n < 0:
            raise ValueError("seg_total %r is not finite, too large, or gives a negative signal length" % total_seconds)
        return n

    def speech_output(self, speech, capacity: int, videos, speech_off, memspace: int = B2_DEVICE) -> None:
        """Set (speech: a device pointer under B2_DEVICE, a float64 numpy array under B2_HOST) or clear (speech None)
        the speech output of the batched sync calls (b2_speech_output): each later call writes the reference signal
        of every video of ``videos`` (increasing) as float64 into speech and fills ``speech_off`` (int64 numpy array,
        len(videos) + 1, kept alive by the caller).  Enqueues nothing."""
        if speech is None:
            self._check(self.lib.b2_speech_output(self.h, None, 0, None, 0, None, 0), "b2_speech_output")
            return
        self._speech_videos = np.ascontiguousarray(videos, dtype=np.int32)
        self._check(self.lib.b2_speech_output(self.h, _ptr(speech), int(capacity), _ptr(self._speech_videos),
                                              len(self._speech_videos), _ptr(speech_off), int(memspace)),
                    "b2_speech_output")

    # -- diagnostics (tests) --------------------------------------------------------------------
    def apply_sync(self, best_score, best_offset, best_k, gss_ratio, cue_start_s, cue_end_s, cue_off, ratios,
                   sample_rate: int, apply_offset_seconds: float = 0.0, gate: bool = False, min_score: float = 0.0,
                   quality_max_offset_seconds: float = 30.0, max_framerate_deviation: float = 0.1,
                   suppress: Optional[float] = None, outs=None, memspace: int = B2_HOST):
        """b2_apply_sync over the T = len(cue_off) - 1 tracks of a finished sync call.  best_* / gss_ratio (None: no
        search) are that call's outputs in memspace; cue times, cue_off and ratios are host arrays.  B2_HOST: returns
        numpy (synced_start_us, synced_end_us, offset_seconds, scale, status).  B2_DEVICE: outs holds those five
        device pointers in that order; enqueued on the handle's stream, returns outs."""
        cue_off = _i64a(cue_off)
        T = len(cue_off) - 1
        if T < 0:
            raise NativeError(-1, "b2_apply_sync", "cue_off needs at least one entry")
        ratios = np.ascontiguousarray(ratios, dtype=np.float64)
        cue_start_s = np.ascontiguousarray(cue_start_s, dtype=np.float64)
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        if memspace == B2_HOST:
            best_score = np.ascontiguousarray(best_score, dtype=np.float64)
            best_offset = np.ascontiguousarray(best_offset, dtype=np.int32)
            best_k = np.ascontiguousarray(best_k, dtype=np.int32)
            gss_ratio = None if gss_ratio is None else np.ascontiguousarray(gss_ratio, dtype=np.float64)
            n = int(cue_off[-1]) if T else 0
            outs = (np.zeros(n, np.int64), np.zeros(n, np.int64), np.empty(T, np.float64), np.empty(T, np.float64),
                    np.empty(T, np.int32))
        st = self.lib.b2_apply_sync(
            self.h, _ptr(best_score), _ptr(best_offset), _ptr(best_k), _ptr(gss_ratio), T, _ptr(cue_start_s),
            _ptr(cue_end_s), _ptr(cue_off), _ptr(ratios), len(ratios), int(sample_rate), float(apply_offset_seconds),
            int(bool(gate)), float(min_score), float(quality_max_offset_seconds), float(max_framerate_deviation),
            int(suppress is not None), 0.0 if suppress is None else float(suppress), *[_ptr(o) for o in outs],
            memspace)
        self._check(st, "b2_apply_sync")
        return outs

    def split_tracks(self, ref, ref_is_f64: bool, ref_off, track_video, cue_start_s, cue_end_s, cue_keep, cue_off,
                     ratio, sample_rate: int, start_seconds: float, max_offset_samples, split_penalty: float,
                     outs=None, memspace: int = B2_HOST):
        """b2_split_tracks: per-segment offsets of the T = len(cue_off) - 1 tracks.  ref (float64 when ref_is_f64, else
        float32) follows memspace; everything else but the outputs is host metadata (ratio: NaN skips a track).
        B2_HOST: returns numpy (cue_offset i32 [cues], n_segments i32 [T], split_score f64 [T]).  B2_DEVICE: outs holds
        those three device pointers in that order; enqueued on the handle's stream, returns outs."""
        return self._split_tracks("b2_split_tracks", ref, ref_is_f64, ref_off, track_video, cue_start_s, cue_end_s,
                                  cue_keep, cue_off, ratio, sample_rate, start_seconds, max_offset_samples,
                                  split_penalty, outs, memspace)

    def split_tracks_wide(self, ref, ref_is_f64: bool, ref_off, track_video, cue_start_s, cue_end_s, cue_keep, cue_off,
                          ratio, sample_rate: int, start_seconds: float, max_offset_samples, split_penalty: float,
                          outs=None, memspace: int = B2_HOST):
        """b2_split_tracks_wide: split_tracks with windows of up to 16384 offsets per CTA of the widest thread-block
        cluster the device co-schedules (262144 offsets at 16 CTAs); same arguments and results."""
        return self._split_tracks("b2_split_tracks_wide", ref, ref_is_f64, ref_off, track_video, cue_start_s,
                                  cue_end_s, cue_keep, cue_off, ratio, sample_rate, start_seconds, max_offset_samples,
                                  split_penalty, outs, memspace)

    def split_tracks_capped(self, ref, ref_is_f64: bool, ref_off, track_video, cue_start_s, cue_end_s, cue_keep,
                            cue_off, ratio, sample_rate: int, start_seconds: float, max_offset_samples,
                            split_penalty: float, max_segments: int, outs=None, memspace: int = B2_HOST):
        """b2_split_tracks_capped: split_tracks_wide with at most max_segments segments per track.  B2_HOST: returns
        numpy (cue_offset i32 [cues], n_segments i32 [T], split_score f64 [T], split_profile f64 [T, max_segments]).
        B2_DEVICE: outs holds those four device pointers in that order; enqueued on the handle's stream, returns outs."""
        return self._split_tracks("b2_split_tracks_capped", ref, ref_is_f64, ref_off, track_video, cue_start_s,
                                  cue_end_s, cue_keep, cue_off, ratio, sample_rate, start_seconds, max_offset_samples,
                                  split_penalty, outs, memspace, max_segments=max_segments)

    def split_tracks_directed(self, ref, ref_is_f64: bool, ref_off, track_video, cue_start_s, cue_end_s, cue_keep,
                              cue_off, ratio, sample_rate: int, start_seconds: float, max_offset_samples,
                              split_penalty: float, direction: int, outs=None, memspace: int = B2_HOST):
        """b2_split_tracks_directed: split_tracks_wide with segment offsets that only grow (direction +1: ad breaks,
        an intermission) or only shrink (-1: a cut video, a pruned recap) along the track; same results."""
        return self._split_tracks("b2_split_tracks_directed", ref, ref_is_f64, ref_off, track_video, cue_start_s,
                                  cue_end_s, cue_keep, cue_off, ratio, sample_rate, start_seconds, max_offset_samples,
                                  split_penalty, outs, memspace, direction=direction)

    def split_tracks_breaks(self, ref, ref_is_f64: bool, ref_off, track_video, cue_start_s, cue_end_s, cue_keep,
                            cue_off, ratio, sample_rate: int, start_seconds: float, max_offset_samples,
                            split_penalty: float, breaks, outs=None, memspace: int = B2_HOST):
        """b2_split_tracks_breaks: split_tracks_wide along the stated breaks (a sequence of +1 / -1, the i-th break of a
        path moving the offset that way).  B2_HOST: returns numpy (cue_offset i32 [cues], n_segments i32 [T],
        split_score f64 [T], split_profile f64 [T, len(breaks) + 1]).  B2_DEVICE: outs holds those four device pointers
        in that order; enqueued on the handle's stream, returns outs."""
        return self._split_tracks("b2_split_tracks_breaks", ref, ref_is_f64, ref_off, track_video, cue_start_s,
                                  cue_end_s, cue_keep, cue_off, ratio, sample_rate, start_seconds, max_offset_samples,
                                  split_penalty, outs, memspace, breaks=breaks)

    def _split_tracks(self, name, ref, ref_is_f64, ref_off, track_video, cue_start_s, cue_end_s, cue_keep, cue_off,
                      ratio, sample_rate, start_seconds, max_offset_samples, split_penalty, outs, memspace,
                      max_segments=None, direction=None, breaks=None):
        ref_off, cue_off = _i64a(ref_off), _i64a(cue_off)
        V, T = len(ref_off) - 1, len(cue_off) - 1
        track_video = np.ascontiguousarray(track_video, dtype=np.int32)
        ratio = np.ascontiguousarray(ratio, dtype=np.float64)
        cue_start_s = np.ascontiguousarray(cue_start_s, dtype=np.float64)
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        keep = None if cue_keep is None else np.ascontiguousarray(cue_keep, dtype=np.uint8)
        if memspace == B2_HOST:
            ref = np.ascontiguousarray(ref, dtype=np.float64 if ref_is_f64 else np.float32)
            n = int(cue_off[-1]) if T >= 0 else 0
            outs = (np.zeros(n, np.int32), np.zeros(max(T, 0), np.int32), np.zeros(max(T, 0), np.float64))
            if max_segments is not None:
                outs += (np.zeros((max(T, 0), max(int(max_segments), 1)), np.float64),)
            if breaks is not None:
                outs += (np.zeros((max(T, 0), len(breaks) + 1), np.float64),)
        cap = () if max_segments is None else (int(max_segments),)
        if direction is not None:
            cap += (int(direction),)
        if breaks is not None:
            brk = np.ascontiguousarray(breaks, dtype=np.int32)
            cap += (_ptr(brk), len(brk))
        st = getattr(self.lib, name)(
            self.h, _ptr(ref), int(bool(ref_is_f64)), _ptr(ref_off), V, _ptr(track_video), T, _ptr(cue_start_s),
            _ptr(cue_end_s), _ptr(keep), _ptr(cue_off), _ptr(ratio), int(sample_rate), float(start_seconds),
            _mask_width(max_offset_samples), float(split_penalty), *cap, *[_ptr(o) for o in outs], memspace)
        self._check(st, name)
        return outs

    def apply_split(self, ratio, n_segments, cue_offset, cue_start_s, cue_end_s, cue_off, sample_rate: int,
                    apply_offset_seconds: float = 0.0, outs=None, memspace: int = B2_HOST):
        """b2_apply_split: the synced cue times with each cue's own offset.  n_segments / cue_offset follow memspace;
        ratio and the cue tables are host arrays.  B2_HOST: returns numpy (synced_start_us, synced_end_us, status).
        B2_DEVICE: outs holds those three device pointers; enqueued on the handle's stream, returns outs."""
        cue_off = _i64a(cue_off)
        T = len(cue_off) - 1
        ratio = np.ascontiguousarray(ratio, dtype=np.float64)
        cue_start_s = np.ascontiguousarray(cue_start_s, dtype=np.float64)
        cue_end_s = np.ascontiguousarray(cue_end_s, dtype=np.float64)
        if memspace == B2_HOST:
            n_segments = np.ascontiguousarray(n_segments, dtype=np.int32)
            cue_offset = np.ascontiguousarray(cue_offset, dtype=np.int32)
            n = int(cue_off[-1]) if T >= 0 else 0
            outs = (np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(T, 0), np.int32))
        st = self.lib.b2_apply_split(self.h, _ptr(ratio), _ptr(n_segments), _ptr(cue_offset), T, _ptr(cue_start_s),
                                     _ptr(cue_end_s), _ptr(cue_off), int(sample_rate), float(apply_offset_seconds),
                                     *[_ptr(o) for o in outs], memspace)
        self._check(st, "b2_apply_split")
        return outs

    @contextlib.contextmanager
    def capture_nominations(self, n_jobs: int, stride: int):
        """While the block runs, the aligner calls on this handle copy their nomination stage (fp32
        window scores, fp32 maximum and tau, candidate count) for jobs 0 .. n_jobs-1 into device
        arrays (b2_capture_nominations).  Yields a dict that holds numpy arrays once the block has
        exited: win [n_jobs, 2] int64, stat [n_jobs, 2] float32, cand [n_jobs] int32 and
        scores [n_jobs, stride] float32 (row j valid up to win[j, 1])."""
        import torch
        dev = torch.device("cuda", self.device)
        t = dict(scores=torch.zeros((n_jobs, stride), dtype=torch.float32, device=dev),
                 win=torch.zeros((n_jobs, 2), dtype=torch.int64, device=dev),
                 stat=torch.zeros((n_jobs, 2), dtype=torch.float32, device=dev),
                 cand=torch.zeros(n_jobs, dtype=torch.int32, device=dev))
        torch.cuda.synchronize(dev)   # the zero fills run on torch's stream, the captures on the handle's
        self._check(self.lib.b2_capture_nominations(self.h, t["scores"].data_ptr(), int(stride), t["win"].data_ptr(),
                                                    t["stat"].data_ptr(), t["cand"].data_ptr()),
                    "b2_capture_nominations")
        out = {}
        try:
            yield out
        finally:
            self._check(self.lib.b2_capture_nominations(self.h, None, 0, None, None, None), "b2_capture_nominations")
            self.synchronize()
            out.update({k: v.cpu().numpy() for k, v in t.items()})

    @contextlib.contextmanager
    def capture_reference(self, capacity: int, max_videos: int):
        """While the block runs, every batched sync call on this handle copies its reference signals into a
        NaN-filled device array of `capacity` floats (b2_capture_reference); the last call's copy is kept.  Yields a
        dict that holds numpy arrays once the block has exited: ref float32[capacity], ref_off int64[max_videos + 1]
        and packed uint8[max_videos] (1: the video's range starts with ceil(R/32) words of packed bits; read
        ref[...].view(np.uint32)).  ref_off is -1 and packed 255 where no call wrote."""
        import torch
        dev = torch.device("cuda", self.device)
        ref = torch.full((max(int(capacity), 1),), float("nan"), dtype=torch.float32, device=dev)
        ref_off = np.full(int(max_videos) + 1, -1, dtype=np.int64)
        packed = np.full(max(int(max_videos), 1), 255, dtype=np.uint8)
        torch.cuda.synchronize(dev)   # the fill runs on torch's stream, the copies on the handle's
        self._check(self.lib.b2_capture_reference(self.h, ref.data_ptr(), int(capacity), _ptr(ref_off), _ptr(packed),
                                                  int(max_videos)), "b2_capture_reference")
        out = {}
        try:
            yield out
        finally:
            self._check(self.lib.b2_capture_reference(self.h, None, 0, None, None, 0), "b2_capture_reference")
            self.synchronize()
            out.update(ref=ref.cpu().numpy()[: int(capacity)], ref_off=ref_off, packed=packed[: int(max_videos)])


def _default_device() -> int:
    """The device a handle is created on when the caller names none: torch's current CUDA device
    when torch is loaded and has a CUDA context (so kernels launch where the caller's ``.cuda()``
    tensors live, also on rank > 0), else LOCAL_RANK when B2_DEVICE_FROM_RANK is set, else 0."""
    import sys
    torch = sys.modules.get("torch")
    if torch is not None:
        try:
            if torch.cuda.is_available() and torch.cuda.is_initialized():
                return int(torch.cuda.current_device())
        except Exception:
            pass
    if os.environ.get("B2_DEVICE_FROM_RANK"):
        return int(os.environ.get("LOCAL_RANK", "0"))
    return 0


def get_handle(device: Optional[int] = None) -> Handle:
    """Per-thread handle (the reference runs several VideoSpeechTransformer.fit on threads)."""
    if device is None:
        device = _default_device()
    handles = getattr(_tls, "handles", None)
    if handles is None:
        handles = _tls.handles = {}
    if device not in handles:
        handles[device] = Handle(device)
    return handles[device]
