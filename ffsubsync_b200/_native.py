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
    "b2_launch_count", "b2_vad_frames_per_window", "b2_vad_num_windows", "b2_vad_energy_zcr",
    "b2_rasterize_lengths", "b2_rasterize", "b2_blend_signals", "b2_first_last_nonzero", "b2_align_batch",
    "b2_reduce_ratios", "b2_sync_batch", "b2_synth_pcm", "b2_vad_stream_begin", "b2_vad_stream_push",
    "b2_vad_stream_windows", "b2_vad_stream_end", "b2_auditok_block_size", "b2_auditok_energy_floor",
    "b2_vad_auditok", "b2_capture_nominations", "b2_sync_tracks", "b2_sync_tracks_gss",
    "b2_sync_tracks_auditok", "b2_sync_tracks_subs",
]
B2_DETECTOR_ENERGY_ZCR, B2_DETECTOR_AUDITOK = 0, 1   # b2_sync_tracks_subs: the detector of the audio videos
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

    # -- diagnostics (tests) --------------------------------------------------------------------
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
