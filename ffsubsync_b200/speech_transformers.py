"""Signal producers of the hot path with the reference's API (ffsubsync/speech_transformers.py):

  * ``_make_energy_zcr_detector``  - detector factory with the reference's factory signature
    (:101-103, :155-157); the per-window work runs in the CUDA VAD kernel.
  * ``VideoSpeechTransformer``      - chunk loop / progress protocol of :609-757 around a detector.
  * ``SubtitleSpeechTransformer``   - cue rasterisation of :946-984 on the GPU rasteriser.
  * ``ComputeSpeechFrameBoundariesMixin`` (:299-317), ``DeserializeSpeechTransformer`` (:987-1009),
    ``make_subtitle_speech_pipeline`` (:56-98), ``_is_metadata`` (:928-943).

  * ``MultiSegmentVideoSpeechTransformer`` (:760-903) - sparse reference from a few sampled
    windows; the windows of an in-memory / raw-PCM reference go through ONE batched VAD launch.

  * ``_make_auditok_detector`` (:101-152) - the reference's auditok detector, energy test +
    StreamTokenizer + impulses/cumsum/clip, on the GPU (no auditok wheel needed).

Out of scope here (SURVEY.md section 2): embedded-subtitle extraction, silero / webrtc detectors
(third-party wheels / model weights).  Other detectors can be plugged in through
``DETECTOR_FACTORIES`` with the reference's factory signature.
"""
import io
import logging
import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor, as_completed
from datetime import timedelta
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple, Union

import numpy as np

from . import _native
from .constants import (
    CHUNK_WINDOWS,
    DEFAULT_ENERGY_THRESHOLD,
    DEFAULT_SCALE_FACTOR,
    DEFAULT_START_SECONDS,
    SAMPLE_RATE,
    detector_chunk_bytes,
)
from .sklearn_shim import Pipeline, TransformerMixin
from .subtitle_transformers import SubtitleScaler

logger: logging.Logger = logging.getLogger(__name__)


class ProgressInfo(NamedTuple):
    """Progress emitted to a ``progress_handler`` during speech extraction
    (same fields as the reference's, speech_transformers.py:38-53)."""

    processed_seconds: float
    total_seconds: Optional[float]

    @property
    def fraction(self) -> Optional[float]:
        if not self.total_seconds:
            return None
        return min(1.0, self.processed_seconds / self.total_seconds)


# ------------------------------------------------------------------------------------ detectors

def _make_energy_zcr_detector(
    sample_rate: int,
    frame_rate: int,
    non_speech_label: float,
    energy_threshold: int = DEFAULT_ENERGY_THRESHOLD,
    z_lo: Optional[int] = None,
    z_hi: Optional[int] = None,
) -> Callable[[Union[bytes, np.ndarray]], np.ndarray]:
    """Frame-energy / zero-crossing VAD (this package's detector; DESIGN.md).

    Same contract as the reference's detector factories: the returned callable takes the raw
    s16le bytes (or a uint8 view) of one chunk and returns one float per 10 ms window
    (1.0 = speech, ``non_speech_label`` otherwise); a trailing partial window is non-speech."""
    handle = _native.get_handle()
    fpw = handle.frames_per_window(frame_rate, sample_rate)
    if fpw <= 0:
        raise ValueError("bad frame_rate=%r / sample_rate=%r" % (frame_rate, sample_rate))

    def _detect(asegment) -> np.ndarray:
        if isinstance(asegment, np.ndarray) and asegment.dtype == np.int16:
            pcm = np.ascontiguousarray(asegment)
        else:
            raw = np.frombuffer(asegment, dtype=np.uint8) if not isinstance(asegment, np.ndarray) \
                else np.ascontiguousarray(asegment).view(np.uint8)
            pcm = raw[: (len(raw) // 2) * 2].view("<i2")
        out, _ = _native.get_handle().vad_energy_zcr(
            pcm, [0, len(pcm)], frame_rate, sample_rate, non_speech_label, energy_threshold,
            -1 if z_lo is None else z_lo, -1 if z_hi is None else z_hi)
        return out.astype(np.float64)

    # streaming form for the chunk loop (b2_vad_stream_*): same windows as one _detect call per
    # chunk, but push() only enqueues copy + kernel, so reading / decoding the next chunk overlaps
    def _stream_begin():
        _native.get_handle().vad_stream_begin(frame_rate, sample_rate, non_speech_label, energy_threshold,
                                              -1 if z_lo is None else z_lo, -1 if z_hi is None else z_hi)

    _detect.stream_begin = _stream_begin
    _detect.stream_push = lambda chunk: _native.get_handle().vad_stream_push(chunk)
    _detect.stream_end = lambda: _native.get_handle().vad_stream_end().astype(np.float64)
    return _detect


def _make_energy_detector(sample_rate: int, frame_rate: int, non_speech_label: float):
    """Energy-only variant (no zero-crossing band): what auditok's energy validator keeps
    (speech_transformers.py:125) before its tokenizer."""
    fpw = int((1.0 / sample_rate) * frame_rate + 0.5)
    return _make_energy_zcr_detector(sample_rate, frame_rate, non_speech_label, z_lo=0, z_hi=fpw)


def _make_auditok_detector(
    sample_rate: int, frame_rate: int, non_speech_label: float
) -> Callable[[Union[bytes, np.ndarray]], np.ndarray]:
    """The reference's auditok detector (speech_transformers.py:101-152) without the auditok wheel:
    energy test per 10 ms block (``AudioEnergyValidator(sample_width=2, energy_threshold=50)``, :125),
    ``StreamTokenizer(min_length=0.2*sample_rate, max_length=5*sample_rate,
    max_continuous_silence=0.25*sample_rate)`` (:126-131), start / end+1 impulses -> cumsum -> clip
    (:146-150) - all on the GPU (b2_vad_auditok: the energy kernel + a per-call tokenizer scan).
    One call = one chunk; like the reference's tokenizer the state restarts in every call."""
    handle = _native.get_handle()
    if handle.lib.b2_auditok_block_size(frame_rate, sample_rate) <= 0:
        raise ValueError("auditok detector: unsupported frame_rate=%r / sample_rate=%r" % (frame_rate, sample_rate))

    def _detect(asegment) -> np.ndarray:
        raw = np.frombuffer(asegment, dtype=np.uint8) if not isinstance(asegment, np.ndarray) \
            else np.ascontiguousarray(asegment).view(np.uint8)
        if len(raw) % 2 != 0:  # auditok's BufferAudioSource refuses such a buffer
            raise ValueError("length of data_buffer must be a multiple of (sample_width * channels)")
        pcm = raw.view("<i2")
        out, _ = _native.get_handle().vad_auditok(pcm, [0, len(pcm)], frame_rate, sample_rate, non_speech_label)
        return out

    return _detect


#: name fragment looked up in ``VideoSpeechTransformer.vad`` -> factory(sample_rate, frame_rate, label)
DETECTOR_FACTORIES: Dict[str, Callable[[int, int, float], Callable]] = {
    "auditok": _make_auditok_detector,
    "energy_only": _make_energy_detector,
    "energy": _make_energy_zcr_detector,
}

_FUSION_STRATEGIES = ("weighted", "intersection", "union")
_FUSION_MODE = {"intersection": 0, "union": 1, "weighted": 2}


def _make_fused_detector(
    sample_rate: int,
    frame_rate: int,
    non_speech_label: float,
    fusion_strategy: str = "weighted",
    factories=None,
) -> Callable[[Union[bytes, np.ndarray]], np.ndarray]:
    """Combine two detectors like the reference's fused VAD (speech_transformers.py:256-296):
    clip both outputs to their common length, then ``intersection`` = element-wise min, ``union`` =
    max, ``weighted`` (default) = 0.6 * first + 0.4 * second (the reference weights silero 0.6 and
    webrtc 0.4).  The blend runs on the GPU (b2_blend_signals).  ``factories`` = two detector
    factories with the reference signature; default: the energy/zero-crossing detector (0.6)
    and its energy-only variant (0.4)."""
    if fusion_strategy not in _FUSION_STRATEGIES:
        raise ValueError("unknown fused VAD strategy %r; choose one of %s"
                         % (fusion_strategy, ", ".join(_FUSION_STRATEGIES)))
    first_factory, second_factory = factories or (_make_energy_zcr_detector, _make_energy_detector)
    first = first_factory(sample_rate, frame_rate, non_speech_label)
    second = second_factory(sample_rate, frame_rate, non_speech_label)
    mode = _FUSION_MODE[fusion_strategy]

    def _detect(asegment) -> np.ndarray:
        a, b = np.asarray(first(asegment), dtype=float), np.asarray(second(asegment), dtype=float)
        if min(len(a), len(b)) == 0:
            return np.zeros(0)
        return _native.get_handle().blend_signals(a, b, mode, 0.6, 0.4).astype(np.float64)

    return _detect


# ---------------------------------------------------------------------------------- boundaries

class ComputeSpeechFrameBoundariesMixin:
    def __init__(self) -> None:
        self.start_frame_: Optional[int] = None
        self.end_frame_: Optional[int] = None

    @property
    def num_frames(self) -> Optional[int]:
        if self.start_frame_ is None or self.end_frame_ is None:
            return None
        return self.end_frame_ - self.start_frame_

    def fit_boundaries(self, speech_frames: np.ndarray) -> "ComputeSpeechFrameBoundariesMixin":
        # the kernel tests float32 x > 0.5f; rounding the float64 signal UP to float32 keeps the
        # reference's float64 test (0.5 is a float32, so x > 0.5 <=> round_up(x) > 0.5): a level of
        # 0.500000005 (ratio 1.99999998) would round to nearest 0.5f and find no speech
        x64 = np.asarray(speech_frames, dtype=np.float64)
        x = x64.astype(np.float32)
        low = x < x64
        x[low] = np.nextafter(x[low], np.float32(np.inf))
        if len(x):
            first, last = _native.get_handle().first_last_nonzero(x, [0, len(x)])
            if last[0] >= 0:
                self.start_frame_ = int(first[0])
                self.end_frame_ = int(last[0])
        return self


# ----------------------------------------------------------------------------- video / PCM side

_PCM_SUFFIXES = (".pcm", ".raw", ".s16le")


class _BoundedReader:
    """.read(n) over at most ``limit`` bytes of a file object."""

    def __init__(self, fh, limit: int) -> None:
        self._fh, self._left = fh, limit

    def read(self, n: int) -> bytes:
        data = self._fh.read(min(n, self._left)) if self._left > 0 else b""
        self._left -= len(data)
        return data


class _DetectorSink:
    """Feeds chunks to a detector.  Detectors with the streaming protocol (``stream_begin`` /
    ``stream_push`` / ``stream_end``: this package's energy detectors, b2_vad_stream_*) only enqueue
    copy + kernel per chunk, so reading / decoding the next chunk overlaps; any other detector
    (auditok, fused, third-party factories) is called once per chunk like the reference does (:746)."""

    def __init__(self, detector) -> None:
        self.detector = detector
        self.streaming = all(hasattr(detector, a) for a in ("stream_begin", "stream_push", "stream_end"))
        self.open = False
        self.pieces: List[np.ndarray] = []

    def feed(self, data: bytes) -> None:
        if not self.streaming:
            self.pieces.append(self.detector(np.frombuffer(data, np.uint8)))
            return
        if not self.open:
            self.detector.stream_begin()
            self.open = True
        self.detector.stream_push(data)

    def abort(self) -> None:
        if self.open:
            self.open = False
            try:
                self.detector.stream_end()
            except Exception:
                pass

    def finish(self) -> List[np.ndarray]:
        if self.open:
            self.open = False
            self.pieces.append(self.detector.stream_end())
        return self.pieces


class VideoSpeechTransformer(TransformerMixin):
    """PCM -> 100 Hz speech signal.  ``fit`` accepts what the reference accepts (a media path,
    decoded through an ffmpeg subprocess when the binary is available) and, because this layer
    starts at decoded audio, also raw s16le mono PCM directly: bytes / bytearray / int16 or uint8
    arrays, a binary file object, or a ``.pcm`` / ``.raw`` / ``.s16le`` file."""

    def __init__(
        self,
        vad: str,
        sample_rate: int,
        frame_rate: int,
        non_speech_label: float,
        start_seconds: int = 0,
        ffmpeg_path: Optional[str] = None,
        ref_stream: Optional[str] = None,
        vlc_mode: bool = False,
        gui_mode: bool = False,
        max_duration_seconds: Optional[float] = None,
        extract_audio_first: bool = False,
        progress_handler: Optional[Callable[["ProgressInfo"], None]] = None,
    ) -> None:
        self.vad: str = vad
        self.sample_rate: int = sample_rate
        self.frame_rate: int = frame_rate
        self._non_speech_label: float = non_speech_label
        self.start_seconds: int = start_seconds
        self.ffmpeg_path: Optional[str] = ffmpeg_path
        self.ref_stream: Optional[str] = ref_stream
        self.vlc_mode: bool = vlc_mode
        self.gui_mode: bool = gui_mode
        self.max_duration_seconds: Optional[float] = max_duration_seconds
        self.extract_audio_first: bool = extract_audio_first
        self.progress_handler = progress_handler
        self.video_speech_results_: Optional[np.ndarray] = None

    # -- detector dispatch (speech_transformers.py:655-679) -----------------------------------
    def _make_detector(self):
        if "fused" in self.vad:  # "fused" or "fused:intersection" ...; default strategy is weighted
            strategy = self.vad.split(":", 1)[1] if ":" in self.vad else "weighted"
            return _make_fused_detector(self.sample_rate, self.frame_rate, self._non_speech_label, strategy)
        for key, factory in DETECTOR_FACTORIES.items():
            if key in self.vad:
                return factory(self.sample_rate, self.frame_rate, self._non_speech_label)
        raise ValueError("unknown vad: %s" % self.vad)

    # -- PCM sources -----------------------------------------------------------------------------
    def _build_ffmpeg_args(self, fname: str) -> List[str]:
        exe = "ffmpeg"
        if self.ffmpeg_path:
            exe = os.path.join(self.ffmpeg_path, "ffmpeg")
        args = [exe]
        if self.start_seconds > 0:
            args += ["-ss", str(timedelta(seconds=self.start_seconds))]
        if self.max_duration_seconds is not None:
            args += ["-t", str(timedelta(seconds=self.max_duration_seconds))]
        args += ["-loglevel", "fatal", "-nostdin", "-i", fname]
        if self.ref_stream is not None and self.ref_stream.startswith("0:a:"):
            args += ["-map", self.ref_stream]
        args += ["-f", "s16le", "-ac", "1", "-acodec", "pcm_s16le", "-af", "aresample=async=1",
                 "-ar", str(self.frame_rate), "-"]
        return args

    def _pcm_window(self, n_bytes: int) -> Tuple[int, int]:
        """Byte range of a raw PCM source that ffmpeg's ``-ss start_seconds -t max_duration_seconds``
        (speech_transformers.py:688-699) would have decoded."""
        lo = min(n_bytes, 2 * int(round(self.start_seconds * self.frame_rate)))
        hi = n_bytes
        if self.max_duration_seconds is not None:
            hi = min(hi, lo + 2 * int(round(self.max_duration_seconds * self.frame_rate)))
        return lo, hi

    def _open_source(self, src):
        """-> (readable with .read(n), total_duration_seconds or None, closer)"""
        bytes_per_second = 2.0 * self.frame_rate
        if isinstance(src, np.ndarray):
            src = np.ascontiguousarray(src).view(np.uint8).tobytes() if src.dtype != np.uint8 else src.tobytes()
        if isinstance(src, (bytes, bytearray, memoryview)):
            lo, hi = self._pcm_window(len(src))
            return io.BytesIO(bytes(src[lo:hi])), (hi - lo) / bytes_per_second, None
        if hasattr(src, "read"):
            return src, None, None
        if isinstance(src, str) and src.lower().endswith(_PCM_SUFFIXES):
            lo, hi = self._pcm_window(os.path.getsize(src))
            fh = open(src, "rb")
            fh.seek(lo)
            return _BoundedReader(fh, hi - lo), (hi - lo) / bytes_per_second, fh.close
        args = self._build_ffmpeg_args(src)
        if shutil.which(args[0]) is None:
            raise ValueError(
                "cannot decode %r: no ffmpeg binary found; pass decoded s16le mono PCM "
                "(bytes / array / .pcm file) instead" % (src,))
        proc = subprocess.Popen(args, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
        return proc.stdout, None, proc.wait

    # -- chunk loop (speech_transformers.py:680-753) -------------------------------------------------
    CHUNK_WINDOWS: int = CHUNK_WINDOWS   # 100 s per detector call at the 100 Hz sample rate (:711,741)

    def _chunks(self, readable):
        """PCM in the reference's read granularity: 10 000 windows of ``2 * frame_rate // sample_rate``
        bytes each (:710-711,741)."""
        n = detector_chunk_bytes(self.frame_rate, self.sample_rate, self.CHUNK_WINDOWS)
        while True:
            data = readable.read(n)
            if not data:
                return
            yield data

    def _report(self, seconds_done: float, seconds_total: Optional[float]) -> None:
        """Progress protocol (:724-739): the optional callback (its exceptions never break a sync) and
        the integer-percent lines VLC mode prints."""
        if self.progress_handler is not None:
            try:
                self.progress_handler(ProgressInfo(processed_seconds=seconds_done, total_seconds=seconds_total))
            except Exception as e:
                logger.warning("progress_handler raised: %s", e)
        if self.vlc_mode and seconds_total is not None:
            print("%d" % int(seconds_done * 100.0 / seconds_total), flush=True)

    def fit(self, fname, *_) -> "VideoSpeechTransformer":
        sink = _DetectorSink(self._make_detector())
        readable, total, closer = self._open_source(fname)
        if total is not None and self.max_duration_seconds is not None:
            total = min(total, self.max_duration_seconds)
        done = 0.0
        try:
            for data in self._chunks(readable):
                seconds = len(data) / 2.0 / self.frame_rate
                done = done + seconds if total is None else min(total, done + seconds)
                self._report(done, total)
                sink.feed(data)
        except BaseException:
            sink.abort()   # close the device-side stream without masking the error
            raise
        finally:
            if closer is not None:
                closer()
        pieces = sink.finish()
        if not pieces:
            raise ValueError(
                "Unable to detect speech. "
                "Perhaps try specifying a different stream / track, or a different vad.")
        self.video_speech_results_ = np.concatenate(pieces)
        logger.info("total of speech segments: %s", np.sum(self.video_speech_results_))
        return self

    def transform(self, *_) -> np.ndarray:
        return self.video_speech_results_


class MultiSegmentVideoSpeechTransformer(TransformerMixin):
    """Sparse reference signal from ``segment_count`` short windows spread over the reference
    (speech_transformers.py:760-903): VAD runs only on the sampled windows, their results are
    written at their true positions of a full-length array that is zero elsewhere, and the normal
    ratio search + cross-correlation runs on that.

    Same constructor, ``_segment_starts`` arithmetic, assembly and error behaviour as the
    reference.  Difference in execution: when the reference audio is raw PCM in memory (or a
    ``.pcm`` file) and the detector is this package's energy detector, all windows are detected by
    ONE batched kernel launch (ragged batch of B = len(starts) signals) instead of up to four
    threads each decoding and detecting one window; other sources / detectors use the
    reference's thread pool of ``VideoSpeechTransformer`` fits."""

    START_MARGIN_SECONDS: int = 30
    END_MARGIN_SECONDS: int = 60

    def __init__(
        self,
        vad: str,
        sample_rate: int,
        frame_rate: int,
        non_speech_label: float,
        segment_count: int = 8,
        segment_duration: int = 60,
        skip_intro_outro: bool = False,
        parallel_workers: int = 4,
        ffmpeg_path: Optional[str] = None,
        ref_stream: Optional[str] = None,
        vlc_mode: bool = False,
        gui_mode: bool = False,
    ) -> None:
        # audio-only sampling: a "subs_then_" prefix is dropped (:799-801)
        self.vad: str = vad.split("subs_then_")[-1]
        self.sample_rate: int = sample_rate
        self.frame_rate: int = frame_rate
        self._non_speech_label: float = non_speech_label
        self.segment_count: int = segment_count
        self.segment_duration: int = segment_duration
        self.skip_intro_outro: bool = skip_intro_outro
        self.parallel_workers: int = parallel_workers
        self.ffmpeg_path: Optional[str] = ffmpeg_path
        self.ref_stream: Optional[str] = ref_stream
        self.vlc_mode: bool = vlc_mode
        self.gui_mode: bool = gui_mode
        self.video_speech_results_: Optional[np.ndarray] = None

    def _segment_starts(self, total_duration: float) -> List[int]:
        """Whole-second start times, evenly spread over [lo, hi - segment_duration] (:812-830)."""
        seg = self.segment_duration
        if total_duration <= seg:
            return [0]
        lo = float(self.START_MARGIN_SECONDS) if self.skip_intro_outro else 0.0
        hi = total_duration - (self.END_MARGIN_SECONDS if self.skip_intro_outro else 0)
        if hi - lo < seg:  # the margins do not leave room for one segment: drop them
            lo, hi = 0.0, total_duration
        room = hi - lo - seg
        count = max(1, self.segment_count)
        if room <= 0 or count == 1:
            return [int(max(0.0, min(lo, total_duration - seg)))]
        last = int(total_duration) - seg
        picked = {max(0, min(int(round(lo + i * (room / (count - 1)))), last)) for i in range(count)}
        return sorted(picked)

    # -- reference duration -----------------------------------------------------------------------
    def _pcm_bytes_of(self, src) -> Optional[int]:
        if isinstance(src, np.ndarray):
            return src.size * src.dtype.itemsize
        if isinstance(src, (bytes, bytearray, memoryview)):
            return len(src)
        if isinstance(src, str) and src.lower().endswith(_PCM_SUFFIXES):
            return os.path.getsize(src)
        return None

    def _probe_duration(self, fname) -> float:
        n_bytes = self._pcm_bytes_of(fname)
        try:
            if n_bytes is not None:
                return n_bytes / (2.0 * self.frame_rate)
            exe = os.path.join(self.ffmpeg_path, "ffprobe") if self.ffmpeg_path else "ffprobe"
            if shutil.which(exe) is None:
                raise RuntimeError("no ffprobe binary found")
            out = subprocess.check_output(
                [exe, "-v", "error", "-show_entries", "format=duration", "-of",
                 "default=noprint_wrappers=1:nokey=1", fname], stderr=subprocess.DEVNULL)
            return float(out.decode().strip())
        except Exception as e:
            raise ValueError("multi-segment sync needs the reference duration, but probing "
                             "'%s' failed: %s" % (fname, e))

    # -- per-segment detection ----------------------------------------------------------------------
    def _extract_segment_speech(self, fname, start: int) -> Tuple[int, np.ndarray]:
        """One window through its own VideoSpeechTransformer (:832-847)."""
        segment = VideoSpeechTransformer(
            vad=self.vad, sample_rate=self.sample_rate, frame_rate=self.frame_rate,
            non_speech_label=self._non_speech_label, start_seconds=start,
            ffmpeg_path=self.ffmpeg_path, ref_stream=self.ref_stream, vlc_mode=self.vlc_mode,
            gui_mode=self.gui_mode, max_duration_seconds=self.segment_duration)
        segment.fit(fname)
        return start, segment.transform()

    def _batched_params(self):
        """(z_lo, z_hi) when ``self.vad`` names the plain energy detectors, else None."""
        if "fused" in self.vad:
            return None
        if "energy_only" in self.vad:
            return 0, int((1.0 / self.sample_rate) * self.frame_rate + 0.5)
        if "energy" in self.vad and DETECTOR_FACTORIES.get("energy") is _make_energy_zcr_detector:
            return -1, -1
        return None

    def _extract_all_batched(self, fname, starts: List[int], band) -> Dict[int, np.ndarray]:
        """All windows of a raw-PCM reference in one VAD launch."""
        if isinstance(fname, str):
            raw = np.memmap(fname, dtype=np.uint8, mode="r")   # an odd trailing byte is ignored
            pcm_all = raw[: (len(raw) // 2) * 2].view("<i2")
        elif isinstance(fname, np.ndarray):
            raw = np.ascontiguousarray(fname).view(np.uint8)
            pcm_all = raw[: (len(raw) // 2) * 2].view("<i2")
        else:
            raw = np.frombuffer(fname, dtype=np.uint8)
            pcm_all = raw[: (len(raw) // 2) * 2].view("<i2")
        pieces, off = [], [0]
        for s in starts:  # whole-second starts: every piece but a clipped last one keeps 16 B alignment
            lo = min(len(pcm_all), int(round(s * self.frame_rate)))
            hi = min(len(pcm_all), lo + int(round(self.segment_duration * self.frame_rate)))
            pieces.append(np.asarray(pcm_all[lo:hi]))
            off.append(off[-1] + (hi - lo))
        out, out_off = _native.get_handle().vad_energy_zcr(
            np.concatenate(pieces) if pieces else np.zeros(0, np.int16), off, self.frame_rate,
            self.sample_rate, self._non_speech_label, DEFAULT_ENERGY_THRESHOLD, band[0], band[1])
        return {s: out[out_off[i]:out_off[i + 1]].astype(np.float64) for i, s in enumerate(starts)}

    def fit(self, fname, *_) -> "MultiSegmentVideoSpeechTransformer":
        total_duration = self._probe_duration(fname)
        starts = self._segment_starts(total_duration)
        logger.info("multi-segment sync: sampling %d segment(s) of up to %ds at %s",
                    len(starts), self.segment_duration, [int(s) for s in starts])
        sparse = np.zeros(int(total_duration * self.sample_rate) + 2, dtype=float)

        def place(start, seg_speech):
            begin = int(start * self.sample_rate)
            end = min(begin + len(seg_speech), len(sparse))
            if end > begin:
                sparse[begin:end] = seg_speech[: end - begin]

        band = self._batched_params()
        own_extract = type(self)._extract_segment_speech is MultiSegmentVideoSpeechTransformer._extract_segment_speech \
            and "_extract_segment_speech" not in self.__dict__
        if band is not None and own_extract and self._pcm_bytes_of(fname) is not None:
            for start, seg_speech in self._extract_all_batched(fname, starts, band).items():
                if len(seg_speech):
                    place(start, seg_speech)
        else:
            workers = max(1, min(self.parallel_workers, len(starts)))
            with ThreadPoolExecutor(max_workers=workers) as executor:
                pending = {executor.submit(self._extract_segment_speech, fname, s): s for s in starts}
                for fut in as_completed(pending):
                    try:
                        start, seg_speech = fut.result()
                    except Exception as e:  # one bad window must not sink the sync (:878-882)
                        logger.warning("failed to extract segment at %ds: %s", pending[fut], e)
                        continue
                    place(start, seg_speech)
        if not np.any(sparse > 0):
            raise ValueError("Unable to detect speech in any sampled segment. "
                             "Perhaps try specifying a different stream / track, or a different vad.")
        self.video_speech_results_ = sparse
        logger.info("total of speech segments: %s", np.sum(self.video_speech_results_))
        return self

    def transform(self, *_) -> np.ndarray:
        return self.video_speech_results_


# ------------------------------------------------------------------------------- subtitle side

_PAIRED_NESTER = {"(": ")", "{": "}", "[": "]", "（": "）", "【": "】", "「": "」"}
_MARKUP_TAG = re.compile(r"<[^>]+>")
_NON_DIALOGUE_SYMBOLS = frozenset("♪♫♬♩\U0001F3B5\U0001F3B6")


def _is_metadata(content: str, is_beginning_or_end: bool) -> bool:
    """Cue text that carries no speech: empty, fully bracketed, music symbols only, or (first /
    last cue) credits-like lines.  Markup tags are ignored."""
    text = _MARKUP_TAG.sub("", content).strip()
    if not text:
        return True
    if _PAIRED_NESTER.get(text[0]) == text[-1]:
        return True
    if all(ch.isspace() or ch in _NON_DIALOGUE_SYMBOLS for ch in text):
        return True
    if is_beginning_or_end:
        return "english" in text.lower() or " - " in text
    return False


class SubtitleSpeechTransformer(TransformerMixin, ComputeSpeechFrameBoundariesMixin):
    def __init__(self, sample_rate: int, start_seconds: int = 0, framerate_ratio: float = 1.0) -> None:
        ComputeSpeechFrameBoundariesMixin.__init__(self)
        self.sample_rate: int = sample_rate
        self.start_seconds: int = start_seconds
        self.framerate_ratio: float = framerate_ratio
        self.subtitle_speech_results_: Optional[np.ndarray] = None
        self.max_time_: Optional[float] = None

    def fit(self, subs, *_) -> "SubtitleSpeechTransformer":
        subs = list(subs)
        n = len(subs)
        starts = np.array([s.start.total_seconds() for s in subs], dtype=np.float64)
        ends = np.array([s.end.total_seconds() for s in subs], dtype=np.float64)
        keep = np.array([not _is_metadata(s.content, i == 0 or i + 1 == n) for i, s in enumerate(subs)],
                        dtype=np.uint8)
        max_time = max([0] + list(ends))
        self.max_time_ = max_time - self.start_seconds
        level = min(1.0 / self.framerate_ratio, 1.0)
        # the cues arrive already scaled (SubtitleScaler ran before us): ratio 1.0 for the times,
        # explicit level for the value (speech_transformers.py:977)
        out, _ = _native.get_handle().rasterize(
            starts, ends, keep, [0, n], [1.0], 1, False, self.sample_rate, float(self.start_seconds),
            levels=[level])
        self.subtitle_speech_results_ = out.astype(np.float64)
        if level != 0.0:  # the kernel writes float32; restore the float64 level the reference writes
            self.subtitle_speech_results_[out != 0] = level
        self.fit_boundaries(self.subtitle_speech_results_)
        return self

    def transform(self, *_) -> np.ndarray:
        assert self.subtitle_speech_results_ is not None
        return self.subtitle_speech_results_


class DeserializeSpeechTransformer(TransformerMixin):
    def __init__(self, non_speech_label: float) -> None:
        self._non_speech_label: float = non_speech_label
        self.deserialized_speech_results_: Optional[np.ndarray] = None

    def fit(self, fname, *_) -> "DeserializeSpeechTransformer":
        speech = np.load(fname)
        if hasattr(speech, "files"):
            if "speech" not in speech.files:
                raise ValueError('could not find "speech" array in serialized file; only contains: %s'
                                 % speech.files)
            speech = speech["speech"]
        speech[speech < 1.0] = self._non_speech_label
        self.deserialized_speech_results_ = speech
        return self

    def transform(self, *_) -> np.ndarray:
        assert self.deserialized_speech_results_ is not None
        return self.deserialized_speech_results_


def make_subtitle_speech_pipeline(
    fmt: str = "srt",
    encoding: str = "infer",
    caching: bool = False,
    max_subtitle_seconds: int = 10,
    start_seconds: int = DEFAULT_START_SECONDS,
    scale_factor: Optional[float] = DEFAULT_SCALE_FACTOR,
    parser=None,
    **kwargs,
) -> Union[Pipeline, Callable[[float], Pipeline]]:
    """parse -> scale -> speech_extract, or (``scale_factor=None``) a maker ``ratio -> Pipeline`` for
    the golden-section search; same positional order and keywords as the reference
    (speech_transformers.py:56-98).  Subtitle *parsing* is outside the hot path (SURVEY.md section 2),
    so where the reference would build a parser from ``fmt`` / ``encoding`` / ... the caller must
    pass ``parser=`` (any transformer whose ``transform`` yields cues with ``.start`` / ``.end`` /
    ``.content``); a parser that carries ``encoding`` / ``max_subtitle_seconds`` / ``start_seconds``
    attributes is checked against the arguments like the reference does (:73-75)."""
    if parser is None:
        raise ValueError(
            "make_subtitle_speech_pipeline(fmt=%r, ...): subtitle parsing is not part of this package; "
            "pass parser=<transformer yielding cues> (the reference builds one with "
            "make_subtitle_parser here)" % (fmt,))
    for name, want in (("encoding", encoding), ("max_subtitle_seconds", max_subtitle_seconds),
                       ("start_seconds", start_seconds)):
        if hasattr(parser, name):
            assert getattr(parser, name) == want, "parser.%s != %r" % (name, want)

    def subpipe_maker(framerate_ratio):
        return Pipeline([
            ("parse", parser),
            ("scale", SubtitleScaler(framerate_ratio)),
            ("speech_extract", SubtitleSpeechTransformer(
                sample_rate=SAMPLE_RATE, start_seconds=start_seconds, framerate_ratio=framerate_ratio)),
        ])

    return subpipe_maker if scale_factor is None else subpipe_maker(scale_factor)
