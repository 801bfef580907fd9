"""The reference's chunk loop around a detector (TEST INFRASTRUCTURE ONLY).

VideoSpeechTransformer.fit reads ffmpeg's pipe ``(2 * frame_rate // sample_rate) * 10000`` bytes at a time and calls
the detector once per read, appending its output (speech_transformers.py:710-746).  Every call has its own window
grid and its own trailing partial window, so the result is the one-call detector's only where a read is a whole
number of windows: for energy / ZCR (int(frame_rate / sample_rate + 0.5)-sample windows) that fails at 22.05 kHz,
where a read is 2 205 000 samples of 221; for auditok the tokenizer restarts in every call, whatever the rate.
"""
import numpy as np

from . import auditok_oracle as au
from . import vad_oracle as vo

DETECTORS = {"energy_zcr": vo.energy_zcr_detect, "auditok": au.auditok_detect_fast}


def read_samples(frame_rate: int, sample_rate: int = 100) -> int:
    """Samples per read of the chunk loop: (2 fr // sr) * 10000 bytes of s16le."""
    return (2 * frame_rate // sample_rate) * 10000 // 2


def chunk_loop(detector: str, pcm, frame_rate: int, sample_rate: int = 100, non_speech_label: float = 0.0,
               chunk=None, **params) -> np.ndarray:
    """The detector ("energy_zcr" or "auditok", with its keyword params) over int16 pcm, one call per read of
    `chunk` samples (default read_samples; 0: one call over the whole signal), outputs concatenated (float64)."""
    detect = DETECTORS[detector]
    pcm = np.asarray(pcm, dtype=np.int16)
    step = read_samples(frame_rate, sample_rate) if chunk is None else chunk
    step = step if step > 0 else max(len(pcm), 1)
    parts = [np.asarray(detect(pcm[i:i + step].tobytes(), sample_rate, frame_rate, non_speech_label, **params),
                        np.float64) for i in range(0, len(pcm), step)]
    return np.concatenate(parts) if parts else np.zeros(0)
