"""Float64 restatement of MultiSegmentVideoSpeechTransformer.fit's sparse reference (ffsubsync/
speech_transformers.py:855-895) as the batched sync calls build it (b2_sync_tracks_seg, csrc/seg_ref.cuh), over
vad_oracle / auditok_oracle per segment.

The reference has int(total * sample_rate) + 2 frames of 0.0; segment s (a whole-second start) writes its detector
output at frames [s * sample_rate, min(s * sample_rate + len, L)).  The reference's threads finish in any order; the
batched calls write in increasing start order, so the later start wins where segments overlap."""
import numpy as np

from . import auditok_oracle as au
from . import chunk_oracle as co

NO_SPEECH = ("Unable to detect speech in any sampled segment. "
             "Perhaps try specifying a different stream / track, or a different vad.")


def length(total: float, sample_rate: int) -> int:
    """The reference's length int(total * sample_rate) + 2 (float64 product, truncated)."""
    return int(float(total) * sample_rate) + 2


def assemble(total: float, sample_rate: int, outputs) -> np.ndarray:
    """The sparse float64 reference of the per-segment outputs ``outputs`` [(start, frames), ...] in increasing start
    order (a failed segment is left out)."""
    x = np.zeros(length(total, sample_rate), dtype=float)
    for start, seg in outputs:
        begin = int(start * sample_rate)
        end = min(begin + len(seg), len(x))
        if end > begin:
            x[begin:end] = seg[: end - begin]
    return x


def has_speech(x) -> bool:
    """The reference's check before it raises NO_SPEECH: some frame > 0."""
    return bool(np.any(np.asarray(x) > 0))


def detect(pcm, detector: str = "energy_zcr", sample_rate: int = 100, frame_rate: int = 16000,
           non_speech_label: float = 0.0, chunk_samples: int = 0, **params) -> np.ndarray:
    """The call's detector on one segment's int16 samples taken as one signal: energy / ZCR (vad_oracle; params:
    energy_threshold, z_lo, z_hi) over the reference's chunk loop from the segment's first sample
    (chunk_oracle.chunk_loop), or auditok over the chunk loop of chunk_samples samples from there (0: one call;
    params: energy_threshold in dB, min_length, max_length, max_continuous_silence)."""
    pcm = np.asarray(pcm, dtype=np.int16)
    if detector == "energy_zcr":
        return co.chunk_loop("energy_zcr", pcm, frame_rate, sample_rate, non_speech_label, **params)
    step = chunk_samples if chunk_samples > 0 else max(len(pcm), 1)
    parts = [au.auditok_detect_fast(pcm[i:i + step].tobytes(), sample_rate, frame_rate, non_speech_label, **params)
             for i in range(0, len(pcm), step)]
    return np.concatenate(parts) if parts else np.zeros(0)


def segment_reference(pcm_video, total: float, starts, lo, hi, sample_rate: int = 100, **det) -> np.ndarray:
    """The float64 reference of one segment video: segment j is pcm_video[lo[j]:hi[j]] starting at starts[j]."""
    outs = [(s, detect(pcm_video[a:b], sample_rate=sample_rate, **det)) for s, a, b in zip(starts, lo, hi)]
    return assemble(total, sample_rate, outs)
