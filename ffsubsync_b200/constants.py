"""Hot-path constants (values from the reference's ffsubsync/constants.py:7-19)."""
from typing import List

import numpy as np

SAMPLE_RATE: int = 100                      # 10 ms windows (constants.py:7)
FRAMERATE_RATIOS: List[float] = [24.0 / 23.976, 25.0 / 23.976, 25.0 / 24.0]  # constants.py:9
DEFAULT_FRAME_RATE: int = 48000             # ffmpeg decode rate (constants.py:11)
DEFAULT_NON_SPEECH_LABEL: float = 0.0       # constants.py:12
DEFAULT_START_SECONDS: int = 0
DEFAULT_SCALE_FACTOR: float = 1
DEFAULT_MAX_OFFSET_SECONDS: int = 60        # constants.py:18
DEFAULT_VAD: str = "energy_zcr"             # the detector this package implements
BATCH_VADS = ("energy_zcr", "auditok")      # detectors the batched sync calls run
# ... and with a video's embedded subtitle stream as its reference where the caller hands one over
BATCH_VADS += ("subs_then_energy_zcr", "subs_then_auditok")

# energy / zero-crossing detector defaults (DESIGN.md): auditok's energy_threshold=50 dB
# (speech_transformers.py:125) is mean(x^2) >= 1e5
DEFAULT_ENERGY_THRESHOLD: int = 100000

# the reference's chunk loop reads 10 000 windows of ``2 * frame_rate // sample_rate`` bytes per detector
# call (speech_transformers.py:710-711,741)
CHUNK_WINDOWS: int = 10000


def detector_chunk_bytes(frame_rate: int, sample_rate: int, windows: int = CHUNK_WINDOWS) -> int:
    """Bytes of s16le PCM per detector call of the reference's chunk loop (half as many samples)."""
    return (2 * frame_rate // sample_rate) * windows


def framerate_ratios_to_try(no_fix_framerate: bool = False, gss: bool = False) -> list:
    """The candidate list try_sync builds (ffsubsync/ffsubsync.py:131-142): the ratios and their
    inverses as float64; ``None`` stands for the golden-section search entry."""
    if no_fix_framerate:
        return []
    r = np.array(FRAMERATE_RATIOS)
    out = list(np.concatenate([r, 1.0 / r]))
    if gss:
        out.append(None)
    return out
