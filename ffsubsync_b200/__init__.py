"""ffsubsync_b200 - the alignment hot path of smacke/ffsubsync on NVIDIA H100 (sm_90a).

Python host layer over a C-ABI CUDA library (include/ffsubsync_b200.h).  Module and class
names mirror the reference so that the new path is a drop-in behind its transformer API:

    from ffsubsync_b200.aligners import FFTAligner, MaxScoreAligner
    from ffsubsync_b200.speech_transformers import VideoSpeechTransformer, SubtitleSpeechTransformer
    from ffsubsync_b200.sklearn_shim import Pipeline, make_pipeline

There is no CPU implementation in this package: every compute call goes to the GPU library
and raises if it (or an H100) is missing.
"""
from .constants import (  # noqa: F401
    DEFAULT_FRAME_RATE,
    DEFAULT_MAX_OFFSET_SECONDS,
    DEFAULT_NON_SPEECH_LABEL,
    FRAMERATE_RATIOS,
    SAMPLE_RATE,
)

__version__ = "0.1.0"
