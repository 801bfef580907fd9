"""SubtitleScaler with the reference's API (ffsubsync/subtitle_transformers.py:29-50) plus the
minimal cue type the hot path needs.

The scaler is host code on purpose: it only rewrites ~1.2 k (start, end) pairs and must go
through ``datetime.timedelta`` to stay bit-compatible with the reference's microsecond rounding.
When the K ratio candidates of a pair are rasterised on the GPU (b2_rasterize), the same
rounding is reproduced inside the kernel and this class is bypassed.
"""
import numbers
from datetime import timedelta
from typing import Any, Iterable, List

from .sklearn_shim import TransformerMixin


class Cue:
    """A subtitle cue: ``start`` / ``end`` are timedeltas, ``content`` its text.  Duck-compatible
    with the reference's GenericSubtitle for everything the hot path reads
    (ffsubsync/generic_subtitles.py:17-41)."""

    __slots__ = ("start", "end", "inner")

    def __init__(self, start: timedelta, end: timedelta, inner: Any = "") -> None:
        self.start = start
        self.end = end
        self.inner = inner

    @property
    def content(self) -> str:
        inner = self.inner
        if isinstance(inner, str):
            return inner
        for attr in ("content", "text"):
            if hasattr(inner, attr):
                return getattr(inner, attr)
        raise NotImplementedError("unsupported subtitle type: %s" % type(inner))

    def __eq__(self, other: object) -> bool:
        return (isinstance(other, Cue) and self.start == other.start and self.end == other.end
                and self.inner == other.inner)

    def __repr__(self) -> str:
        return "Cue(%r, %r, %r)" % (self.start, self.end, self.inner)


def cues_from_seconds(starts: Iterable[float], ends: Iterable[float], contents=None) -> List[Cue]:
    starts, ends = list(starts), list(ends)
    if contents is None:
        contents = ["x"] * len(starts)
    return [Cue(timedelta(seconds=float(s)), timedelta(seconds=float(e)), c)
            for s, e, c in zip(starts, ends, contents)]


class SubtitleScaler(TransformerMixin):
    def __init__(self, scale_factor) -> None:
        assert isinstance(scale_factor, numbers.Number)
        self.scale_factor = scale_factor
        self.subs_ = None

    def fit(self, subs, *_) -> "SubtitleScaler":
        scaled = []
        for sub in subs:
            start = timedelta(seconds=sub.start.total_seconds() * self.scale_factor)
            end = timedelta(seconds=sub.end.total_seconds() * self.scale_factor)
            scaled.append(type(sub)(start, end, sub.inner))
        # the reference keeps the file-level properties (encoding, format) of its container
        self.subs_ = subs.clone_props_for_subs(scaled) if hasattr(subs, "clone_props_for_subs") else scaled
        return self

    def transform(self, *_):
        return self.subs_


class SubtitleShifter(TransformerMixin):
    """The reference's SubtitleShifter (ffsubsync/subtitle_transformers.py:13-26): every cue moved by
    ``timedelta(seconds=td_seconds)`` (or the timedelta given), for the single-pair Pipeline.  The batched calls'
    output step is b2_apply_sync (sync_output.py), which reproduces this rounding on the GPU."""

    def __init__(self, td_seconds) -> None:
        self.td_seconds = td_seconds if isinstance(td_seconds, timedelta) else timedelta(seconds=td_seconds)
        self.subs_ = None

    def fit(self, subs, *_) -> "SubtitleShifter":
        if hasattr(subs, "offset"):   # the reference's GenericSubtitlesFile
            self.subs_ = subs.offset(self.td_seconds)
        else:
            self.subs_ = [type(s)(s.start + self.td_seconds, s.end + self.td_seconds, s.inner) for s in subs]
        return self

    def transform(self, *_):
        return self.subs_
