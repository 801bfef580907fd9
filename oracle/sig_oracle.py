"""Float64 restatement of the serialized-speech reference (ffsubsync/speech_transformers.py:987-1009,
DeserializeSpeechTransformer) as the batched sync calls apply it (b2_sync_tracks_sig, csrc/sig_ref.cuh).

The reference loads the stored array (np.load: float64 for every artefact it writes) and sets every value < 1.0 to
the non-speech label; the batched calls round that result once to float32.  Their domain is x < 1.0 or x == 1.0."""
import numpy as np


def deserialize(x, label: float) -> np.ndarray:
    """DeserializeSpeechTransformer(label) on the stored float64 values x: float64."""
    x = np.array(x, dtype=np.float64)
    x[x < 1.0] = label
    return x


def frames(x, label: float) -> np.ndarray:
    """The reference frames of a signal video: the rule in float64, rounded once to float32."""
    return deserialize(x, label).astype(np.float32)


def out_of_domain(x) -> np.ndarray:
    """Values outside the domain (> 1.0 or NaN)."""
    return ~(np.asarray(x, dtype=np.float64) <= 1.0)


def first_bad_frame(x) -> int:
    """The first out-of-domain frame, -1 when there is none."""
    bad = np.flatnonzero(out_of_domain(x))
    return int(bad[0]) if len(bad) else -1


def packed_words(f) -> np.ndarray:
    """ceil(R/32) uint32 words of the bits m = (f == 1.0f), frame 32w + l at bit l, zero bits past R."""
    m = np.asarray(f, dtype=np.float32) == np.float32(1.0)
    W = (len(m) + 31) // 32
    bits = np.zeros(W * 32, dtype=np.uint64)
    bits[: len(m)] = m
    return (bits.reshape(W, 32) << np.arange(32, dtype=np.uint64)).sum(axis=1).astype(np.uint32)


def stored_signal(golden, name: str) -> np.ndarray:
    """The stored float64 values of fixture signal `name` (tests/golden/signal_ref.json's "stored" table)."""
    s = [r for r in golden["stored"] if r["name"] == name][0]
    return from_runs(s["levels"], s["starts"], s["length"])


def from_runs(levels, starts, length: int) -> np.ndarray:
    """float64 signal of `length` frames from run lengths (levels, starts) as tests/golden/signal_ref.json keeps
    them (levels may be repr strings such as '-inf')."""
    x = np.empty(length, dtype=np.float64)
    bounds = list(starts) + [length]
    for lv, a, b in zip(levels, bounds[:-1], bounds[1:]):
        x[a:b] = float(lv)
    return x
