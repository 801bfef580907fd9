"""CPU restatement of the reference's auditok detector (TEST INFRASTRUCTURE ONLY).

What is restated, and from where
--------------------------------
* ``_make_auditok_detector._detect`` - /root/reference/ffsubsync/speech_transformers.py:101-152
  (present in the reference tree; restated line by line in ``auditok_detect``).
* The third-party arithmetic it calls lives in ``auditok==0.1.5`` (pinned in
  /root/reference/requirements.txt:1), which is NOT installed in this image and not vendored in
  the reference.  Its published algorithm (auditok 0.1.5, ``auditok/util.py``:
  ``AudioEnergyValidator``, ``BufferAudioSource``, ``ADSFactory.ads``; ``auditok/core.py``:
  ``StreamTokenizer``) is restated here from its documentation:

    - ``ADSFactory.ads(block_dur=d)`` reads blocks of ``int(sampling_rate * d)`` samples; the last
      block of a buffer may be shorter; ``BufferAudioSource`` rejects a buffer whose length is not
      a multiple of the sample width.
    - ``AudioEnergyValidator(sample_width=2, energy_threshold=T).is_valid(block)``:
      ``x = float64(int16 samples)``; ``energy = dot(x, x) / len(x)``;
      ``log_energy = 10 * log10(energy)`` (``-200`` when ``energy <= 0``); valid iff
      ``log_energy >= T``.
    - ``StreamTokenizer(validator, min_length, max_length, max_continuous_silence)`` (default
      ``init_min = init_max_silence = 0``, ``mode = 0``): the four-state machine SILENCE /
      POSSIBLE_NOISE / NOISE / POSSIBLE_SILENCE over the per-block validity; a token is delivered
      as ``(data, start_frame, end_frame)`` and INCLUDES up to ``max_continuous_silence`` trailing
      non-valid frames; a token that reaches ``max_length`` is delivered ("truncated") and the
      next one starts at the following frame and is delivered even when shorter than
      ``min_length`` (contiguous token, non-strict mode); ``tokenize()`` resets the machine.

Pins (tests/test_oracle_golden.py::test_auditok_*): the known-answer examples of the
``StreamTokenizer`` documentation / test-suite of auditok 0.1.5 - quoted from memory because the
package cannot be installed here (no network) - which this restatement reproduces:

    "aaaAAAABBbbb"     min 1 max 9999 silence 0  ->  [(3, 8)]
    "aaaAAAABBbbb"     min 3 max 4    silence 0  ->  [(3, 6), (7, 8)]       (contiguous short token kept)
    "aaaAAAaaaBBbbbb"  min 3 max 6    silence 3  ->  [(3, 8), (9, 13)]      (trailing silence included)
    "aAaaaAaAaaAaAaaaaaaaAAAAAAAA" min 5 max 20 silence 4 -> [(1, 16), (20, 27)]

(valid = upper case).  The energy rule is additionally pinned arithmetically: for int16 blocks
``10*log10(E/n) >= 50  <=>  E >= n * 10**5`` (E = integer sum of squares), checked over random blocks
straddling the edge.  PARITY STATUS: pinned to the dependency's published algorithm and examples,
not to an execution of the dependency.
"""
from typing import List, Sequence, Tuple

import numpy as np

SILENCE, POSSIBLE_NOISE, NOISE, POSSIBLE_SILENCE = 0, 1, 2, 3


# ------------------------------------------------------------------------------ energy validator

def block_log_energy(block: np.ndarray) -> float:
    """AudioEnergyValidator._signal_log_energy for one block of int16 samples."""
    x = np.array(np.asarray(block, dtype=np.int16), dtype=np.float64)
    energy = float(np.dot(x, x)) / len(x)
    if energy <= 0:
        return -200.0
    return float(10.0 * np.log10(energy))


def block_is_valid(block: np.ndarray, energy_threshold: float = 50) -> bool:
    return block_log_energy(block) >= energy_threshold


def energy_floor(n_samples: int, energy_threshold: float = 50) -> int:
    """Smallest integer sum of squares E for which a block of ``n_samples`` is valid, found by
    evaluating the validator's own float64 expression (monotone in E)."""
    def valid(e: int) -> bool:
        if e <= 0:
            return -200.0 >= energy_threshold
        return float(10.0 * np.log10(float(e) / n_samples)) >= energy_threshold

    if valid(0):
        return 0
    hi = max(1, int(n_samples * 10.0 ** (energy_threshold / 10.0)))
    while not valid(hi):
        hi *= 2
    lo = 0  # invariant: not valid(lo), valid(hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if valid(mid):
            hi = mid
        else:
            lo = mid
    return hi


def read_blocks(pcm: np.ndarray, block_size: int) -> List[np.ndarray]:
    """ADSFactory.ads(...).read() until None: consecutive blocks, a shorter last one included."""
    return [pcm[i:i + block_size] for i in range(0, len(pcm), block_size)]


# ----------------------------------------------------------------------------------- tokenizer

def tokenize(valid: Sequence[bool], min_length: float, max_length: int, max_continuous_silence: float,
             init_min: int = 0, init_max_silence: int = 0) -> List[Tuple[int, int]]:
    """StreamTokenizer(...).tokenize() over per-frame validity -> [(start_frame, end_frame)].

    Only what the reference configures is modelled (mode 0: no STRICT_MIN_LENGTH, no
    DROP_TRAILING_SILENCE); ``init_min`` / ``init_max_silence`` are kept for the general machine."""
    if max_length <= 0 or min_length <= 0 or min_length > max_length:
        raise ValueError("bad min_length / max_length")
    if max_continuous_silence >= max_length or init_min >= max_length:
        raise ValueError("bad max_continuous_silence / init_min")
    tokens: List[Tuple[int, int]] = []
    st = {"state": SILENCE, "n": 0, "sil": 0, "init": 0, "start": 0, "contig": False, "cur": -1}

    def end_of_detection(truncated: bool) -> None:
        n = st["n"]
        if n >= min_length or (n > 0 and st["contig"]):
            tokens.append((st["start"], st["start"] + n - 1))
            if truncated:
                st["start"] = st["cur"] + 1
                st["contig"] = True
            else:
                st["contig"] = False
        else:
            st["contig"] = False
        st["n"] = 0

    for cur, ok in enumerate(valid):
        st["cur"] = cur
        state = st["state"]
        if state == SILENCE:
            if ok:
                st["init"], st["sil"], st["start"] = 1, 0, cur
                st["n"] += 1
                if st["init"] >= init_min:
                    st["state"] = NOISE
                    if st["n"] >= max_length:
                        end_of_detection(True)
                else:
                    st["state"] = POSSIBLE_NOISE
        elif state == POSSIBLE_NOISE:
            if ok:
                st["sil"] = 0
                st["init"] += 1
                st["n"] += 1
                if st["init"] >= init_min:
                    st["state"] = NOISE
                    if st["n"] >= max_length:
                        end_of_detection(True)
            else:
                st["sil"] += 1
                if st["sil"] > init_max_silence or st["n"] + 1 >= max_length:
                    st["n"] = 0
                    st["state"] = SILENCE
                else:
                    st["n"] += 1
        elif state == NOISE:
            if ok:
                st["n"] += 1
                if st["n"] >= max_length:
                    end_of_detection(True)
            elif max_continuous_silence <= 0:
                end_of_detection(False)
                st["state"] = SILENCE
            else:
                st["sil"] = 1
                st["n"] += 1
                st["state"] = POSSIBLE_SILENCE
                if st["n"] == max_length:
                    end_of_detection(True)   # the silence count is deliberately kept
        else:  # POSSIBLE_SILENCE
            if ok:
                st["n"] += 1
                st["sil"] = 0
                st["state"] = NOISE
                if st["n"] >= max_length:
                    end_of_detection(True)
            elif st["sil"] >= max_continuous_silence:
                if st["sil"] < st["n"]:
                    end_of_detection(False)
                else:
                    st["n"] = 0
                st["state"] = SILENCE
                st["sil"] = 0
            else:
                st["n"] += 1
                st["sil"] += 1
                if st["n"] >= max_length:
                    end_of_detection(True)   # the silence count is deliberately kept
    if st["state"] in (NOISE, POSSIBLE_SILENCE) and st["n"] > 0 and st["n"] > st["sil"]:
        end_of_detection(False)
    return tokens


# ------------------------------------------------------------------- the reference's _detect

def auditok_detect(asegment, sample_rate: int = 100, frame_rate: int = 16000, non_speech_label: float = 0.0,
                   energy_threshold: float = 50) -> np.ndarray:
    """One call of the closure returned by _make_auditok_detector(sample_rate, frame_rate,
    non_speech_label) (speech_transformers.py:133-150) on one chunk of s16le bytes."""
    if isinstance(asegment, (bytes, bytearray, memoryview)):
        raw = np.frombuffer(asegment, dtype=np.uint8)
    else:
        raw = np.asarray(asegment)
        if raw.dtype != np.uint8:
            raw = np.ascontiguousarray(raw).view(np.uint8)
    bytes_per_frame = 2
    if len(raw) % bytes_per_frame != 0:   # BufferAudioSource.__init__
        raise ValueError("length of data_buffer must be a multiple of (sample_width * channels)")
    frames_per_window = frame_rate // sample_rate                       # :122
    block_size = int(frame_rate * (1.0 / sample_rate))                   # ADSFactory.ads(block_dur=1.0/sample_rate), :140
    pcm = raw.view("<i2")
    valid = [block_is_valid(b, energy_threshold) for b in read_blocks(pcm, block_size)]
    tokens = tokenize(valid, min_length=0.2 * sample_rate, max_length=int(5 * sample_rate),
                      max_continuous_silence=0.25 * sample_rate)        # :126-131
    length = (len(raw) // bytes_per_frame + frames_per_window - 1) // frames_per_window   # :143-145
    media_bstring = np.zeros(length + 1)
    for start, end in tokens:                                             # :147-149 (assignment, not +=)
        media_bstring[start] = 1.0
        media_bstring[end + 1] = non_speech_label - 1.0
    return np.clip(np.cumsum(media_bstring)[:-1], 0.0, 1.0)              # :150


def auditok_detect_fast(asegment, sample_rate: int = 100, frame_rate: int = 16000, non_speech_label: float = 0.0,
                        energy_threshold: float = 50, min_length=None, max_length=None,
                        max_continuous_silence=None) -> np.ndarray:
    """Same result as ``auditok_detect`` with the per-block validity vectorised through the integer
    energy floor (tests check the two agree); used for the long (250 s ... 2 h) parity inputs.  The
    tokenizer parameters (in blocks) default to the reference's 0.2 s, 5 s and 0.25 s."""
    raw = np.frombuffer(asegment, dtype=np.uint8) if isinstance(asegment, (bytes, bytearray, memoryview)) \
        else np.ascontiguousarray(asegment).view(np.uint8)
    if len(raw) % 2 != 0:
        raise ValueError("length of data_buffer must be a multiple of (sample_width * channels)")
    frames_per_window = frame_rate // sample_rate
    block_size = int(frame_rate * (1.0 / sample_rate))
    pcm = raw.view("<i2").astype(np.int64)
    n_full = len(pcm) // block_size
    energy = (pcm[: n_full * block_size].reshape(n_full, block_size) ** 2).sum(axis=1)
    valid = list(energy >= energy_floor(block_size, energy_threshold))
    tail = pcm[n_full * block_size:]
    if len(tail):
        valid.append(bool((tail * tail).sum() >= energy_floor(len(tail), energy_threshold)))
    tokens = tokenize(valid, 0.2 * sample_rate if min_length is None else min_length,
                      int(5 * sample_rate) if max_length is None else int(max_length),
                      0.25 * sample_rate if max_continuous_silence is None else max_continuous_silence)
    length = (len(raw) // 2 + frames_per_window - 1) // frames_per_window
    media_bstring = np.zeros(length + 1)
    for start, end in tokens:
        media_bstring[start] = 1.0
        media_bstring[end + 1] = non_speech_label - 1.0
    return np.clip(np.cumsum(media_bstring)[:-1], 0.0, 1.0)
