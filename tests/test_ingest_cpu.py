"""CPU suite for the batched ingest session's span planner (csrc/ingest_plan.h), run through
tests/host_emul/ingest_emul: under random push sequences the spans tile each video's stream exactly, start on a window
boundary of their detector call and end on one or at the call's end, never cross a call, write the frames the one-shot
detector gives those samples, and hold back exactly the unfinished window until the stream ends."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT

EMUL = os.path.join(ROOT, "tests", "host_emul", "ingest_emul")


def _run(V, fpw, auditok, chunk, ops, db=50.0):
    """ops: ("p", v, n_bytes) or ("f", v).  Returns (per op: (spans [(v, s0, s1, frame, tail)], calls [(v, f0, f1)]),
    frames [V], base [V])."""
    if not os.path.exists(EMUL):
        import sys
        sys.path.insert(0, ROOT)
        import __graft_entry__ as ge
        ge.build()
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            f.write("%d %d %d %d %r\n" % (V, fpw, int(auditok), chunk, db))
            for op in ops:
                f.write(" ".join(str(x) for x in op) + "\n")
        subprocess.check_call([EMUL, src, dst])
        per_op, frames, base = [], None, None
        for line in open(dst).read().splitlines():
            k, *rest = line.split()
            vals = [int(x) for x in rest]
            if k == "op":
                per_op.append(([], []))
            elif k == "s":
                per_op[-1][0].append(tuple(vals))
            elif k == "c":
                per_op[-1][1].append(tuple(vals))
            elif k == "frames":
                frames = vals
            elif k == "base":
                base = vals
        return per_op, frames, base


def _length(n, fpw, chunk):
    if chunk <= 0:
        return -(-n // fpw)
    return n // chunk * -(-chunk // fpw) + -(-(n % chunk) // fpw)


def _held_base(n, fpw, chunk):
    """The first sample of the unfinished window of a stream of n samples (n itself when none is unfinished)."""
    c0 = n // chunk * chunk if chunk > 0 else 0
    return c0 + (n - c0) // fpw * fpw


def _random_ops(rng, V, fpw, chunk):
    """Pushes of 1 byte, odd lengths, less than a window, window- and call-straddling ones and long ones, videos
    interleaved at random; some videos get nothing; every video is finished at the end."""
    ops = []
    sizes = [1, 3, 2 * fpw - 1, 2 * fpw + 1, 2 * fpw * 3, 2 * (chunk or 7 * fpw) + 5, 2 * (chunk or 11 * fpw) * 2 + 1]
    for _ in range(rng.randint(10, 60)):
        v = int(rng.randint(V))
        nb = int(sizes[rng.randint(len(sizes))] if rng.rand() < 0.6 else rng.randint(0, 4 * fpw * 8))
        ops.append(("p", v, nb))
    ops += [("f", v) for v in range(V)]
    return ops


@pytest.mark.parametrize("auditok,fpw,chunk", [(False, 160, 0), (False, 480, 0), (False, 7, 30), (False, 221, 2205),
                                               (True, 160, 0), (True, 160, 1600), (True, 160, 1000), (True, 80, 333),
                                               (True, 480, 4800)])
@pytest.mark.parametrize("seed", range(6))
def test_spans_tile_the_stream_at_window_and_call_boundaries(auditok, fpw, chunk, seed):
    rng = np.random.RandomState(seed * 101 + fpw + chunk)
    V = 4
    check_spans(V, fpw, auditok, chunk, _random_ops(rng, V, fpw, chunk))


def check_spans(V, fpw, auditok, chunk, ops):
    """Runs ops through the planner and checks every span and completed call it returns against the stream's
    window and call grid."""
    per_op, frames, base = _run(V, fpw, auditok, chunk, ops)
    c = chunk   # energy / ZCR too: its calls where they do not divide into windows (b2_vad_call_samples)
    per_call = -(-c // fpw) if c > 0 else 0
    nbytes = [0] * V
    at = [0] * V                      # next sample each video's spans must start at
    fr = [0] * V                      # frames written so far
    calls = {v: [] for v in range(V)}
    for op, (spans, done_calls) in zip(ops, per_op):
        v = op[1]
        final = op[0] == "f"
        if not final:
            nbytes[v] += op[2]
        n = nbytes[v] // 2
        for (w, s0, s1, frame, tail) in spans:
            assert w == v and s0 == at[v] and s1 > s0
            c0 = s0 // c * c if c > 0 else 0
            c1 = c0 + c if c > 0 else None
            assert (s0 - c0) % fpw == 0                              # starts on a window of its detector call
            assert c1 is None or s1 <= c1                            # never crosses a call
            closes = (c1 is not None and s1 == c1) or (final and s1 == n)
            assert (s1 - c0) % fpw == 0 or closes                    # ends on a window or where the call ends
            assert frame == (s0 // c) * per_call + (s0 - c0) // fpw if c > 0 else frame == s0 // fpw
            assert frame == fr[v]
            assert (tail > 0) == (auditok and (s1 - c0) % fpw != 0)  # a call's short last block: its own floor
            fr[v] = frame + -(-(s1 - s0) // fpw)
            at[v] = s1
        for (w, f0, f1) in done_calls:
            assert w == v
            calls[v].append((f0, f1))
        if final:
            assert at[v] == n and fr[v] == _length(n, fpw, c)      # the whole stream, the one-shot detector's frames
        else:
            assert at[v] == _held_base(n, fpw, c)                   # exactly the unfinished window held back
    assert frames == fr and base == at
    for v in range(V):
        n = nbytes[v] // 2
        if not auditok:
            assert calls[v] == []
            continue
        # every detector call of the stream, each once, in order: the tokenizer's chunks
        want, s = [], 0
        while s < n:
            e = min(n, s + c) if c > 0 else n
            k = s // c if c > 0 else 0
            want.append((k * per_call, k * per_call + -(-(e - s) // fpw)))
            s = e
        assert calls[v] == want


def test_a_call_completes_in_the_push_that_ends_it():
    """auditok, 1000-sample calls of 160-sample blocks: a push that reaches a call's end closes the call (its short
    last block and its tokenizer chunk) at once; a push that stops short holds the unfinished block back."""
    per_op, frames, base = _run(1, 160, True, 1000, [("p", 0, 2 * 990), ("p", 0, 2 * 10), ("p", 0, 2 * 170),
                                                     ("f", 0)])
    assert per_op[0] == ([(0, 0, 960, 0, 0)], [])
    spans, calls = per_op[1]
    assert [s[:4] for s in spans] == [(0, 960, 1000, 6)] and spans[0][4] > 0 and calls == [(0, 0, 7)]
    assert per_op[2] == ([(0, 1000, 1160, 7, 0)], [])
    spans, calls = per_op[3]
    assert [s[:4] for s in spans] == [(0, 1160, 1170, 8)] and calls == [(0, 7, 9)]
    assert frames == [9] and base == [1170]


def test_odd_bytes_join_the_next_push():
    per_op, frames, base = _run(2, 160, False, 0, [("p", 0, 1)] * 321 + [("p", 1, 3), ("f", 0), ("f", 1)])
    spans = [s for sp, _ in per_op for s in sp]
    assert spans == [(0, 0, 160, 0, 0), (1, 0, 1, 0, 0)]
    assert frames == [1, 1] and base == [160, 1]


def test_the_flush_closes_a_call_without_a_span():
    """auditok: a stream that ends on a window boundary inside a detector call holds nothing back, so the end of the
    stream adds no span, yet it closes the call: its tokenizer chunk must still run."""
    per_op, frames, base = _run(1, 160, True, 1600000, [("p", 0, 3200), ("f", 0)])
    assert per_op[0] == ([(0, 0, 1600, 0, 0)], [])
    assert per_op[1] == ([], [(0, 0, 10)])
    assert frames == [10] and base == [1600]
