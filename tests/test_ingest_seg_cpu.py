"""CPU suite for the ingest session's streams with sampled segments (csrc/ingest_plan.h IngestStreams feeding the
per-stream IngestPlanner), run through tests/host_emul/ingest_seg_emul: under random push sequences that interleave
audio videos and segments, every live segment's spans tile its own stream and write the frames the one-shot detector
gives its samples (its windows, or auditok's calls restarting at the segment's first sample), interleaving changes
nothing, windows() counts the live segments, and every refusal leaves the state as it was."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT

EMUL = os.path.join(ROOT, "tests", "host_emul", "ingest_seg_emul")


def _run(V, fpw, auditok, chunk, ops, db=50.0, sr=100):
    """ops: ("S", videos, totals, off, starts), ("p", [(v, nb)]), ("q", [(v, j, nb)]), ("d", v, j) or ("f",).
    Returns (per op: (status, message, spans [(k, s0, s1, frame, tail)], calls [(k, f0, f1)], windows [V]),
    streams [(live, frames)])."""
    if not os.path.exists(EMUL):
        import sys
        sys.path.insert(0, ROOT)
        import __graft_entry__ as ge
        ge.build()
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            f.write("%d %d %d %d %r %d\n" % (V, fpw, int(auditok), chunk, db, sr))
            for op in ops:
                if op[0] == "S":
                    _, vid, tot, off, st = op
                    f.write(" ".join(["S", str(len(vid))] + [str(x) for x in vid] + [repr(float(x)) for x in tot]
                                     + [str(x) for x in off] + [str(x) for x in st]) + "\n")
                elif op[0] in "pq":
                    f.write(" ".join([op[0], str(len(op[1]))] + [str(x) for c in op[1] for x in c]) + "\n")
                else:
                    f.write(" ".join(str(x) for x in op) + "\n")
        subprocess.check_call([EMUL, src, dst])
        per_op, streams = [], []
        for line in open(dst).read().splitlines():
            k, _, rest = line.partition(" ")
            if k == "op":
                per_op.append([int(rest.split()[1]), None, [], [], None])
            elif k == "e":
                per_op[-1][1] = rest
            elif k == "s":
                per_op[-1][2].append(tuple(int(x) for x in rest.split()))
            elif k == "c":
                per_op[-1][3].append(tuple(int(x) for x in rest.split()))
            elif k == "w":
                per_op[-1][4] = [int(x) for x in rest.split()]
            elif k == "k":
                streams.append(tuple(int(x) for x in rest.split()))
        return per_op, streams


def _length(n, fpw, chunk):
    if chunk <= 0:
        return -(-n // fpw)
    return n // chunk * -(-chunk // fpw) + -(-(n % chunk) // fpw)


def _calls(n, fpw, chunk):
    """The detector calls (f0, f1) of a stream of n samples, in order."""
    per_call = -(-chunk // fpw) if chunk > 0 else 0
    out, s = [], 0
    while s < n:
        e = min(n, s + chunk) if chunk > 0 else n
        k = s // chunk if chunk > 0 else 0
        out.append((k * per_call, k * per_call + -(-(e - s) // fpw)))
        s = e
    return out


# videos 1 and 3 have segments (3 and 2), videos 0 and 2 are audio
TABLE = ("S", [1, 3], [300.0, 50.0], [0, 3, 5], [0, 120, 240, 0, 30])
SEGS = {1: 3, 3: 2}


def _random_ops(rng, fpw, chunk):
    """Pushes of 1 byte, odd lengths, sub-window, window- and call-straddling and long ones, to audio videos and
    segments in random order and batches; a few segments dropped part-way; one never pushed; then the flush."""
    sizes = [1, 3, 2 * fpw - 1, 2 * fpw + 1, 2 * fpw * 3, 2 * (chunk or 7 * fpw) + 5, 2 * (chunk or 11 * fpw) * 2 + 1]
    targets = [(0, None), (2, None), (1, 0), (1, 1), (3, 0), (3, 1)]   # (1, 2) is never pushed
    ops, dropped = [TABLE], set()
    for _ in range(rng.randint(10, 60)):
        batch = []
        for _ in range(rng.randint(1, 4)):
            v, j = targets[rng.randint(len(targets))]
            if (v, j) in dropped:
                continue
            nb = int(sizes[rng.randint(len(sizes))] if rng.rand() < 0.6 else rng.randint(0, 4 * fpw * 8))
            batch.append((v, j, nb))
        audio = [(v, nb) for v, j, nb in batch if j is None]
        seg = [(v, j, nb) for v, j, nb in batch if j is not None]
        if audio:
            ops.append(("p", audio))
        if seg:
            ops.append(("q", seg))
        if rng.rand() < 0.05:
            v, j = targets[2 + rng.randint(4)]
            ops.append(("d", v, j))
            dropped.add((v, j))
    ops.append(("f",))
    return ops


def _check(ops, per_op, streams, fpw, chunk, auditok):
    V = 4
    c = chunk if auditok else 0
    first = {1: 0, 3: 3}
    stream = lambda v, j: v if j is None else V + first[v] + j
    nbytes, at, fr, calls = {}, {}, {}, {}
    dropped = set()
    for op, (status, msg, spans, done, windows) in zip(ops, per_op):
        assert status == 0, msg
        if op[0] == "d":
            dropped.add(stream(op[1], op[2]))
        for (v, *rest) in op[1] if op[0] in "pq" else []:
            j, nb = (None, rest[0]) if op[0] == "p" else rest
            k = stream(v, j)
            nbytes[k] = nbytes.get(k, 0) + nb
        for (k, s0, s1, frame, tail) in spans:
            assert k not in dropped
            assert s0 == at.get(k, 0) and s1 > s0
            c0 = s0 // c * c if c > 0 else 0
            assert (s0 - c0) % fpw == 0 and (c == 0 or s1 <= c0 + c)
            assert frame == fr.get(k, 0)
            fr[k] = frame + -(-(s1 - s0) // fpw)
            at[k] = s1
        for (k, f0, f1) in done:
            calls.setdefault(k, []).append((f0, f1))
        # windows: an audio video's frames, a segment video's live segments' together
        want = [fr.get(0, 0), sum(fr.get(stream(1, j), 0) for j in range(3) if stream(1, j) not in dropped),
                fr.get(2, 0), sum(fr.get(stream(3, j), 0) for j in range(2) if stream(3, j) not in dropped)]
        assert windows == want
    # after the flush every live stream is its one-shot detector's output: frames and calls
    assert len(streams) == V + 5
    for k, (live, frames) in enumerate(streams):
        assert live == (k in (0, 2) or (k >= V and k not in dropped))
        if not live:
            continue
        n = nbytes.get(k, 0) // 2
        assert at.get(k, 0) == n and frames == fr.get(k, 0) == _length(n, fpw, c)
        assert calls.get(k, []) == (_calls(n, fpw, c) if auditok else [])
    return {k: (nbytes.get(k, 0), fr.get(k, 0)) for k in range(V + 5) if streams[k][0]}


@pytest.mark.parametrize("auditok,fpw,chunk", [(False, 160, 0), (False, 480, 0), (True, 160, 1600), (True, 80, 333),
                                               (True, 480, 4800)])
@pytest.mark.parametrize("seed", range(6))
def test_segment_streams_tile_at_window_and_call_boundaries(auditok, fpw, chunk, seed):
    rng = np.random.RandomState(seed * 131 + fpw + chunk)
    ops = _random_ops(rng, fpw, chunk)
    per_op, streams = _run(4, fpw, auditok, chunk, ops)
    _check(ops, per_op, streams, fpw, chunk, auditok)


@pytest.mark.parametrize("auditok,fpw,chunk", [(False, 160, 0), (True, 160, 1600)])
def test_interleaving_changes_nothing(auditok, fpw, chunk):
    """The same bytes per stream, cut the same way, pushed stream after stream or interleaved at random across videos
    and segments: every stream ends with the same frames and calls."""
    rng = np.random.RandomState(7)
    per_stream = {t: [int(x) for x in rng.randint(1, 6 * fpw, size=8)] for t in
                  [(0, None), (2, None), (1, 0), (1, 1), (1, 2), (3, 0), (3, 1)]}

    def ops_of(order):
        ops = [TABLE]
        for (v, j), nb in order:
            ops.append(("p", [(v, nb)]) if j is None else ("q", [(v, j, nb)]))
        return ops + [("f",)]

    serial = [(t, nb) for t, sizes in per_stream.items() for nb in sizes]
    queues = {t: list(sizes) for t, sizes in per_stream.items()}
    mixed = []
    while any(queues.values()):
        t = [t for t in queues if queues[t]][rng.randint(len([t for t in queues if queues[t]]))]
        mixed.append((t, queues[t].pop(0)))
    results = []
    for order in (serial, mixed):
        ops = ops_of(order)
        per_op, streams = _run(4, fpw, auditok, chunk, ops)
        results.append((_check(ops, per_op, streams, fpw, chunk, auditok), streams))
    assert results[0] == results[1]


def test_refusals_leave_the_session_as_it_was():
    V = 4
    good = ("q", [(1, 0, 320)])
    cases = [
        (("p", [(0, 10), (1, 10)]), "ingest_push: chunk 1: video 1 has sampled segments"),
        (("q", [(1, 0, 10), (0, 0, 10)]), "ingest_push_segments: chunk 1: video 0 has no sampled segments"),
        (("q", [(1, 3, 10)]), "ingest_push_segments: chunk 0: segment 3 of video 1 is out of [0, 3)"),
        (("q", [(1, -1, 10)]), "ingest_push_segments: chunk 0: segment -1 of video 1 is out of [0, 3)"),
        (("q", [(3, 0, 10), (1, 1, 10)]), "ingest_push_segments: chunk 1: segment 1 of video 1 was dropped"),
        (("p", [(5, 10)]), "ingest_push: chunk 0: video 5 is out of [0, 4)"),
        (("d", 0, 0), "ingest_drop_segment: video 0 has no sampled segments"),
        (("d", 1, 7), "ingest_drop_segment: segment 7 of video 1 is out of [0, 3)"),
        (TABLE, "ingest_segments: the session's segments are already declared"),
    ]
    for bad, msg in cases:
        ops = [TABLE, ("d", 1, 1), ("p", [(0, 100)]), bad, good, ("f",)]
        per_op, streams = _run(V, 160, False, 0, ops)
        assert per_op[3][0] != 0 and per_op[3][1].startswith(msg), (bad, per_op[3][1])
        assert per_op[3][2] == [] and per_op[3][4] == per_op[2][4]
        assert per_op[4][0] == 0 and per_op[4][2] == [(V, 0, 160, 0, 0)]   # the session goes on
        assert [f for _, f in streams] == [1, 0, 0, 0, 1, 0, 0, 0, 0]


@pytest.mark.parametrize("table,msg", [
    (("S", [0, 2], [60.0, 60.0], [0, 1, 2], [0, 0]), "ingest_segments: video 0 already has pushes"),
    (("S", [2, 1], [60.0, 60.0], [0, 1, 2], [0, 0]), "ingest_segments: seg_video[1] = 1 is out of [0, 4) or not "
                                                     "increasing"),
    (("S", [1], [float("nan")], [0, 1], [0]), "ingest_segments: seg_total[0] = nan"),
    (("S", [1], [60.0], [0, 2], [5, 5]), "ingest_segments: segment 1 of video 1 starts at 5 s, not after"),
    (("S", [1], [60.0], [0, 1], [-1]), "ingest_segments: segment 0 of video 1 starts at -1 s, outside"),
    (("S", [1], [60.0], [1, 0], []), "ingest_segments: seg_off not monotone at 0"),
])
def test_bad_tables_are_refused(table, msg):
    """b2_sync_tracks_seg's checks of the table, and a video that already has pushes; the session then takes a good
    table."""
    per_op, streams = _run(4, 160, False, 0, [("p", [(0, 2)]), table, TABLE, ("q", [(3, 1, 320)]), ("f",)])
    assert per_op[1][0] != 0 and per_op[1][1].startswith(msg), per_op[1][1]
    assert per_op[2][0] == 0 and per_op[3][2] == [(4 + 4, 0, 160, 0, 0)]
