"""CPU suite for the host half of b2_ingest_sync_refs (csrc/ingest_plan.h ingest_refs_check, csrc/sync_plan.h with
SyncRequest::ready and reference tables), run through tests/host_emul/ingest_refs_emul: a session's pushes, the check
that no text, PGS or signal video took pushed bytes, and the plan of the sync.  Each video's reference length equals
the whole call's (plan_emul over the pushed samples back to back): the pushes' frames for audio videos,
int(max_end * sr) + 2 for text and PGS, the stored length for signals, int(total * sr) + 2 for segment videos.  The
combinations the whole call refuses are refused here with the same messages."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from sync_plan import plan

EMUL = os.path.join(ROOT, "tests", "host_emul", "ingest_refs_emul")
GRID = [0.96, 1.0, 1.04]
FR, SR = 16000, 100


def _run(**req):
    """req: the fields ingest_refs_emul.cu reads.  Returns {"status", "err", tables as int64 arrays, "two_level",
    "ref_label"}."""
    if not os.path.exists(EMUL):
        import sys
        sys.path.insert(0, ROOT)
        import __graft_entry__ as ge
        ge.build()
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            for k, v in req.items():
                if v is None:
                    continue
                vals = [v] if np.isscalar(v) else list(np.asarray(v).ravel())
                f.write("%s %d %s\n" % (k, len(vals), " ".join(repr(float(x)) if isinstance(x, (float, np.floating))
                                                              else str(int(x)) for x in vals)))
        subprocess.check_call([EMUL, src, dst])
        out = {}
        for line in open(dst).read().splitlines():
            k, _, rest = line.partition(" ")
            if k == "status":
                out[k] = int(rest)
            elif k == "err":
                out[k] = rest
            elif k == "two_level":
                a, b = rest.split()
                out[k], out["ref_label"] = bool(int(a)), float(b)
            else:
                out[k] = np.array([int(x) for x in rest.split()], dtype=np.int64)
        return out


def _tracks(V, rng):
    tv = np.arange(V, dtype=np.int32)
    starts = np.sort(rng.uniform(0, 50, (V, 4)), axis=1).ravel()
    return dict(track_video=tv, cue_start=starts, cue_end=starts + 1.5, cue_off=np.arange(V + 1) * 4, ratios=GRID)


def _library(seed, V=8):
    """A mixed library: per video its kind ("audio", "text", "pgs", "sig") and the tables of both calls."""
    rng = np.random.RandomState(seed)
    kinds = [["audio", "text", "pgs", "sig"][i % 4] for i in range(V)]
    rng.shuffle(kinds)
    samples = [int(rng.randint(0, 40 * FR)) if k == "audio" else 0 for k in kinds]
    is_subs = np.array([k == "text" for k in kinds], np.uint8)
    is_pgs = np.array([k == "pgs" for k in kinds], np.uint8)
    is_sig = np.array([k == "sig" for k in kinds], np.uint8)
    ncue = [int(rng.randint(1, 6)) if k == "text" else 0 for k in kinds]
    npgs = [int(rng.randint(1, 6)) if k == "pgs" else 0 for k in kinds]
    nsig = [int(rng.randint(0, 3000)) if k == "sig" else 0 for k in kinds]
    rs = rng.uniform(0, 60, sum(ncue))
    ps = rng.uniform(0, 60, sum(npgs))
    tables = dict(ref_is_subs=is_subs, ref_cue_start=rs, ref_cue_end=rs + rng.uniform(0.1, 3, len(rs)),
                  ref_cue_off=np.concatenate([[0], np.cumsum(ncue)]), ref_is_pgs=is_pgs, pgs_start=ps,
                  pgs_end=ps + rng.uniform(0.1, 3, len(ps)), pgs_off=np.concatenate([[0], np.cumsum(npgs)]),
                  ref_is_sig=is_sig, sig_off=np.concatenate([[0], np.cumsum(nsig)]))
    return kinds, samples, tables, rng


def _pushes(samples, rng):
    """Random cuts of every audio video's bytes (a video's push sizes in any order), interleaved across videos:
    (push_video, push_bytes)."""
    order = []
    for v, n in enumerate(samples):
        left = 2 * n
        while left > 0:
            m = min(left, int(rng.choice([1, 3, 321, 2 * FR + 1, 200 * FR])))
            order.append((v, m))
            left -= m
    rng.shuffle(order)
    return [v for v, _ in order], [m for _, m in order]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("auditok", [False, True])
def test_reference_lengths_equal_the_whole_call(seed, auditok):
    kinds, samples, tables, rng = _library(seed)
    V = len(kinds)
    det = dict(detector=1 if auditok else 0, chunk_samples=100 * FR if auditok else 0, frame_rate=FR, sample_rate=SR)
    pv, pb = _pushes(samples, rng)
    trk = _tracks(V, rng)
    got = _run(V=V, push_video=pv, push_bytes=pb, **det, **tables, **trk)
    assert got["status"] == 0, got["err"]
    want = plan(pcm_off=np.concatenate([[0], np.cumsum(samples)]), **det, **tables, **trk,
                auditok_label=0.0, pcm=1)
    assert want["status"] == 0, want["err"]
    assert np.array_equal(got["ref_off"], want["ref_off"])
    for k in ("sub_video", "pgs_video", "sig_video"):
        assert np.array_equal(got[k], want[k]), k
    lens = np.diff(got["ref_off"])
    for v, k in enumerate(kinds):
        if k == "sig":
            assert lens[v] == tables["sig_off"][v + 1] - tables["sig_off"][v]
        elif k == "text":
            c0, c1 = tables["ref_cue_off"][v], tables["ref_cue_off"][v + 1]
            assert lens[v] == int(tables["ref_cue_end"][c0:c1].max() * SR) + 2
        elif k == "pgs":
            c0, c1 = tables["pgs_off"][v], tables["pgs_off"][v + 1]
            assert lens[v] == int(tables["pgs_end"][c0:c1].max() * SR) + 2
    assert got["two_level"] == want["two_level"] and got["ref_label"] == want["ref_label"]


def test_segment_videos_beside_references_keep_their_lengths():
    kinds, samples, tables, rng = _library(11, V=6)
    audio = [v for v, k in enumerate(kinds) if k == "audio"]
    seg = audio[:1]
    samples[seg[0]] = 0
    pv, pb = _pushes(samples, rng)
    got = _run(V=6, push_video=pv, push_bytes=pb, seg_video=seg, seg_total=[301.5], seg_off=[0, 2],
               seg_start=[0, 120], **tables, **_tracks(6, rng))
    assert got["status"] == 0, got["err"]
    assert np.diff(got["ref_off"])[seg[0]] == int(301.5 * SR) + 2
    assert got["seg_video"].tolist() == seg


@pytest.mark.parametrize("kind", ["text", "pgs", "sig"])
def test_a_pushed_reference_video_is_refused_by_name(kind):
    kinds, samples, tables, rng = _library(3)
    v = kinds.index(kind)
    pv, pb = _pushes(samples, rng)
    pv, pb = pv + [v, v], pb + [1, 6]
    got = _run(V=len(kinds), push_video=pv, push_bytes=pb, **tables, **_tracks(len(kinds), rng))
    what = {"text": "text subtitle", "pgs": "PGS", "sig": "serialized signal"}[kind]
    assert got["status"] == -1
    assert got["err"] == ("ingest_sync_refs: video %d has a %s reference and received 7 pushed bytes; its audio is "
                          "never read, so it takes no pushes" % (v, what))
    # an empty push leaves P_v empty: accepted
    got = _run(V=len(kinds), push_video=pv[:-2] + [v], push_bytes=pb[:-2] + [0], **tables,
               **_tracks(len(kinds), rng))
    assert got["status"] == 0, got["err"]


def test_the_whole_calls_combination_refusals():
    kinds, samples, tables, rng = _library(5)
    V = len(kinds)
    trk = _tracks(V, rng)
    pv, pb = _pushes(samples, rng)
    sig = kinds.index("sig")
    # a video both text and signal: the whole call's message
    both = dict(tables, ref_is_subs=tables["ref_is_subs"].copy())
    both["ref_is_subs"][sig] = 1
    off = tables["ref_cue_off"]
    both["ref_cue_off"] = off   # no cues of its own: the flags alone make it both
    got = _run(V=V, push_video=pv, push_bytes=pb, **both, **trk)
    assert got["status"] == -1
    assert got["err"] == "ingest_sync_refs: video %d is marked both as a signal and as a text subtitle reference" % sig
    # a segment video given a reference
    pgs = kinds.index("pgs")
    got = _run(V=V, push_video=pv, push_bytes=pb, seg_video=[pgs], seg_total=[100.0], seg_off=[0, 1], seg_start=[0],
               **tables, **trk)
    assert got["status"] == -1
    assert got["err"] == ("ingest_sync_refs: video %d has sampled segments and a PGS reference; a video has one "
                          "reference" % pgs)
    # the search at a non-zero label with text references: the whole call's B2_ERR_UNSUPPORTED and message
    got = _run(V=V, push_video=pv, push_bytes=pb, label=0.3, gss=1, **tables, **trk)
    want = plan(pcm_off=np.concatenate([[0], np.cumsum(samples)]), label=0.3, gss=1, pcm=1, who="x", **tables, **trk)
    assert got["status"] == want["status"] == -6
    assert got["err"].split(": ", 1)[1] == want["err"].split(": ", 1)[1]
    assert got["err"].startswith("ingest_sync_refs (search): ")
    # a bad PGS list: the whole call's message
    bad = dict(tables, pgs_end=tables["pgs_end"].copy())
    bad["pgs_end"][tables["pgs_off"][pgs]] = np.inf
    got = _run(V=V, push_video=pv, push_bytes=pb, **bad, **trk)
    want = plan(pcm_off=np.concatenate([[0], np.cumsum(samples)]), pcm=1, who="x", **bad, **trk)
    assert got["status"] == want["status"] == -1
    assert got["err"].split(": ", 1)[1] == want["err"].split(": ", 1)[1]


def test_signal_only_sessions_keep_the_packed_reference():
    kinds, samples, tables, rng = _library(7, V=4)
    sig_only = dict(ref_is_sig=np.ones(4, np.uint8), sig_off=np.arange(5) * 2000)
    got = _run(V=4, lane=1, **sig_only, **_tracks(4, rng))
    assert got["status"] == 0, got["err"]
    want = plan(pcm_off=np.zeros(5, np.int64), lane=1, **sig_only, **_tracks(4, np.random.RandomState(7)))
    assert got["ref_packed"].tolist() == want["ref_packed"].tolist()
    # an audio video among them: the ingested floats
    got = _run(V=5, lane=1, push_video=[4], push_bytes=[2 * FR], ref_is_sig=[1, 1, 1, 1, 0],
               sig_off=[0, 2000, 4000, 6000, 8000, 8000], **_tracks(5, rng))
    assert got["status"] == 0 and got["ref_packed"].tolist() == [0]
