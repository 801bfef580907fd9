"""The batched sync calls' host planner (csrc/sync_plan.h) on several hundred seeded random requests
(tests/random_requests.py) through plan_emul: the invariants every plan keeps whatever the request, and the exact
status and message of every bad request the generator makes (about one seed in ten).

Invariants: the sub-batch cuts run from 0 to V, strictly increasing, none without tracks; trk_off is the running sum
of tracks per video; ref_off tiles the reference buffer with each video's length by the oracle of its kind (the
detector's chunk loop, raster_oracle, pgs_oracle, the stored values, segment_oracle); the chunk and tokenizer tables
cover each audio video's samples once, in detector calls that start at multiples of the call length."""
import numpy as np
import pytest

import random_requests as rr
from oracle import raster_oracle as ro
from sync_plan import plan

SEEDS = range(400)
# 22.05 kHz beside the generator's rates: its 100 s read is not a whole number of 221-sample windows, so energy / ZCR
# videos are cut into detector calls and their chunk table is checked too
RATES = rr.RATES + [22050]


def check_plan(req, p):
    vids = req["videos"]
    V = len(vids)
    per = np.bincount([t["video"] for t in req["tracks"]], minlength=V)
    T = int(per.sum())
    trk, cut = p["trk_off"], p["cut"]
    assert np.array_equal(trk, np.concatenate([[0], np.cumsum(per)])), trk
    assert cut[0] == 0 and cut[-1] == V and np.all(np.diff(cut) > 0), cut
    assert np.all(np.diff(trk[cut]) > 0), (cut, trk)                  # no sub-batch without tracks
    assert p["n_sub"][0] == len(cut) - 1 <= max(1, min(T, int(req["knobs"]["B2_SUBBATCHES"])))
    assert len(p["ref_packed"]) == len(cut) - 1
    want = np.array([rr.ref_length(req, d) for d in vids], np.int64)
    assert np.array_equal(p["ref_off"], np.concatenate([[0], np.cumsum(want)])), (p["ref_off"], want)
    for k in ("subs", "pgs", "sig", "seg"):
        got = p.get(k + "_video" if k != "subs" else "sub_video", np.zeros(0, np.int64))
        assert got.tolist() == [v for v, d in enumerate(vids) if d["kind"] == k], k
    # the subtitle signals of every (track, ratio) job, end to end
    lens = [len(ro.rasterize(t["starts"], t["ends"], None, rr.SR, 0.0, r)[0]) for t in req["tracks"]
            for r in req["ratios"]]
    assert np.array_equal(p["sub_off"], np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
    if not p["call"][1]:                                              # one detector call per video: no chunk table
        assert p["ch_pcm"].size == 0 or req["detector"] != "auditok"
        return
    # chunk table: each audio video cut into calls of rr.detector_call samples from its first sample, each a ceil(len / fpw)
    # range of the output; a video with another reference is one chunk over its reference's frames (a segment video's
    # samples are read through its segments' own table)
    fpw, pcm_off = rr.window(req), rr.arrays(req)["pcm_off"]
    first, ch_pcm, ch_out = p["ch_first"], p["ch_pcm"], p["ch_out"]
    any_ref = any(d["kind"] != "audio" for d in vids)
    tok = []
    for v, d in enumerate(vids):
        c0, c1 = int(first[v]), int(first[v + 1])
        assert ch_out[c0] == p["ref_off"][v] and ch_out[c1] == p["ref_off"][v + 1], v
        if d["kind"] != "audio" and any_ref:
            assert c1 - c0 == 1 and (ch_pcm[c0], ch_pcm[c1]) == (pcm_off[v], pcm_off[v + 1]), v
            continue
        n, step = d["n"], rr.detector_call(req, d["n"])
        edges = [pcm_off[v] + min(i, n) for i in range(0, n, step)] + [pcm_off[v + 1]]
        assert ch_pcm[c0:c1 + 1].tolist() == (edges if n else [pcm_off[v]]), (v, ch_pcm[c0:c1 + 1], edges)
        assert np.array_equal(np.diff(ch_out[c0:c1 + 1]), -(-np.diff(ch_pcm[c0:c1 + 1]) // fpw)), v
        tok += [(ch_out[c], ch_out[c + 1]) for c in range(c0, c1)]
    if any_ref:   # the tokenizer's chunks: the audio videos' chunks alone, in order
        assert list(zip(p["tok_off"].tolist(), p["tok_end"].tolist())) == [(int(a), int(b)) for a, b in tok]


# ---------------------------------------------------------------- bad requests: (mutation, status, message check)

def _bad(req, p, rng):
    """A copy of plan request p made invalid in one of the ways the request allows, with its expected status and a
    check of its message."""
    e, who = req["entry"], rr.WHO[req["entry"]]
    q = dict(p)
    ways = ["ratio"]
    if e in ("batch", "tracks", "gss", "auditok") and len(p["pcm_off"]) > 1:
        ways.append("pcm_off")
    if len(p["cue_end"]):
        ways.append("nan_end")
    if e != "batch" and len(p["track_video"]) > 1 and len(set(p["track_video"].tolist())) > 1:
        ways.append("track_video")
    if e == "gss":
        ways.append("gss_mos")
    if e == "auditok":
        ways.append("tokenizer")
    if "ref_is_subs" in p and any(d["kind"] == "audio" and d["n"] > 0 for d in req["videos"]):
        ways.append("subs_pcm")
    way = ways[rng.randint(len(ways))]
    if way == "ratio":
        r = list(p["ratios"])
        r[rng.randint(len(r))] = float(rng.choice([-1.0, 0.0, np.inf, np.nan]))
        q["ratios"] = r
        return q, -1, lambda err: err.startswith(who + ": ") and "ratio is not a finite positive number" in err
    if way == "pcm_off":
        off = np.array(p["pcm_off"])
        v = rng.randint(len(off) - 1)
        off[v + 1] = off[v] - 1
        q["pcm_off"] = off
        return q, -1, lambda err: err == who + ": pcm_off not monotone"
    if way == "nan_end":
        ends = np.array(p["cue_end"])
        i = rng.randint(len(ends))
        ends[i] = np.nan
        q["cue_end"] = ends
        return q, -1, lambda err: (err.startswith(who + ": ") and "cue end time" in err and "index %d:" % i in err)
    if way == "track_video":
        tv = np.array(p["track_video"])
        tv[[0, -1]] = tv[[-1, 0]]                                    # decreasing
        q["track_video"] = tv
        return q, -1, lambda err: "track_video[" in err and "is out of [0, %d) or decreases" % (len(p["pcm_off"]) - 1) in err
    if way == "gss_mos":
        q["max_offset_samples"] = int(rng.choice([rr.GSS_MAX_MOS * 2 + 1, -1, rr.INT64_MIN]))
        return q, -6, lambda err: err.startswith("sync_tracks_gss: max_offset_samples must lie in [0, %d]" % rr.GSS_MAX_MOS)
    if way == "tokenizer":
        q.update(rng.choice([dict(max_length=0), dict(min_length=0.0), dict(max_continuous_silence=500.0)]))
        return q, -1, lambda err: err == "sync_tracks_auditok: bad tokenizer parameters"
    v = [v for v, d in enumerate(req["videos"]) if d["kind"] == "audio" and d["n"] > 0][0]
    subs = np.array(p["ref_is_subs"])
    subs[v] = 1
    q["ref_is_subs"] = subs
    n = req["videos"][v]["n"]
    return q, -1, lambda err: err == ("%s: video %d has a subtitle reference and a non-empty PCM range (%d samples); "
                                      "its audio is never read" % (who, v, n))


@pytest.mark.parametrize("seed", SEEDS)
def test_random_plan(seed):
    req = rr.draw(seed, RATES)
    a = rr.arrays(req)
    p = rr.plan_request(req, a)
    rng = np.random.RandomState(seed + 7919)
    if rng.rand() < 0.1:
        q, status, ok = _bad(req, p, rng)
        got = plan(**q)
        assert got["status"] == status and ok(got["err"]), (rr.summary(req), got["status"], got["err"])
        return
    got = plan(**p)
    assert got["status"] == 0, (rr.summary(req), got["err"])
    check_plan(req, got)
