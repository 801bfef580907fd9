"""CPU suite for the reference format of the batched sync calls (csrc/sync_plan.h plan_ref_format): which
sub-batches have their VAD write the reference as packed bits.  That is the case exactly when the sub-batch's
correlation chain takes the run path, its detector is the lane-per-window energy kernel and it holds no subtitle
reference; the planner decides it with the aligner's own path choice (csrc/align_path.h).  Checked here, through
tests/host_emul/ref_format_emul, against a restatement of the launcher's rule over the planner's fixtures:
B2_ALIGN_PATH, a capture, float subtitle signals, the B2_REF_PACKED knob, auditok at labels 0 and 0.3, mixed
subtitle / audio calls and sub-batch cuts."""
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from test_plan_cpu import _subs, _tracks

EMUL = os.path.join(ROOT, "tests", "host_emul", "ref_format_emul")


def plan(**req):
    """req: the fields ref_format_emul.cu reads (arrays as sequences).  Returns "status", "err", the plan's cut /
    trk_off / ref_off / sub_off / ref_packed tables as int64 arrays, "two_level" and "ref_label"."""
    if not os.path.exists(EMUL):
        import sys
        sys.path.insert(0, ROOT)
        import __graft_entry__ as ge
        ge.build()
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.txt"), os.path.join(d, "out.txt")
        with open(src, "w") as f:
            for k, v in req.items():
                vals = [v] if np.isscalar(v) or isinstance(v, str) else list(np.asarray(v).ravel())
                f.write("%s %d %s\n" % (k, len(vals), " ".join(
                    x if isinstance(x, str) else repr(float(x)) if isinstance(x, (float, np.floating)) else str(int(x))
                    for x in vals)))
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

BLOCK = 32768            # overlap-save block (corr.cuh kP)
RUN_COST = 5.6e5         # kRunCostPerBlock
RUN_MAX_WINDOW = 32768
RUN_MAX_CUES = 16384
BIG_MIN_TILES = 4
BIG_LOG2 = (17, 23)


def _padded(n):
    k = 0
    while (1 << k) < n:
        k += 1
    return 1 << k


def _job(R, S, mo):
    """aligners.py:31-66 for one job: None (empty or all masked) or (N, o_lo, o_hi)."""
    if R == 0 or S == 0:
        return None
    N = _padded(R + S)
    a, b = N - 1 - mo - S, N - 1 + mo - S
    lo = min(a, N) if a >= 0 else max(a + N, 0)
    hi = min(b, N) if b >= 0 else max(b + N, 0)
    if lo >= hi:
        return None
    return N, N - S - hi, N - 1 - S - lo


def _chain_takes_runs(R, S, cues, trk, K, mo, env):
    """The launcher's path choice for one chain: R [V] reference lengths, S [T*K] subtitle lengths, cues [T] cue
    counts, trk [V+1] track offsets of the chain."""
    jobs, wins, big_ok = {}, [], True
    for v in range(len(R)):
        lo_v = hi_v = None
        for t in range(trk[v], trk[v + 1]):
            for k in range(K):
                jp = _job(R[v], S[t * K + k], mo)
                if jp is None:
                    continue
                N, o_lo, o_hi = jp
                big_ok &= (1 << BIG_LOG2[0]) <= N <= (1 << BIG_LOG2[1])
                jobs[t * K + k] = (o_lo, o_hi)
                lo_v = o_lo if lo_v is None else min(lo_v, o_lo)
                hi_v = o_hi if hi_v is None else max(hi_v, o_hi)
        wins.append(None if lo_v is None else hi_v - lo_v + 1)
    max_w = max([1] + [w for w in wins if w is not None])
    Wt = 32 * ((max_w + 30) // 32) + 1 if max_w <= BLOCK // 2 + 1 else BLOCK // 2 + 1
    L = BLOCK - Wt + 1
    path = env.get("align_path")
    use_big = big_ok and max_w > BIG_MIN_TILES * (BLOCK // 2 + 1)
    if path in ("tiled", "runs"):
        use_big = False
    if path == "big" and big_ok:
        use_big = True
    if env.get("capture") and path != "runs" or use_big or path == "tiled":
        return False
    fits = pays = True
    for v in range(len(R)):
        n_tiles = math.ceil(wins[v] / Wt) if wins[v] is not None else 0
        for t in range(trk[v], trk[v + 1]):
            for k in range(K):
                if t * K + k not in jobs:
                    continue
                o_lo, o_hi = jobs[t * K + k]
                w = o_hi - o_lo + 1
                fits &= w <= RUN_MAX_WINDOW and cues[t] <= RUN_MAX_CUES and max(abs(o_lo), abs(o_hi)) <= 1 << 30
                pays &= cues[t] * w <= RUN_COST * n_tiles * (math.ceil(S[t * K + k] / L) + 1)
    return fits and (pays or path == "runs")


def _expected(req, p):
    """The packed flag of every sub-batch of the plan p of request req."""
    K = len(req["ratios"])
    mo = req.get("max_offset_samples", 6000)
    auditok = req.get("detector", 0) == 1
    is_subs = np.asarray(req.get("ref_is_subs", [0] * (len(p["ref_off"]) - 1)))
    off = lambda a, i, j: a[i:j + 1] - a[i]   # noqa: E731
    cue_n = np.diff(np.asarray(req["cue_off"]))
    out = []
    for i in range(len(p["cut"]) - 1):
        v0, v1 = p["cut"][i], p["cut"][i + 1]
        t0, t1 = p["trk_off"][v0], p["trk_off"][v1]
        ok = (not auditok and req.get("fused", 1) and req.get("ref_packed") != "0" and req.get("lane", 0)
              and not is_subs[v0:v1].any() and p["two_level"] and math.isfinite(p["ref_label"]))
        if ok:
            R = np.diff(p["ref_off"][v0:v1 + 1])
            S = np.diff(p["sub_off"][t0 * K:t1 * K + 1])
            ok = _chain_takes_runs(R, S, cue_n[t0:t1], off(p["trk_off"], v0, v1), K, mo, req)
        out.append(int(bool(ok)))
    return out


def _check(**req):
    p = plan(**req)
    assert p["status"] == 0, p["err"]
    got = p["ref_packed"].tolist()
    assert got == _expected(req, p), (req, got)
    return got


def test_default_call_is_packed():
    assert _check(**_tracks(lane=1)) == [1]
    assert _check(**_tracks(lane=1, label=0.3)) == [1]
    assert _check(**_tracks(lane=1, label=-0.5, gss=1, who="sync_tracks_gss")) == [1]


@pytest.mark.parametrize("over", [dict(lane=0), dict(align_path="tiled"), dict(capture=1), dict(fused=0),
                                  dict(ref_packed="0"), dict(label=float("nan"))])
def test_floats_where_the_run_path_or_the_lane_kernel_is_not_taken(over):
    assert _check(**dict(_tracks(lane=1), **over)) == [0]


@pytest.mark.parametrize("path", ["runs", "big", "tiled", None])
@pytest.mark.parametrize("capture", [0, 1])
def test_align_path_and_capture(path, capture):
    req = _tracks(lane=1, capture=capture)
    if path:
        req["align_path"] = path
    got = _check(**req)
    assert got == [int(path != "tiled" and (not capture or path == "runs"))]


@pytest.mark.parametrize("label", [0.0, 0.3])
def test_auditok_keeps_floats(label):
    req = _tracks(lane=1, who="sync_tracks_auditok", detector=1, chunk_samples=320 * 5000, auditok_label=label)
    assert _check(**req) == [0]


@pytest.mark.parametrize("label", [0.0, 0.3])
def test_mixed_subtitle_and_audio_references(label):
    """Only a sub-batch of audio references is packed, and only when the call's reference has two levels."""
    assert _check(**_subs(lane=1, label=label)) == [0]
    got = _check(**_subs(lane=1, label=label, subbatches="4"))
    assert got == ([0, 1, 0] if label == 0.0 else [0, 0, 0])


@pytest.mark.parametrize("mos", [0, 300, 6000, 40000, 1 << 40])
@pytest.mark.parametrize("n_sub", ["1", "3"])
def test_windows_and_sub_batches(mos, n_sub):
    rng = np.random.RandomState(mos % 1000 + len(n_sub))
    per = rng.randint(0, 4, 12)
    per[[0, 5]] = 0
    _check(**_tracks(12, per, 16000 * 30, lane=1, max_offset_samples=mos, subbatches=n_sub))
    _check(**_tracks(12, per, 16000 * 30, lane=1, max_offset_samples=mos, subbatches=n_sub, align_path="runs"))
