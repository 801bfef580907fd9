"""Seeded random requests of every batched sync entry point against the composition of the existing oracles (run on
an H100).  tests/random_requests.py draws each request; a failure prints its summary line, and the seed alone
replays it.

Per seed:
  * the reference of every video (b2_capture_reference) against chunk_oracle.chunk_loop over the energy / ZCR or
    auditok detector, raster_oracle.rasterize, pgs_oracle.pgs_signal, sig_oracle.frames or
    segment_oracle.segment_reference, frame for frame (packed bits where the call packed);
  * the speech output (b2_speech_output) of a random subset of the videos: those references widened to float64;
  * every (track, ratio) score and offset against the exact correlation of those references with
    raster_oracle.rasterize's signal at the kernels' level: the largest score of the window, ties to the largest
    offset, bit for bit.  The levels (1, float32(1 / r), labels 0, 1 and -0.5) make every score a float64-exact sum.
    Only a job whose captured candidate count exceeds the re-score budget (B2_ALIGN_CAND_OVERFLOW) may return
    another offset: the exact score of that offset, at most the maximum.  An empty reference (B2_ALIGN_EMPTY) scores
    0.0 at offset 0; an all-masked window -inf at N - 1 - S;
  * b2_sync_tracks_gss: the search's 17 evaluated ratios against gss_oracle.golden_section_trace over the exact
    maxima, its ratio the last of them and its candidate the exact argmax there;
  * best_* against MaxScoreAligner.transform (aligner_oracle.max_score_select) over the per-ratio results, the
    search's candidate last, a video without speech in its segments B2_BEST_K_NO_SPEECH;
  * the winner-only call (nominations captured) returns the same best_*, and every pruned ratio (B2_ALIGN_APPROX)
    was one nomination_check._check_approx allows to be pruned;
  * the call with no capture returns identical outputs (with a capture the aligner keeps the FFT paths, without it
    the run path may take the job);
  * the synced cue times, offsets, scales and statuses of the call's best_* (b2_apply_sync, with and without
    try_sync's gate) against sync_output_oracle.apply_sync;
  * b2_sync_batch: two B2_DEVICE_RESIDENT calls back to back return what the ordered calls did."""
import contextlib

import numpy as np
import pytest

import nomination_check as nc
import random_requests as rr
from oracle import aligner_oracle as ao
from oracle import chunk_oracle as co
from oracle import gss_oracle as go
from oracle import pgs_oracle as po
from oracle import raster_oracle as ro
from oracle import segment_oracle as so
from oracle import sig_oracle as sgo
from oracle import sync_output_oracle as sync_out
from oracle import vad_oracle as vo
from test_gpu_reference_exact import _check as check_capture
from test_gpu_reference_exact import _poison
from test_gpu_speech_out import _output as speech_out

pytestmark = pytest.mark.gpu

SEEDS = list(range(96))
THR = 100000
Q = 2.0 ** 24          # every score is a multiple of 2^-24: products of +-1, -2 and 2 float32(1 / r) - 1
SEEN = {"entry": set(), "knobs": set(), "memspace": set(), "zero_track_cut": 0, "sub_window": 0, "zero_cue": 0,
        "one_offset_window": 0, "one_offset_window_split": 0, "all_masked": 0, "K1": 0, "approx": 0, "empty": 0,
        "overflow": 0, "seeds": set()}


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


# ------------------------------------------------------------------------------------------- inputs and oracles

def _pcm(n, fr, seed):
    """n samples of vad_oracle.synth_pcm over window classes in runs (silence, voiced, loud hiss)."""
    if n == 0:
        return np.zeros(0, np.int16)
    fpw = fr // rr.SR
    rng = np.random.RandomState(seed)
    cls, i, W = np.empty(-(-n // fpw), np.uint8), 0, -(-n // fpw)
    while i < W:
        L = rng.randint(1, 80)
        cls[i:i + L] = rng.choice(3, p=[0.45, 0.45, 0.1])
        i += L
    return vo.synth_pcm(cls, fpw, seed)[:n]


def _detect(req, pcm):
    det = dict(non_speech_label=req["label"])
    if req["detector"] == "auditok":
        return co.chunk_loop("auditok", pcm, req["fr"], rr.SR, chunk=req["chunk"], **det)
    return co.chunk_loop("energy_zcr", pcm, req["fr"], rr.SR, energy_threshold=THR, **det)


def _reference(req, d, pcm):
    """The float32 reference of video d."""
    k = d["kind"]
    if k == "audio":
        w = _detect(req, pcm)
    elif k == "subs":
        w = ro.rasterize(d["starts"], d["ends"], np.asarray(d["keep"], bool), rr.SR, 0.0, 1.0)[0]
    elif k == "pgs":
        w = po.pgs_signal(list(zip(d["starts"], d["ends"])), rr.SR)
    elif k == "sig":
        return sgo.frames(d["x"], req["label"])
    else:
        det = dict(non_speech_label=req["label"], frame_rate=req["fr"])
        if req["detector"] == "auditok":
            det.update(detector="auditok", chunk_samples=req["chunk"])
        else:
            det.update(energy_threshold=THR)
        w = so.segment_reference(pcm, d["total"], d["starts"], d["lo"], d["hi"], rr.SR, **det)
    return np.asarray(w, np.float64).astype(np.float32)


def _sub(t, r, keep):
    """The subtitle signal of track t at ratio r as the kernels hold it: level float32(min(1 / r, 1))."""
    level = float(np.float32(min(1.0 / r, 1.0)))
    return (ro.rasterize(t["starts"], t["ends"], keep, rr.SR, 0.0, r)[0] != 0) * level


def _exact_result(exact, ref, sub, mos):
    """(score, offset, near) of the exact argmax of the window, ties to the largest offset; near: the offsets within
    3 tau (nomination_check.Exact.tau) of the maximum, the most that can be candidates (an fp32 score within tau of
    the exact one, at or above the fp32 maximum less tau)."""
    if len(ref) == 0:
        return 0.0, 0, 0
    o_lo, o_hi = ao.offset_range(len(ref), len(sub), mos)
    if o_lo > o_hi:
        return -np.inf, ao.padded_length(len(ref), len(sub)) - 1 - len(sub), 0
    ex = np.round(exact.window(ref, sub, o_lo, o_hi - o_lo + 1) * Q) / Q
    m = int(np.flatnonzero(ex == ex.max())[-1])
    best = float(ex[m])
    assert best == ao.exact_score(ref, sub, o_lo + m), (best, o_lo + m)   # the rounded FFT is the exact sum
    near = int(np.count_nonzero(ex >= best - 3.0 * (1.0 + 1e-6) * exact.tau(ref, sub)))
    return best, o_lo + m, near


# ------------------------------------------------------------------------------------------- the call

def _call(handle, req, a, pcm, memspace, want_all, resident=False, keep=None):
    """One call of the request's entry point; returns host numpy (bs, bo, bk, a_s, a_o[, gss_ratio, gss_evals]),
    or with `resident` the device tensors, unsynchronised.  pcm: host int16 samples, or (device calls) the int
    address of device samples that a["pcm_off"] indexes."""
    import torch
    from ffsubsync_b200 import _native as N
    e, T, K = req["entry"], len(req["tracks"]), len(req["ratios"])
    gss = e == "gss"
    cols = K + 1 if gss else K
    ms = N.B2_HOST if memspace == "host" else (N.B2_DEVICE_RESIDENT if resident else N.B2_DEVICE)
    x = a.get("x")
    outs, dev = {}, {}
    if ms != N.B2_HOST:
        dev = dict(pcm=None if isinstance(pcm, int) else torch.from_numpy(pcm).cuda() if len(pcm) else None,
                   best_score=torch.full((T,), 7.0, dtype=torch.float64, device="cuda"),
                   best_offset=torch.full((T,), 7, dtype=torch.int32, device="cuda"),
                   best_k=torch.full((T,), 7, dtype=torch.int32, device="cuda"))
        if want_all:
            dev.update(all_score=torch.full((T * cols,), 7.0, dtype=torch.float64, device="cuda"),
                       all_offset=torch.full((T * cols,), 7, dtype=torch.int32, device="cuda"))
        if gss:
            dev["gss_ratio"] = torch.full((T,), 7.0, dtype=torch.float64, device="cuda")
            if want_all:
                dev["gss_evals"] = torch.full((T * N.GSS_EVALS,), 7.0, dtype=torch.float64, device="cuda")
        if x is not None:
            dev["x"] = torch.from_numpy(x).cuda() if len(x) else None
        torch.cuda.synchronize()
        outs = {k: v.data_ptr() for k, v in dev.items() if k not in ("x", "pcm")}
        x = dev["x"].data_ptr() if dev.get("x") is not None else None
        if not isinstance(pcm, int):
            pcm = dev["pcm"].data_ptr() if dev["pcm"] is not None else None
        if keep is not None:   # the tensors outlive calls that nothing synchronises
            keep.append(dev)
    common = dict(memspace=ms, want_all=want_all, **outs)
    if gss:
        common.update(gss_ratio=outs.get("gss_ratio"), want_evals=want_all)
    fr, label, mos = req["fr"], req["label"], req["mos"]
    cue = (a["cue_start"], a["cue_end"], a["cue_keep"], a["cue_off"], req["ratios"], 0.0, mos)
    det = dict(detector=int(req["detector"] == "auditok"), energy_threshold=THR, chunk_samples=req["chunk"])
    if e == "batch":
        r = handle.sync_batch(pcm, a["pcm_off"], fr, rr.SR, label, THR, -1, -1, *cue, **common)
    elif e == "tracks":
        r = handle.sync_tracks(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, THR, -1, -1, *cue, **common)
    elif e == "gss":
        r = handle.sync_tracks_gss(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, THR, -1, -1, *cue, **common)
    elif e == "auditok":
        r = handle.sync_tracks_auditok(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, *cue, req["chunk"],
                                       **common)
    elif e == "subs":
        r = handle.sync_tracks_subs(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, a["ref_is_subs"],
                                    a["ref_cue_start"], a["ref_cue_end"], a["ref_cue_keep"], a["ref_cue_off"], *cue,
                                    **det, **common)
    else:
        subs = dict(ref_is_subs=a["ref_is_subs"], ref_cue_start_s=a["ref_cue_start"], ref_cue_end_s=a["ref_cue_end"],
                    ref_cue_keep=a["ref_cue_keep"], ref_cue_off=a["ref_cue_off"])
        pgs = (a["ref_is_pgs"], a["pgs_start"], a["pgs_end"], a["pgs_off"])
        if e == "pgs":
            r = handle.sync_tracks_pgs(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, *pgs, *cue, **subs,
                                       **det, **common)
        else:
            pgs = dict(zip(("ref_is_pgs", "pgs_start_s", "pgs_end_s", "pgs_off"), pgs))
            if e == "sig":
                r = handle.sync_tracks_sig(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, a["ref_is_sig"], x,
                                           a["sig_off"], *cue, **subs, **pgs, **det, **common)
            else:
                r = handle.sync_tracks_seg(pcm, a["pcm_off"], a["track_video"], fr, rr.SR, label, a["seg_video"],
                                           a["seg_total"], a["seg_off"], a["seg_start"], a["seg_lo"], a["seg_hi"],
                                           *cue, ref_is_sig=a["ref_is_sig"], x=x, sig_off=a["sig_off"], **subs, **pgs,
                                           **det, **common)
    if ms == N.B2_HOST:
        return [None if v is None else np.array(v, copy=True) for v in (r[:5] + (r[5:7] if gss else ()))]
    if resident:
        return dev
    handle.synchronize()
    names = ["best_score", "best_offset", "best_k", "all_score", "all_offset"] + (["gss_ratio", "gss_evals"] if gss else [])
    return [dev[k].cpu().numpy() if k in dev else None for k in names]


def _same(x, y, where):
    for i, (p, q) in enumerate(zip(x, y)):
        assert (p is None) == (q is None), (where, i)
        if p is not None:
            assert p.dtype == q.dtype and np.array_equal(p, q, equal_nan=True), (where, i, p, q)


# ------------------------------------------------------------------------------------------- the checks

def _coverage(req, a, refs):
    from sync_plan import plan
    e = req["entry"]
    SEEN["seeds"].add(req["seed"])
    SEEN["entry"].add(e)
    SEEN["knobs"].add(tuple(sorted(req["knobs"].items())))
    SEEN["memspace"].add(req["memspace"])
    per = np.bincount(a["track_video"], minlength=len(refs)) if e != "batch" else np.ones(len(refs), int)
    p = plan(**rr.plan_request(req, a))
    # a video without tracks in front of a cut or right behind it
    SEEN["zero_track_cut"] += any(per[v] == 0 or per[v - 1] == 0 for v in p["cut"][1:-1])
    SEEN["sub_window"] += any(d["kind"] == "audio" and 0 < d["n"] < rr.window(req) for d in req["videos"])
    SEEN["zero_cue"] += any(len(t["starts"]) == 0 for t in req["tracks"])
    SEEN["K1"] += len(req["ratios"]) == 1


def _count_window(req, ref, sub):
    """Coverage of the job's window: empty reference, all masked, one offset (on the split tiled path)."""
    if len(ref) == 0:
        SEEN["empty"] += 1
        return
    o_lo, o_hi = ao.offset_range(len(ref), len(sub), req["mos"])
    SEEN["all_masked"] += o_lo > o_hi
    if o_hi == o_lo:
        SEEN["one_offset_window"] += 1
        SEEN["one_offset_window_split"] += "B2_ALIGN_SPLIT" in req["knobs"] and req["knobs"].get("B2_ALIGN_PATH") == "tiled"


def _check_job(exact, ref, sub, mos, got_s, got_o, overflow, w):
    """One (score, offset) against the exact argmax of its window.  overflow: the job had more candidates than the
    re-score budget (B2_ALIGN_CAND_OVERFLOW): then the score is the exact score of its offset, at most the maximum."""
    ws, wo, _ = _exact_result(exact, ref, sub, mos)
    w = "%s: got (%r, %d), exact (%r, %d)" % (w, float(got_s), int(got_o), ws, wo)
    if (got_s, got_o) != (ws, wo):
        assert overflow, w
        SEEN["overflow"] += 1
        lo, hi = ao.offset_range(len(ref), len(sub), mos)
        assert lo <= got_o <= hi and got_s == ao.exact_score(ref, sub, int(got_o)) and got_s <= ws, w


def _gss_trace(exact, ref, tr, keep, mos):
    """golden_section_trace over [0.9, 1.1] of -(exact maximum of the window) at each ratio: the ratios it evaluates
    and the (score, offset, near) of its last evaluation, the search's candidate."""
    last = []

    def f(x, _):
        last[:] = [_exact_result(exact, ref, _sub(tr, x, keep), mos)]
        return -last[0][0]

    _, calls = go.golden_section_trace(f, 0.9, 1.1)
    return np.array([x for x, _ in calls]), last[0]


def _check_outputs(req, a, out, ref64, subs, exact, overflow, traces, where, count=False):
    """Every output of one call: per (track, ratio) against the exact argmax, the search's evaluations and candidate
    against its trace, best_* against MaxScoreAligner.transform over the per-ratio results (the search's candidate
    last).  overflow[t, k]: the job may have overflowed its re-score budget."""
    from ffsubsync_b200 import _native as N
    vids, trk, grid, mos = req["videos"], req["tracks"], req["ratios"], req["mos"]
    T, K = len(trk), len(grid)
    gss = req["entry"] == "gss"
    cols = K + 1 if gss else K
    bs, bo, bk = out[:3]
    a_s, a_o = out[3].reshape(T, cols), out[4].reshape(T, cols)
    for t, tr in enumerate(trk):
        v = tr["video"]
        ref = ref64[v]
        if vids[v]["kind"] == "seg" and not so.has_speech(ref):   # the reference raises: the call flags it
            assert bk[t] == N.B2_BEST_K_NO_SPEECH, (where, t)
            continue
        for k in range(K):
            if count:
                _count_window(req, ref, subs[t][k])
            _check_job(exact, ref, subs[t][k], mos, a_s[t, k], a_o[t, k], overflow[t, k],
                       "%s: track %d video %d (%s, %d frames) ratio %d" % (where, t, v, vids[v]["kind"], len(ref), k))
        if gss:
            r_g, evals = float(out[5][t]), out[6].reshape(T, N.GSS_EVALS)[t]
            if len(ref) == 0:
                assert np.isnan(r_g) and np.isnan(evals).all(), (where, t)
            else:
                xs, (ws, wo, near) = traces[t]
                assert np.array_equal(evals, xs) and r_g == xs[-1], (where, "search", t, evals, xs)
                _check_job(exact, ref, _sub(tr, r_g, tr["keep"]), mos, a_s[t, K], a_o[t, K], near > nc.K_CAND,
                           "%s: track %d search at %r" % (where, t, r_g))
        live = [k for k in range(cols) if len(ref) > 0]
        res = [(float(a_s[t, k]), int(a_o[t, k])) for k in live]
        try:
            i = ao.max_score_select(res, mos)
            want = (res[i][0], res[i][1], live[i])
        except ao.OracleAlignmentFailure:
            want = (0.0, 0, -1)
        assert (bs[t], bo[t], bk[t]) == want, (where, "best", t, (bs[t], bo[t], bk[t]), want)


def _window_stride(req, ref64, subs):
    w = [ao.offset_range(len(ref64[tr["video"]]), len(s), req["mos"]) for t, tr in enumerate(req["tracks"])
         for s in subs[t] if len(ref64[tr["video"]]) > 0]
    return max([1] + [hi - lo + 1 for lo, hi in w])


# ------------------------------------------------------------------------------------------- the test

@pytest.mark.parametrize("seed", SEEDS)
def test_random_request(handle, seed, monkeypatch):
    from ffsubsync_b200 import _native as N
    req = rr.draw(seed)
    where = rr.summary(req)
    for k, v in req["knobs"].items():
        monkeypatch.setenv(k, v)
    a = rr.arrays(req)
    vids, trk, grid, mos = req["videos"], req["tracks"], req["ratios"], req["mos"]
    V, T, K = len(vids), len(trk), len(grid)
    gss = req["entry"] == "gss"
    rng = np.random.RandomState(seed + 104729)
    pcms = [_pcm(d["n"], req["fr"], seed * 97 + v) if d["kind"] in ("audio", "seg") else np.zeros(0, np.int16)
            for v, d in enumerate(vids)]
    pcm = np.concatenate(pcms)
    refs = [_reference(req, d, pcms[v]) for v, d in enumerate(vids)]
    ref64 = [r.astype(np.float64) for r in refs]
    _coverage(req, a, refs)
    keep = None if a["cue_keep"] is None else a["cue_keep"].astype(bool)
    for t, tr in enumerate(trk):
        tr["keep"] = None if keep is None else keep[a["cue_off"][t]:a["cue_off"][t + 1]]
    subs = [[_sub(tr, r, tr["keep"]) for r in grid] for tr in trk]
    exact = nc.Exact()
    traces = {t: _gss_trace(exact, ref64[tr["video"]], tr, tr["keep"], mos) for t, tr in enumerate(trk)
              if gss and len(ref64[tr["video"]]) > 0}

    # 1. per-ratio outputs with the reference, the nominations (not the search's rounds) and the speech output of a
    #    random subset of the videos captured
    cap_n = int(sum(len(r) for r in refs)) + 4096
    speech = sorted(int(v) for v in rng.choice(V, rng.randint(0, V + 1), replace=False))
    ms_out = N.B2_HOST if req["memspace"] == "host" else N.B2_DEVICE
    _poison(handle, cap_n)
    with contextlib.ExitStack() as stack:
        cap = stack.enter_context(handle.capture_reference(cap_n, V + 3))
        nom = None if gss else stack.enter_context(handle.capture_nominations(T * K, _window_stride(req, ref64, subs)))
        sp = stack.enter_context(speech_out(handle, speech, int(sum(len(refs[v]) for v in speech)), ms_out)) \
            if speech else None
        got = _call(handle, req, a, pcm, req["memspace"], want_all=True)
    check_capture(cap, refs, where=where)
    if sp is not None:
        lens = [len(refs[v]) for v in speech]
        assert np.array_equal(sp["off"], np.concatenate([[0], np.cumsum(lens)])), (where, "speech_off", sp["off"])
        for i, v in enumerate(speech):
            assert np.array_equal(sp["buf"][sp["off"][i]:sp["off"][i + 1]], ref64[v]), (where, "speech", v)
        assert np.isnan(sp["buf"][sp["off"][-1]:]).all(), (where, "speech written past speech_off[n]")
    if gss:   # no capture: the rounds run on the run path, whose candidates lie within 3 tau of the exact maximum
        overflow = np.array([[_exact_result(exact, ref64[tr["video"]], s, mos)[2] > nc.K_CAND for s in subs[t]]
                             for t, tr in enumerate(trk)], bool).reshape(T, K)
    else:
        overflow = (nom["cand"] > nc.K_CAND).reshape(T, K)
    _check_outputs(req, a, got, ref64, subs, exact, overflow, traces, where, count=True)

    # 2. winner-only with the nominations captured: the same best_*, and only ratios that cannot win pruned
    live_t = [t for t, tr in enumerate(trk) if len(ref64[tr["video"]]) > 0]
    if not gss and live_t and req["knobs"].get("B2_ALIGN_PATH") != "runs":
        jobs = [t * K + k for t in live_t for k in range(K)]
        with handle.capture_nominations(T * K, _window_stride(req, ref64, subs)) as nom:
            win = _call(handle, req, a, pcm, req["memspace"], want_all=False)
        sub_cap = {k: v[jobs] for k, v in nom.items()}
        nc.check_jobs(sub_cap, [(ref64[trk[j // K]["video"]], subs[j // K][j % K]) for j in jobs], mos, exact, where,
                      winner_only=True, K=K)
        SEEN["approx"] += int(np.count_nonzero(sub_cap["cand"] == -1))
    else:
        win = _call(handle, req, a, pcm, req["memspace"], want_all=False)
    _same(win[:3], got[:3], (where, "winner-only"))

    # 3. the same request without any capture (the aligner may now take the run path): the same outputs, or where a
    #    job overflowed its re-score budget, outputs that pass the same checks
    plain = _call(handle, req, a, pcm, req["memspace"], want_all=True)
    if overflow.any():
        _check_outputs(req, a, plain, ref64, subs, exact, overflow, traces, (where, "no capture"))
    else:
        _same(plain, got, (where, "no capture"))

    # 4. the synced cue times and try_sync's gate of the call's best_* (b2_apply_sync) against sync_output_oracle
    rule = dict(gate=bool(rng.rand() < 0.5), min_score=float(rng.choice([0.0, 50.0])),
                apply_offset_seconds=float(rng.choice([0.0, -1.25])), suppress=[None, 0.0][rng.randint(2)])
    g_ratio = got[5] if gss else None
    cue = (a["cue_start"], a["cue_end"], a["cue_off"], grid, rr.SR)
    synced = handle.apply_sync(got[0], got[1], got[2], g_ratio, *cue, **rule)
    want = sync_out.apply_sync(got[0], got[1], got[2], g_ratio, *cue, **rule)
    _same(list(synced), list(want), (where, "apply_sync", rule))

    # 5. b2_sync_batch: a resident pair back to back equals the ordered calls
    if req["entry"] == "batch":
        hold = []
        pair = [_call(handle, req, a, pcm, "device", want_all=True, resident=True, keep=hold) for _ in range(2)]
        handle.synchronize()
        for d in pair:
            _same([d[k].cpu().numpy() for k in ("best_score", "best_offset", "best_k", "all_score", "all_offset")],
                  got, (where, "resident pair"))


def test_generator_reached_every_edge():
    """Over the seeds above, the generator drew every entry point, knob set and memspace, and each edge case."""
    if SEEN["seeds"] != set(SEEDS):
        pytest.skip("only part of the seeds ran")
    assert SEEN["entry"] == set(rr.ENTRIES), SEEN["entry"]
    assert SEEN["knobs"] == {tuple(sorted(k.items())) for k in rr.KNOBS}, SEEN["knobs"]
    assert SEEN["memspace"] == {"host", "device"}
    for k in ("zero_track_cut", "sub_window", "zero_cue", "one_offset_window", "one_offset_window_split", "all_masked",
              "K1", "approx", "empty"):
        assert SEEN[k] > 0, (k, SEEN)
