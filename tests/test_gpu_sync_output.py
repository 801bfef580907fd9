"""GPU tests of try_sync's epilogue over the batched calls (b2_apply_sync; run on an H100).

Yardstick: oracle/sync_output_oracle.py (checked against the reference's own try_sync in the CPU suite) applied to
each call's own results.  After every batched path - the grid, the search (device-driven and composed), auditok,
the subs_then_ detectors, PGS and serialized-signal references, on host and device memory - every synced cue time
and every status bit must equal the oracle's.  Also: resident sync calls stay chained across apply_sync, the
argument checks, and the launch count of a sync call."""
import re

import numpy as np
import pytest

from oracle import sync_output_oracle as so
from test_gpu_sig_ref import _sig_corpus

pytestmark = pytest.mark.gpu

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
KINDS = ["audio", "text", "pgs", "sig"]
# (vad, search, non_speech_label, reference kinds handed over)
ARMS = [("energy_zcr", False, 0.0, ()), ("energy_zcr", True, 0.0, ()), ("auditok", False, 0.0, ()),
        ("auditok", True, 0.3, ()),   # the search at a non-zero label: composed on the host
        ("subs_then_energy_zcr", False, 0.0, ("text",)), ("subs_then_auditok", True, 0.0, ("text",)),
        ("energy_zcr", False, 0.0, ("pgs",)), ("subs_then_energy_zcr", True, 0.0, ("text", "pgs", "sig"))]
RULES = [dict(),
         dict(skip_sync_on_low_quality=True, min_score=20.0, quality_max_offset_seconds=3.0,
              max_framerate_deviation=0.03, apply_offset_seconds=0.1234565, suppress_output_if_offset_less_than=-1.5),
         dict(apply_offset_seconds=-2.5, suppress_output_if_offset_less_than=0.0)]


@pytest.fixture(scope="module")
def handle():
    from ffsubsync_b200 import _native
    return _native.get_handle()


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.RandomState(5)
    videos = [(60.0 + 3 * (v % 4), KINDS[v % 4] if v % 5 else "audio",
               [(GRID[int(rng.randint(0, 5))], int(rng.randint(-700, 700))) for _ in range(1 + v % 2)])
              for v in range(12)]
    return _sig_corpus(videos, seed0=23)


def _streams(c, kinds, on_device):
    s = {}
    if "text" in kinds:
        tv = np.flatnonzero(c["is_subs"])
        s.update(ref_cue_start=c["ref_start"], ref_cue_end=c["ref_end"],
                 ref_cue_off=np.concatenate([[0], np.cumsum(np.diff(c["ref_off"])[tv])]), ref_stream_video=tv,
                 ref_cue_keep=c["ref_keep"])
    if "pgs" in kinds:
        pv = np.flatnonzero(c["is_pgs"])
        s.update(pgs_start=c["pgs_start"], pgs_end=c["pgs_end"],
                 pgs_off=np.concatenate([[0], np.cumsum(np.diff(c["pgs_off"])[pv])]), pgs_video=pv)
    if "sig" in kinds:
        import torch
        sv = np.flatnonzero(c["is_sig"])
        x = np.concatenate([c["x"][c["sig_off"][v]: c["sig_off"][v + 1]] for v in sv])
        s.update(sig=torch.from_numpy(x).cuda() if on_device else x,
                 sig_off=np.concatenate([[0], np.cumsum(np.diff(c["sig_off"])[sv])]), sig_video=sv)
    return s


def _oracle_rule(rule):
    return dict(apply_offset_seconds=rule.get("apply_offset_seconds", 0),
                gate=rule.get("skip_sync_on_low_quality", False), min_score=rule.get("min_score", 0.0),
                quality_max_offset_seconds=rule.get("quality_max_offset_seconds", 30.0),
                max_framerate_deviation=rule.get("max_framerate_deviation", 0.1),
                suppress=rule.get("suppress_output_if_offset_less_than"))


def _check(got, bs, bo, bk, ratio, c, s, rule, where):
    want = so.apply_sync(bs, bo, bk, ratio, c["cue_start"], c["cue_end"], c["cue_off"], list(s.ratios), 100,
                         **_oracle_rule(rule))
    for key, w in zip(("synced_start_us", "synced_end_us", "offset_seconds", "scale", "status"), want):
        g = np.asarray(got[key])
        assert g.shape == w.shape and np.array_equal(g, w, equal_nan=key in ("offset_seconds", "scale")), (where, key)
    return want[4]


@pytest.mark.parametrize("arm", range(len(ARMS)))
def test_equals_the_oracle_after_every_path(handle, corpus, arm):
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    vad, gss, label, kinds = ARMS[arm]
    c = corpus
    s = BatchSynchronizer(GRID + ([None] if gss else []), vad=vad, non_speech_label=label)
    seen = 0
    for on_device in (False, True):
        streams = _streams(c, kinds, on_device)
        if on_device:
            out = s.sync_device_tracks(torch.from_numpy(c["pcm"]).cuda(), c["pcm_off"], c["track_video"],
                                       c["cue_start"], c["cue_end"], c["cue_off"], **streams)
            results = [s.apply_sync(out, c["cue_start"], c["cue_end"], c["cue_off"], **r) for r in RULES]
            torch.cuda.synchronize()
            res = [out[k].cpu().numpy() for k in ("best_score", "best_offset", "best_k")]
            res.append(out["gss_ratio"].cpu().numpy() if gss else None)
            results = [{k: v.cpu().numpy() for k, v in r.items()} for r in results]
        else:
            host = s.sync_host_tracks(c["pcm"], c["pcm_off"], c["track_video"], c["cue_start"], c["cue_end"],
                                      c["cue_off"], **streams)
            results = [s.apply_sync_host(host, c["cue_start"], c["cue_end"], c["cue_off"], **r) for r in RULES]
            res = list(host[:3]) + [host[-1] if gss else None]
        for r, got in zip(RULES, results):
            st = _check(got, *res, c, s, r, (ARMS[arm], on_device, r))
            seen |= int(np.bitwise_or.reduce(st))
    # the rules reach the written, applied, successful and gated outcomes on every path
    assert seen & so.WRITTEN and seen & so.APPLIED and seen & so.SUCCESSFUL, seen
    assert seen & (so.LOW_SCORE | so.LOW_OFFSET | so.LOW_FRAMERATE | so.SUPPRESSED), seen


def test_failed_and_offset_cue_tables(handle):
    """Failed tracks (best_k -1, -2, out of range, a search point outside [0.9, 1.1]), a cue_off that does not
    start at 0, empty tracks and 4-hour times, fed to both memspaces directly."""
    import torch
    from ffsubsync_b200 import _native
    rng = np.random.RandomState(3)
    T, K = 9, 3
    ratios = np.array([1.0, 25 / 24.0, 24 / 25.0])
    lens = np.array([3, 0, 5, 1, 4, 0, 2, 6, 3])
    cue_off = np.concatenate([[7], 7 + np.cumsum(lens)]).astype(np.int64)
    n = int(cue_off[-1])
    cs = np.round(rng.uniform(-5, 14400, n) * 1e6) / 1e6
    ce = cs + np.round(rng.uniform(0, 5, n), 6)
    bs = rng.uniform(-10, 100, T)
    bo = rng.randint(-6000, 6000, T).astype(np.int32)
    bk = np.array([0, 1, 2, 3, -1, -2, 3, 7, 3], np.int32)
    g = np.array([1.0, 1.0, 1.0, 1.05, 1.0, 1.0, 1.2, 1.0, np.nan])
    rule = dict(apply_offset_seconds=0.0000005, gate=True, min_score=0.0, quality_max_offset_seconds=40.0,
                max_framerate_deviation=0.045, suppress=-10.0)
    want = so.apply_sync(bs, bo, bk, g, cs, ce, cue_off, ratios, 100, **rule)
    got = handle.apply_sync(bs, bo, bk, g, cs, ce, cue_off, ratios, 100, **rule)
    dev = [torch.from_numpy(a).cuda() for a in (bs, bo, bk, g)]
    outs = [torch.empty(n, dtype=torch.int64, device="cuda"), torch.empty(n, dtype=torch.int64, device="cuda"),
            torch.empty(T, dtype=torch.float64, device="cuda"), torch.empty(T, dtype=torch.float64, device="cuda"),
            torch.empty(T, dtype=torch.int32, device="cuda")]
    handle.apply_sync(*[a.data_ptr() for a in dev], cs, ce, cue_off, ratios, 100, **rule,
                      outs=[o.data_ptr() for o in outs], memspace=_native.B2_DEVICE)
    handle.synchronize()
    for i, w in enumerate(want):
        assert np.array_equal(got[i][7:] if i < 2 else got[i], w[7:] if i < 2 else w, equal_nan=True), i
        d = outs[i].cpu().numpy()
        assert np.array_equal(d[7:] if i < 2 else d, w[7:] if i < 2 else w, equal_nan=True), i
    assert [bool(v & so.FAILED) for v in want[4]] == [False, False, False, False, True, True, True, True, True]


def test_resident_chain_survives_apply_sync(handle, corpus, monkeypatch, capfd):
    """Unsynchronised resident sync_device calls with apply_sync between them return what the same calls return
    unchained, and every call after the first is still chained (B2_PIPE_TRACE's `chained`)."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    audio = np.flatnonzero(np.diff(c["pcm_off"]) > 0)
    tv = c["track_video"]
    pick = np.flatnonzero(np.isin(tv, audio))
    cs = np.concatenate([c["cue_start"][c["cue_off"][t]: c["cue_off"][t + 1]] for t in pick])
    ce = np.concatenate([c["cue_end"][c["cue_off"][t]: c["cue_off"][t + 1]] for t in pick])
    co = np.concatenate([[0], np.cumsum(np.diff(c["cue_off"])[pick])]).astype(np.int64)
    s = BatchSynchronizer(GRID)
    s.use_torch_stream()
    pcm = torch.from_numpy(c["pcm"]).cuda()
    monkeypatch.setenv("B2_SUBBATCHES", "3")
    rule = RULES[1]

    def step(resident):
        out = s.sync_device_tracks(pcm, c["pcm_off"], tv[pick], cs, ce, co, inputs_resident=resident)
        return out, s.apply_sync(out, cs, ce, co, **rule)

    want = []
    for _ in range(3):
        o, a = step(False)
        torch.cuda.synchronize()
        want.append(({k: v.cpu().numpy() for k, v in o.items()}, {k: v.cpu().numpy() for k, v in a.items()}))
    capfd.readouterr()
    monkeypatch.setenv("B2_PIPE_TRACE", "1")
    got = [step(True) for _ in range(3)]
    torch.cuda.synchronize()
    err = capfd.readouterr().err
    chained = [int(m) for m in re.findall(r"chained=(\d)", err)]
    assert chained == [0, 1, 1], err
    for (o, a), (wo, wa) in zip(got, want):
        for k in wo:
            assert np.array_equal(o[k].cpu().numpy(), wo[k]), k
        for k in wa:
            assert np.array_equal(a[k].cpu().numpy(), wa[k], equal_nan=True), k


def test_launch_count_of_a_sync_call(handle, corpus):
    """A sync call issues the same launches whether or not apply_sync ran before it; apply_sync is one launch."""
    import torch
    from ffsubsync_b200.batch import BatchSynchronizer
    c = corpus
    audio = np.flatnonzero(np.diff(c["pcm_off"]) > 0)
    pick = np.flatnonzero(np.isin(c["track_video"], audio))
    s = BatchSynchronizer(GRID)
    h = s.handle
    pcm = torch.from_numpy(c["pcm"]).cuda()
    co = np.concatenate([[0], np.cumsum(np.diff(c["cue_off"])[pick])]).astype(np.int64)
    cs = np.concatenate([c["cue_start"][c["cue_off"][t]: c["cue_off"][t + 1]] for t in pick])
    ce = np.concatenate([c["cue_end"][c["cue_off"][t]: c["cue_off"][t + 1]] for t in pick])

    def sync():
        n0 = h.launch_count
        out = s.sync_device_tracks(pcm, c["pcm_off"], c["track_video"][pick], cs, ce, co)
        return out, h.launch_count - n0

    out, first = sync()
    n0 = h.launch_count
    s.apply_sync(out, cs, ce, co)
    assert h.launch_count - n0 == 1
    _, second = sync()
    torch.cuda.synchronize()
    assert first == second > 0


def test_bad_arguments(handle):
    import torch
    from ffsubsync_b200 import _native
    bs, bo, bk = np.array([1.0, 2.0]), np.array([3, -4], np.int32), np.array([0, 1], np.int32)
    cs, ce, co, ratios = np.array([1.0, 2.0, 3.0]), np.array([1.5, 2.5, 3.5]), np.array([0, 2, 3]), [1.0, 1.04]

    def err(**kw):
        a = dict(best_score=bs, best_offset=bo, best_k=bk, gss_ratio=None, cue_start_s=cs, cue_end_s=ce, cue_off=co,
                 ratios=ratios, sample_rate=100)
        a.update(kw)
        with pytest.raises(_native.NativeError) as e:
            handle.apply_sync(**a)
        assert e.value.status == -1
        return str(e.value)

    assert "monotone" in err(cue_off=np.array([0, 3, 2]))
    assert "not finite" in err(cue_start_s=np.array([1.0, np.nan, 3.0])) and "cue 1" in err(
        cue_start_s=np.array([1.0, np.nan, 3.0]))
    assert "not finite" in err(cue_end_s=np.array([1.0, 2.0, np.inf]))
    assert "B2_MAX_CUE_SECONDS" in err(cue_end_s=np.array([1.0, 2.0, 9.0e9]))
    assert "B2_MAX_CUE_SECONDS" in err(cue_end_s=np.array([1.0, 2.0, 8.0e9]), ratios=[1.0, 1.2])
    assert "apply_offset_seconds" in err(apply_offset_seconds=float("nan"))
    assert "ratio" in err(ratios=[1.0, float("inf")])
    assert "sample_rate" in err(sample_rate=0)
    # null and host outputs / inputs under B2_DEVICE
    d = [torch.from_numpy(a).cuda() for a in (bs, bo, bk)]
    outs = [torch.empty(3, dtype=torch.int64, device="cuda"), torch.empty(3, dtype=torch.int64, device="cuda"),
            torch.empty(2, dtype=torch.float64, device="cuda"), torch.empty(2, dtype=torch.float64, device="cuda"),
            torch.empty(2, dtype=torch.int32, device="cuda")]
    ptrs = [o.data_ptr() for o in outs]
    dev = dict(best_score=d[0].data_ptr(), best_offset=d[1].data_ptr(), best_k=d[2].data_ptr(),
               memspace=_native.B2_DEVICE)
    assert "null" in err(outs=[None] + ptrs[1:], **dev)
    assert "null" in err(outs=ptrs[:4] + [None], **dev)
    host_out = np.zeros(3, np.int64)
    assert "host pointer" in err(outs=[host_out.ctypes.data] + ptrs[1:], **dev)
    assert "host pointer" in err(outs=ptrs, **dict(dev, best_k=bk.ctypes.data))
    assert "memspace" in err(outs=ptrs, **dict(dev, memspace=_native.B2_DEVICE_RESIDENT))
    # nothing was written by the refused calls, and a good call still runs
    handle.apply_sync(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), None, cs, ce, co, ratios, 100, outs=ptrs,
                      memspace=_native.B2_DEVICE)
    handle.synchronize()
    want = so.apply_sync(bs, bo, bk, None, cs, ce, co, ratios, 100)
    assert np.array_equal(outs[0].cpu().numpy(), want[0]) and np.array_equal(outs[4].cpu().numpy(), want[4])
