"""CPU suite for the golden-section search inside the batched sync (b2_sync_tracks_gss).

The arithmetic the GSS rounds run on the device - the search step, the signal length S(ratio) and the per-job
window plan shared with the host planner (csrc/job_plan.cuh, csrc/raster_math.cuh) - runs here on the CPU
through tests/host_emul/gss_emul.cu and is compared with the reference's Python: golden_section_search.gss,
the signal length over timedelta and the slice arithmetic of FFTAligner (ffsubsync/aligners.py:31-48)."""
import ctypes
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT

EXE = os.path.join(ROOT, "tests", "host_emul", "gss_emul")
NONE = -(1 << 63)


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


def _run(mode, payload: bytes) -> bytes:
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(payload)
        subprocess.check_call([EXE, mode, fin, fout])
        with open(fout, "rb") as f:
            return f.read()


# ---------------------------------------------------------------- the search step

def _emulate_gss(scores: np.ndarray, lo=0.9, hi=1.1):
    """scores: [lanes, n + 1] (the score each round's point gets).  -> constants, points [lanes, n + 1],
    final intervals [lanes, 2]."""
    lanes, n1 = scores.shape
    head = np.array([lanes, n1 - 1], np.int64).tobytes() + np.array([lo, hi], np.float64).tobytes()
    raw = np.frombuffer(_run("step", head + np.ascontiguousarray(scores, np.float64).tobytes()), np.float64)
    consts = raw[:2], int(raw[2:3].view(np.int64)[0])
    body = raw[3:].reshape(lanes, n1 + 2)
    return consts, body[:, :n1], body[:, n1:]


def _python_gss(scores_row, lo=0.9, hi=1.1, tol=1e-4):
    """golden_section_search.gss with f = -score of the i-th call; returns (points, interval)."""
    from ffsubsync_b200.golden_section_search import gss
    pts = []

    def f(x, last):
        pts.append(x)
        return -scores_row[len(pts) - 1]

    interval = gss(f, lo, hi, tol)
    return pts, interval


def test_gss_constants(built):
    from ffsubsync_b200.golden_section_search import invphi, invphi2
    from ffsubsync_b200.aligners import MAX_FRAMERATE_RATIO, MIN_FRAMERATE_RATIO
    from oracle import gss_oracle as go
    (c, evals), _, _ = _emulate_gss(np.zeros((1, 17)))
    assert c[0] == invphi and c[1] == invphi2
    assert evals == go.num_iterations(MIN_FRAMERATE_RATIO, MAX_FRAMERATE_RATIO) + 1 == 17


def test_gss_step_reproduces_golden_quadratic(built, golden):
    want = golden["gss_quadratic"]
    # the quadratic's objective is (x - 1.0417)^2, i.e. score = -(x - 1.0417)^2: feed the points back
    # round by round (each score depends on the point the step produced)
    xs, scores = [], []
    for r in range(17):
        s = np.zeros((1, 17))
        s[0, :len(scores)] = scores
        _, pts, _ = _emulate_gss(s)
        x = pts[0, r]
        xs.append(x)
        scores.append(-((x - 1.0417) ** 2))
    _, pts, iv = _emulate_gss(np.array([scores]))
    assert [float(x) for x in pts[0]] == [c[0] for c in want["calls"]]
    assert list(iv[0]) == want["interval"]
    assert [c[1] for c in want["calls"]] == [False] * 16 + [True]   # only the 17th is the candidate


def _random_scores(rng, lanes, n1):
    """Score sequences with exact ties (few distinct values), -inf (all-masked windows) and plain noise."""
    s = rng.randint(-3, 4, size=(lanes, n1)).astype(np.float64)
    s[lanes // 3: 2 * lanes // 3] = rng.randn(lanes - lanes // 3 - (lanes - 2 * lanes // 3), n1) * 1e3
    s[rng.rand(lanes, n1) < 0.15] = -np.inf
    s[:4] = -np.inf                      # every window empty
    s[4:8] = 7.0                         # every round tied
    return s


def test_gss_step_matches_python_on_random_lanes(built):
    rng = np.random.RandomState(5)
    s = _random_scores(rng, 600, 17)
    _, pts, iv = _emulate_gss(s)
    for lane in range(len(s)):
        want_pts, want_iv = _python_gss(list(s[lane]))
        assert [float(x) for x in pts[lane]] == want_pts, lane
        assert tuple(float(v) for v in iv[lane]) == tuple(want_iv), lane


def test_gss_step_other_intervals_and_single_iteration(built):
    from oracle import gss_oracle as go
    rng = np.random.RandomState(9)
    # (lo, hi, tol) with n = 1 (two evaluations, both flagged last) up to n = 20
    for lo, hi, tol in [(0.9, 1.1, 0.15), (1.0, 1.3, 0.2), (0.5, 2.0, 1e-3), (1.1, 0.9, 1e-4), (0.0, 1.0, 1e-5)]:
        n = go.num_iterations(lo, hi, tol)
        assert n >= 1
        s = _random_scores(rng, 64, n + 1)
        _, pts, iv = _emulate_gss(s, lo, hi)
        for lane in range(len(s)):
            want_pts, want_iv = _python_gss(list(s[lane]), lo, hi, tol)
            assert [float(x) for x in pts[lane]] == want_pts, (lo, hi, tol, lane)
            assert tuple(float(v) for v in iv[lane]) == tuple(want_iv), (lo, hi, tol, lane)
    assert go.num_iterations(0.9, 1.1, 0.15) == 1


# ---------------------------------------------------------------- S(ratio)

def _emulate_len(max_end, ratio, sample_rate):
    rec = np.zeros(len(max_end), dtype=[("e", "<f8"), ("r", "<f8"), ("sr", "<i8")])
    rec["e"], rec["r"], rec["sr"] = max_end, ratio, sample_rate
    return np.frombuffer(_run("len", rec.tobytes()), np.int64)


def test_signal_length_equals_reference_formula(built):
    """S(x) as the GSS rounds compute it (b2_signal_length of the track's largest unscaled cue end) against the
    reference's own formula evaluated in Python over every cue: int(max(0, max over cues of
    timedelta(seconds=end * x).total_seconds()) * sample_rate) + 2 (speech_transformers.py:958-962)."""
    from datetime import timedelta
    rng = np.random.RandomState(11)
    T = 120
    counts = rng.randint(0, 30, T)
    counts[:3] = 0                                   # tracks without cues
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    ends = rng.rand(off[-1]) * 8000.0
    ratios = np.concatenate([rng.uniform(0.9, 1.1, 24), [0.9, 1.1, 1.0, 25 / 24, 24 / 25, 1.0001, 0.9999]])
    # microsecond rounding edges: ends that a ratio of the list maps onto half-microsecond ties
    for i in range(0, off[-1], 5):
        r = ratios[i % len(ratios)]
        ends[i] = (rng.randint(0, 7_200_000_000) + 0.5) / 1e6 / r
    ends[5::11] = -np.abs(ends[5::11])               # negative ends: no time beyond 0
    max_end = np.array([ends[off[t]:off[t + 1]].max() if counts[t] else 0.0 for t in range(T)])
    for sr in (100, 48):
        want = np.empty((T, len(ratios)), np.int64)
        for t in range(T):
            for k, r in enumerate(ratios):
                mt = 0.0
                for e in ends[off[t]:off[t + 1]]:
                    mt = max(mt, timedelta(seconds=float(e) * float(r)).total_seconds())
                want[t, k] = int(mt * sr) + 2
        got = _emulate_len(np.repeat(max_end, len(ratios)), np.tile(ratios, T), sr).reshape(T, -1)
        assert np.array_equal(got, want)
        # monotone in the ratio: the mask capacity planned at 1.1 covers every point of the search
        assert np.all(_emulate_len(max_end, np.full(T, 1.1), sr) >= want.max(axis=1))


# ---------------------------------------------------------------- the shared job plan

def _quirk_mask():
    m = 0
    for k in range(63):
        if math.ceil(math.log(float(1 << k)) / math.log(2.0)) > k:
            m |= 1 << k
    return m


def _old_planner(R, S, mo, mask):
    """The inline planner b2i_align_launch had before the plan moved to job_plan.cuh, transcribed."""
    if R == 0 or S == 0:
        return (1, 0, 0, 0, 0, -1, 0)
    k = 0
    while (1 << k) < R + S:
        k += 1
    if (1 << k) == R + S and (mask >> k) & 1:
        k += 1
    N = 1 << k
    lo, hi = 0, N
    if mo != NONE:
        m = max(-(1 << 40), min(1 << 40, mo))
        a, bb = N - 1 - m - S, N - 1 + m - S
        lo = min(a, N) if a >= 0 else max(a + N, 0)
        hi = min(bb, N) if bb >= 0 else max(bb + N, 0)
    if lo >= hi:
        return (2, N, 0, 0, 0, -1, N - 1 - S)
    return (0, N, lo, hi, N - S - hi, N - 1 - S - lo, 0)


def _python_window(R, S, mo):
    """FFTAligner.fit's window in the reference's own terms: padded length from math.log, the mask by numpy
    slicing of a length-N array, the offsets of the surviving indices (aligners.py:31-48)."""
    N = int(2 ** math.ceil(math.log(R + S, 2)))
    keep = np.ones(N, bool)
    if mo != NONE:
        keep[: N - 1 - mo - S] = False
        keep[N - 1 + mo - S:] = False
    idx = np.nonzero(keep)[0]
    return N, (None if len(idx) == 0 else (int(N - 1 - S - idx[-1]), int(N - 1 - S - idx[0])))


def _emulate_plan(cases, mask):
    rec = np.zeros(len(cases), dtype=[("R", "<i8"), ("S", "<i8"), ("mo", "<i8"), ("m", "<u8")])
    for i, (R, S, mo) in enumerate(cases):
        rec[i] = (R, S, mo, mask)
    raw = np.frombuffer(_run("plan", rec.tobytes()), np.int64).reshape(-1, 7)
    return [tuple(int(v) for v in row) for row in raw]


def test_job_plan_equals_old_planner_and_reference(built):
    mask = _quirk_mask()
    assert mask != 0   # the corner exists with this libm (k = 29, ...)
    rng = np.random.RandomState(4)
    cases = []
    for k in list(range(1, 31)):
        p = 1 << k
        for n in (p - 1, p, p + 1):               # R + S around every power of two, quirk lengths included
            for S in (1, 2, n // 2, n - 1):
                R = n - S
                if R < 0 or S < 0:
                    continue
                for mo in (NONE, 0, 1, 6000, -1, -5, p, -p, 1 << 41, -(1 << 41), 1 << 62):
                    cases.append((R, S, mo))
    for _ in range(3000):                          # random shapes, tiny references (negative-slice corners)
        R = int(rng.choice([0, 1, 2, 3, rng.randint(0, 50), rng.randint(0, 1 << 20)]))
        S = int(rng.choice([0, 1, 2, rng.randint(1, 100), rng.randint(1, 1 << 20)]))
        mo = int(rng.choice([NONE, rng.randint(-200, 200), rng.randint(-(1 << 21), 1 << 21)]))
        cases.append((R, S, mo))
    got = _emulate_plan(cases, mask)
    n_checked = 0
    for (R, S, mo), g in zip(cases, got):
        assert g == _old_planner(R, S, mo, mask), (R, S, mo, g)
        if g[0] != 1 and R + S <= 1 << 16 and abs(mo) < 1 << 20 or (mo == NONE and g[0] != 1 and R + S <= 1 << 16):
            N, win = _python_window(R, S, mo)
            assert g[1] == N, (R, S, mo)
            if win is None:
                assert g[0] == 2 and g[6] == N - 1 - S
            else:
                assert g[0] == 0 and (g[4], g[5]) == win, (R, S, mo, g, win)
            n_checked += 1
    assert n_checked > 1000


def test_mask_window_bound(built):
    """The envelope of b2_sync_tracks_gss: for 0 <= max_offset_samples the surviving window holds at most
    2 max_offset_samples offsets whatever R and S are."""
    mask = _quirk_mask()
    rng = np.random.RandomState(8)
    cases = [(int(rng.randint(1, 1 << 22)), int(rng.randint(1, 1 << 22)), int(rng.randint(0, 16385)))
             for _ in range(5000)]
    cases += [(R, S, mo) for R in (1, 2, 3, 100) for S in (1, 2, 5, 1000, 70000) for mo in (0, 1, 2, 16384)]
    for (R, S, mo), g in zip(cases, _emulate_plan(cases, mask)):
        if g[0] == 0:
            assert g[5] - g[4] + 1 <= 2 * mo, (R, S, mo, g)


# ---------------------------------------------------------------- ABI

def test_sync_tracks_gss_is_exported(built):
    from ffsubsync_b200 import _native
    assert "b2_sync_tracks_gss" in _native.EXPORTS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), "b2_sync_tracks_gss")
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    assert "int b2_sync_tracks_gss(" in header
    # a handle-less call is refused before anything is read
    assert _native.load().b2_sync_tracks_gss(None, None, None, 0, None, 0, 16000, 100, 0.0, 0, -1, -1, None, None,
                                             None, None, None, 1, 0.0, 0, None, None, None, None, None, None, None,
                                             0) == -1


def test_sync_tracks_gss_raises_without_gpu(built):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from ffsubsync_b200 import _native
    with pytest.raises(_native.NativeError):
        h = _native.get_handle()
        h.sync_tracks_gss(np.zeros(1600, np.int16), [0, 1600], [0], 16000, 100, 0.0, 100000, -1, -1,
                          [1.0], [2.0], None, [0, 1], [1.0], 0.0, 100)


def test_batch_synchronizer_ratio_list():
    from ffsubsync_b200 import _native
    from ffsubsync_b200.batch import BatchSynchronizer
    from ffsubsync_b200.constants import framerate_ratios_to_try

    def make(r):
        try:
            return BatchSynchronizer(r)
        except _native.NativeError:   # no GPU here: the ratio list was accepted before the handle was made
            return None

    for bad in ([None, 1.0], [1.0, None, 1.1], [None, None], [None]):
        with pytest.raises(ValueError):
            BatchSynchronizer(bad)
    make([1.0, None])
    make(framerate_ratios_to_try(gss=True))


def test_combine_gss_rule():
    from ffsubsync_b200.gss_batch import GssResult, combine_gss
    K = 2
    bs = np.array([5.0, 5.0, 5.0, 0.0, 5.0, 5.0])
    bo = np.array([1, 1, 1, 0, 1, 1], np.int32)
    bk = np.array([0, 1, 0, -1, 0, 0], np.int32)
    g = GssResult(score=np.array([6.0, 5.0, 4.0, 1.0, 9.0, -np.inf]), offset=np.array([2, 2, 2, 3, 7000, 4], np.int32),
                  ratio=np.array([1.01, 1.02, 1.03, 1.04, 1.05, 1.06]), evals=np.zeros((6, 17)),
                  status=np.array([0, 0, 0, 0, 0, 2], np.int32))
    s, o, k, r, a_s, a_o = combine_gss(bs, bo, bk, g, K, 6000, np.arange(12.0), np.arange(12, dtype=np.int32))
    assert list(k) == [2, 1, 0, 2, 0, 0]         # wins; exact tie keeps the grid; loses; no grid survivor; filter
    assert list(s) == [6.0, 5.0, 5.0, 1.0, 5.0, 5.0] and list(o) == [2, 1, 1, 3, 1, 1]
    assert a_s.reshape(6, 3)[:, 2].tolist() == list(g.score) and a_o.reshape(6, 3)[:, :2].ravel().tolist() == list(range(12))
    g2 = g._replace(status=np.array([1, 0, 0, 0, 0, 0], np.int32))
    s, o, k, r, _, _ = combine_gss(bs, bo, bk, g2, K, 6000)
    assert k[0] == 0 and np.isnan(r[0]) and r[1] == 1.02


def test_constants_list_has_gss():
    from ffsubsync_b200.constants import framerate_ratios_to_try
    lst = framerate_ratios_to_try(gss=True)
    assert lst[-1] is None and all(x is not None for x in lst[:-1])


def _gather_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    from ffsubsync_b200 import distributed as D
    D.init_from_env("gloo")
    track_video = np.repeat(np.arange(4), [3, 1, 0, 2])
    _, _, t0, t1 = D.shard_videos(track_video, rank, world)
    T = len(track_video)

    def rows(a, b):
        return {"best_score": torch.arange(a, b, dtype=torch.float64) * 2.5,
                "best_k": torch.arange(a, b, dtype=torch.int32),
                "gss_ratio": torch.tensor([0.9 + 0.01 * t if t != 3 else float("nan") for t in range(a, b)],
                                          dtype=torch.float64)}

    got = D.gather_track_results(rows(t0, t1), track_video, rank, world, dst=None)
    want = rows(0, T)
    ok = set(got) == set(want) and all(torch.equal(got[k].nan_to_num(-1), want[k].nan_to_num(-1)) for k in want)
    pair = D.gather_pair_results(rows(*D.shard_pairs(5, rank, world)), 5, rank, world)
    ok = ok and ((pair is None) if rank else torch.equal(pair["best_k"], torch.arange(5, dtype=torch.int32)))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()
    q.put((rank, ok))


def test_gather_carries_gss_ratio_gloo_world_size_2():
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gather_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert sorted(q.get(timeout=5) for _ in range(2)) == [(0, True), (1, True)]
