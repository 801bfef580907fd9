"""CPU checks of the per-segment offsets (b2_split_tracks): the oracle's programme against exhaustive enumeration,
its no-split answer against the aligner oracle, the kernel arithmetic (csrc/split.cuh) run thread by thread
(tests/host_emul/split_emul.cu) against the oracle bit for bit, and the ABI symbols and refusals."""
import itertools
import math
import os
import re
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from oracle import aligner_oracle as ao
from oracle import split_oracle as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "host_emul", "split_emul")


def _random_case(rng, R, S, label):
    m = rng.rand(R) < 0.5
    mask = np.zeros(S, bool)
    for _ in range(int(rng.randint(0, 4))):
        a = int(rng.randint(0, S))
        mask[a: a + int(rng.randint(1, 3))] = True
    return np.where(m, 1.0, label), mask


def _table(ref, mask, offsets, level=1.0):
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(1.0 / level if level < 1 else 1.0, beta)
    units = sp.units_of(sp.runs_of(mask), len(mask))
    return units, m, lv, [[sp.unit_score_brute(m, mask, u, o, lv) for o in offsets] for u in units]


@pytest.mark.parametrize("seed", range(40))
def test_programme_equals_enumeration(seed):
    """Every assignment of offsets to the units (at most 4 units, windows up to 9), scored with the penalty per change:
    the programme's path attains the optimum; where exactly one assignment does, the path is that assignment; and its
    split_score is the path's sum without penalties.  (Among several optimal assignments the choice is fixed by the
    programme's local rules, which test_kernel_arithmetic_equals_oracle checks cell by cell.)"""
    rng = np.random.RandomState(seed)
    R, S = int(rng.randint(3, 12)), int(rng.randint(3, 12))
    ref, mask = _random_case(rng, R, S, [0.0, 0.3, -0.5][seed % 3])
    o_lo = int(rng.randint(-S, R))
    W = int(rng.randint(1, 10))
    offsets = list(range(o_lo, o_lo + W))
    units, m, lv, U = _table(ref, mask, offsets)
    assert len(units) <= 4   # _random_case draws at most three runs
    pen = [0.0, 0.5, 2.0, 7.0, math.inf][seed % 5]
    path, score = sp.solve(U, offsets, pen)
    best, argbest = -math.inf, []
    for choice in itertools.product(range(W), repeat=len(units)):
        v = U[0][choice[0]]
        for j in range(1, len(units)):
            v = v + U[j][choice[j]] - (pen if choice[j] != choice[j - 1] else 0.0)
        if v > best:
            best, argbest = v, [choice]
        elif v == best:
            argbest.append(choice)
    exact = lv[0] == 1.0 and lv[1] == -1.0
    if exact and len(argbest) == 1:
        assert path == [offsets[i] for i in argbest[0]], (seed, path, argbest)
    got = U[0][offsets.index(path[0])]
    for j in range(1, len(units)):
        got = got + U[j][offsets.index(path[j])] - (pen if path[j] != path[j - 1] else 0.0)
    if exact:   # +-1: exact integers, every order agrees
        assert got == best, (seed, path, got, best)
    else:
        assert abs(got - best) <= 1e-9 * max(1.0, abs(best)), (seed, got, best)
    assert score == sum_path(U, offsets, path)


def sum_path(U, offsets, path):
    s = 0.0
    for j, o in enumerate(path):
        s = s + U[j][offsets.index(o)]
    return s


@pytest.mark.parametrize("seed", range(24))
def test_no_splits_is_the_aligner(seed):
    """split_penalty = inf: one offset, the aligner oracle's best (exactly for +-1, within the run path's epsilon
    otherwise), over labels 0 / 0.3 / -0.5, levels 1 / 0.96, R << S, S << R and windows past both ends."""
    rng = np.random.RandomState(100 + seed)
    label = [0.0, 0.3, -0.5][seed % 3]
    ratio = [1.0, 1 / 0.96][(seed // 3) % 2]
    R, S_cues = [(40, 300), (300, 40), (150, 150)][seed % 3]
    ref = np.where(rng.rand(R) < 0.4, 1.0, label)
    n = int(rng.randint(1, 8))
    cs = np.sort(np.round(rng.uniform(0, S_cues / 100.0, n), 2))
    ce = np.round(cs + rng.uniform(0.02, 0.3, n), 2)
    mos = [None, 30, 400][seed % 3]
    co, ns, sc = sp.split_track(ref, cs, ce, None, ratio, 100, 0.0, mos, math.inf)
    sub = sp.ro.rasterize(cs, ce, None, 100, 0.0, ratio)[0].astype(np.float32)   # the level as the calls round it
    s_want, o_want = ao.exact_align(ref, sub, mos)
    assert ns == 1 and len(set(co)) == 1
    if label == 0.0 and ratio == 1.0:   # +-1: exact
        assert co[0] == o_want and sc == s_want
    else:   # the chosen offset attains the maximum within the run path's margin
        assert abs(ao.exact_score(ref, sub, co[0]) - s_want) <= 1e-9 * max(1.0, abs(s_want))
        assert abs(sc - s_want) <= 1e-9 * max(1.0, abs(s_want))


def _emulate(m, mask, o_lo, W, level, beta, pen):
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        with open(fin, "wb") as f:
            f.write(struct.pack("<4if2d", len(m), len(mask), o_lo, W, level, beta, pen))
            f.write(np.asarray(m, np.uint8).tobytes())
            f.write(np.asarray(mask, np.uint8).tobytes())
        subprocess.check_call([EXE, fin, fout])
        raw = open(fout, "rb").read()
    nu = struct.unpack_from("<i", raw)[0]
    mx, args = [], []
    for j in range(nu):
        a, b = struct.unpack_from("<di", raw, 4 + 12 * j)
        mx.append(a)
        args.append(b)
    sw = np.frombuffer(raw[4 + 12 * nu:], np.uint8).reshape(max(nu - 1, 0), W)
    return mx, args, sw


@pytest.mark.parametrize("seed", range(16))
def test_kernel_arithmetic_equals_oracle(seed):
    """split.cuh thread by thread: every unit's maximum and argmax and every switch bit equal the oracle's
    programme bit for bit.  Runs at frame 0 and S - 1, one-frame runs, windows over both reference ends."""
    rng = np.random.RandomState(200 + seed)
    R, S = int(rng.randint(1, 400)), int(rng.randint(2, 400))
    label = [0.0, 0.3, -0.5, 0.96][seed % 4]
    level = [1.0, np.float32(1 / (25 / 24.0))][seed % 2]
    ref = np.where(rng.rand(R) < 0.5, 1.0, label)
    mask = rng.rand(S) < [0.1, 0.5, 0.9][seed % 3]
    mask[0] = mask[-1] = bool(seed % 2)
    if seed % 5 == 0:
        mask[:] = False
    W = int(rng.randint(1, 200))
    o_lo = int(rng.randint(-S - 20, max(R + 20 - W, -S - 19))) if seed % 4 else -S
    pen = [0.0, 1.5, 30.0, math.inf][seed % 4]
    offsets = list(range(o_lo, o_lo + W))
    m, beta = sp.ref_levels(ref)
    lv = sp.levels(1.0 / float(level), beta)
    units = sp.units_of(sp.runs_of(mask), S)
    U = [sp.unit_scores(m, u, offsets, lv) for u in units]
    mx, args, sw = _emulate(m, mask, o_lo, W, float(level), beta, pen)
    assert len(mx) == len(units)
    V = list(U[0])
    for j in range(len(units)):
        if j:
            c = pmx - pen
            want_sw = [c > V[i] for i in range(W)]
            assert list(sw[j - 1].astype(bool)) == want_sw, (seed, j)
            V = [U[j][i] + (c if want_sw[i] else V[i]) for i in range(W)]
        pmx = max(V)
        k = max(i for i in range(W) if V[i] == pmx)
        assert mx[j] == pmx and args[j] == offsets[k], (seed, j, mx[j], pmx, args[j], offsets[k])
    # brute-force counts agree with the frame sums the oracle uses
    for u in units[:3]:
        for o in offsets[:: max(1, W // 7)]:
            assert sp.unit_score_brute(m, mask, u, o, lv) == sp.unit_scores(m, u, [o], lv)[0]


def test_symbols_and_handleless_refusal():
    from ffsubsync_b200 import _native
    header = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    for name in ("b2_split_tracks", "b2_apply_split"):
        assert name in _native.EXPORTS and re.search(r"\b%s\s*\(" % name, header)
    assert "ffsubsync/aligners.py:24-86" in header and "ffsubsync/ffsubsync.py:272-286" in header
    lib = _native.load()
    assert lib.b2_split_tracks(None, None, 1, None, 0, None, 0, None, None, None, None, None, 100, 0.0, 0, 1.0,
                               None, None, None, 0) == -1
    assert lib.b2_apply_split(None, None, None, None, 0, None, None, None, 100, 0.0, None, None, None, 0) == -1


def test_three_level_reference_is_named():
    ref = np.array([1.0, 0.0, 1.0, 0.5, 0.0])
    with pytest.raises(sp.ThreeLevels) as e:
        sp.ref_levels(ref)
    assert e.value.args[0] == 3
    assert sp.ref_levels(np.ones(4))[1] == 0.0
