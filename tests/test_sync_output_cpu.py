"""CPU suite for try_sync's epilogue over the batched calls (b2_apply_sync: synced cue times, the low-quality gate,
suppression and sync_was_successful).

Checks what can be checked without a GPU: the oracle against the reference's own try_sync
(tests/golden/make_golden_sync_output.py), the package's assess_alignment_quality / reasons / SubtitleShifter, the
header arithmetic of sync_output.cuh run on the CPU (tests/host_emul/sync_output_emul) against Python's timedelta
on the fixture's edges and on 10^6 seeded random (time, ratio, offset) triples, and the symbol's signature."""
import json
import math
import os
import re
import subprocess
import sys
import tempfile
from datetime import timedelta

import numpy as np
import pytest

from conftest import ROOT
from oracle import sync_output_oracle as so

GOLDEN = os.path.join(ROOT, "tests", "golden", "sync_output.json")
EMUL = os.path.join(ROOT, "tests", "host_emul", "sync_output_emul")
US = timedelta(microseconds=1)

IN_DT = np.dtype([(k, "<f8") for k in ("t", "ratio", "gss_ratio", "best_score", "apply", "min_score", "max_off",
                                        "max_dev", "suppress")]
                 + [(k, "<i8") for k in ("best_offset", "best_k", "sample_rate", "gate", "has_suppress", "has_gss")])
OUT_DT = np.dtype([("scale", "<f8"), ("offset_seconds", "<f8")]
                  + [(k, "<i8") for k in ("status", "shift_us", "synced_us", "scaled_us")])


def _f(x):
    return float(x) if isinstance(x, str) else x


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    return ge


@pytest.fixture(scope="module")
def golden():
    with open(GOLDEN) as fh:
        return json.load(fh)


def _rule(s):
    return dict(apply_offset_seconds=s["apply_offset_seconds"], gate=s["gate"], min_score=_f(s["min_score"]),
                quality_max_offset_seconds=_f(s["quality_max_offset_seconds"]),
                max_framerate_deviation=_f(s["max_framerate_deviation"]),
                suppress=None if s["suppress"] is None else _f(s["suppress"]))


def _oracle(s):
    n = len(s["cue_start"])
    return so.apply_sync([_f(s["best_score"])], [s["best_offset"]], [s["best_k"]],
                         [_f(s["gss_ratio"])] if s["gss"] else None, s["cue_start"], s["cue_end"], [0, n],
                         s["ratios"], 100, **_rule(s))


# ---------------------------------------------------------------- oracle vs the reference's try_sync

def test_fixture_covers_the_edges(golden):
    names = {s["name"] for s in golden["scenarios"]}
    assert {"qg_low_quality_written_original", "qg_applied_when_acceptable", "qg_ignored_without_flag", "failed",
            "gss", "scale_1.1", "scale_0.9", "score_equals_min", "offset_equals_max", "suppress_zero",
            "suppress_none", "four_hours", "half_us_products", "apply_offset"} <= names
    # 1.1 - 1.0 > 0.1 is true in float64: the reference gates a 1.1 scale at the default deviation
    assert [s["reasons"] for s in golden["scenarios"] if s["name"] == "scale_1.1"] == [
        ["framerate deviation 0.100 > 0.100"]]


def test_oracle_reproduces_try_sync(golden):
    for s in golden["scenarios"]:
        su, eu, off, sc, st = _oracle(s)
        st = int(st[0])
        got = [[int(a), int(b)] for a, b in zip(su, eu)]
        name = s["name"]
        assert bool(st & so.WRITTEN) == (s["written"] is not None), name
        assert bool(st & so.SUCCESSFUL) == s["sync_was_successful"], name
        assert bool(st & so.FAILED) == (s["best_k"] == -1), name
        assert bool(st & so.APPLIED) == (s["shifted"] is not None), name
        assert bool(st & so.SUPPRESSED) == (s["shifted"] is not None and s["written"] is None), name
        if st & so.APPLIED:
            assert got == s["shifted"], name
        if s["written"] is not None:
            assert got == s["written"], name
        if st & (so.FAILED | so.LOW_SCORE | so.LOW_OFFSET | so.LOW_FRAMERATE):
            # the originals: timedelta(seconds=t) is the parsed cue
            assert got == [[so.td_us(a), so.td_us(b)] for a, b in zip(s["cue_start"], s["cue_end"])], name
        # result["offset_seconds"] / ["framerate_scale_factor"] are set exactly for the tracks the gate let through
        if s["offset_seconds"] is not None:
            assert off[0] == _f(s["offset_seconds"]) and sc[0] == _f(s["framerate_scale_factor"]), name
            assert not st & (so.FAILED | so.LOW_SCORE | so.LOW_OFFSET | so.LOW_FRAMERATE), name
        else:
            assert st & (so.FAILED | so.LOW_SCORE | so.LOW_OFFSET | so.LOW_FRAMERATE), name
        low = [st & b != 0 for b in (so.LOW_SCORE, so.LOW_OFFSET, so.LOW_FRAMERATE)]
        want = s["reasons"] or []
        assert low == [any(r.startswith(p) for r in want) for p in ("score", "|offset|", "framerate")], name


def test_package_gate_and_reasons(golden):
    from ffsubsync_b200 import sync_output
    for a in golden["assess"]:
        score, off, scale, ms, mo, md = a["args"]
        assert sync_output.assess_alignment_quality(score, off, scale, min_score=ms, max_offset_seconds=mo,
                                                    max_framerate_deviation=md) == a["reasons"]
    for s in golden["scenarios"]:
        if not s["reasons"]:
            continue
        su, eu, off, sc, st = _oracle(s)
        r = _rule(s)
        assert sync_output.reasons(int(st[0]), _f(s["best_score"]), off[0], sc[0], min_score=r["min_score"],
                                   max_offset_seconds=r["quality_max_offset_seconds"],
                                   max_framerate_deviation=r["max_framerate_deviation"]) == s["reasons"], s["name"]
    assert [sync_output.WRITTEN, sync_output.APPLIED, sync_output.SUCCESSFUL, sync_output.FAILED,
            sync_output.SUPPRESSED, sync_output.LOW_SCORE, sync_output.LOW_OFFSET, sync_output.LOW_FRAMERATE] == \
        [so.WRITTEN, so.APPLIED, so.SUCCESSFUL, so.FAILED, so.SUPPRESSED, so.LOW_SCORE, so.LOW_OFFSET,
         so.LOW_FRAMERATE]


def test_constants_and_shifter():
    from ffsubsync_b200 import constants
    from ffsubsync_b200.subtitle_transformers import SubtitleScaler, SubtitleShifter, cues_from_seconds
    assert (constants.DEFAULT_APPLY_OFFSET_SECONDS, constants.DEFAULT_MIN_SCORE,
            constants.DEFAULT_QUALITY_MAX_OFFSET_SECONDS, constants.DEFAULT_MAX_FRAMERATE_DEVIATION) == (0, 0.0, 30.0, 0.1)
    cues = cues_from_seconds([1.234567, 10.0], [2.0000005, 11.0])
    scaled = SubtitleScaler(25.0 / 24.0).fit(cues).transform()
    shifted = SubtitleShifter(-1.2345675).fit(scaled).transform()
    td = timedelta(seconds=-1.2345675)
    assert [(c.start, c.end) for c in shifted] == [(c.start + td, c.end + td) for c in scaled]
    assert SubtitleShifter(td).td_seconds is td


# ---------------------------------------------------------------- the header's arithmetic on the CPU

def _emul(rec):
    with tempfile.TemporaryDirectory() as tmp:
        fin, fout = os.path.join(tmp, "in.bin"), os.path.join(tmp, "out.bin")
        np.ascontiguousarray(rec, IN_DT).tofile(fin)
        subprocess.check_call([EMUL, fin, fout])
        return np.fromfile(fout, OUT_DT)


def _record(t, ratio, best_offset, apply=0.0, best_k=0, gss_ratio=0.0, has_gss=0, best_score=1.0, gate=0,
            min_score=0.0, max_off=30.0, max_dev=0.1, suppress=None, sample_rate=100):
    return (t, ratio, gss_ratio, best_score, apply, min_score, max_off, max_dev, 0.0 if suppress is None else suppress,
            best_offset, best_k, sample_rate, gate, suppress is not None, has_gss)


def test_emulator_matches_the_oracle_on_the_fixture(built, golden):
    rec, want = [], []
    for s in golden["scenarios"]:
        r = _rule(s)
        k, ratios = s["best_k"], s["ratios"]
        # the emulator's grid is one ratio: the winning one (or any, for the search's point and failures)
        ratio = ratios[k] if 0 <= k < len(ratios) else ratios[0]
        ek = 0 if 0 <= k < len(ratios) else (1 if k == len(ratios) else -1)
        su, eu, off, sc, st = _oracle(s)
        for i, t in enumerate(s["cue_start"] + s["cue_end"]):
            rec.append(_record(t, ratio, s["best_offset"], r["apply_offset_seconds"], ek,
                               _f(s["gss_ratio"]) if s["gss"] else 0.0, int(s["gss"]), _f(s["best_score"]),
                               int(r["gate"]), r["min_score"], r["quality_max_offset_seconds"],
                               r["max_framerate_deviation"], r["suppress"]))
            want.append((int(st[0]), off[0], sc[0], int(np.concatenate([su, eu])[i])))
    got = _emul(rec)
    for g, w, s in zip(got, want, [r for r in rec]):
        assert int(g["status"]) == w[0] and int(g["synced_us"]) == w[3], (s, g, w)
        assert (g["offset_seconds"] == w[1] or math.isnan(w[1]) and math.isnan(g["offset_seconds"]))
        assert (g["scale"] == w[2] or math.isnan(w[2]) and math.isnan(g["scale"]))


def test_emulator_rounding_bit_for_bit(built):
    """10^6 seeded (time, ratio, offset) triples: timedelta(seconds=t * ratio) + timedelta(seconds=offset)."""
    rng = np.random.default_rng(20261016)
    n = 1_000_000
    mag = 10.0 ** rng.uniform(-6, 4.2, n)                  # 1 us .. 4.4 h
    t = np.where(rng.random(n) < 0.1, -mag, mag)
    t = np.where(rng.random(n) < 0.5, np.round(t * 1e6) / 1e6, t)   # parsed times: whole microseconds
    grid = np.array([1.0, 24 / 23.976, 25 / 23.976, 25 / 24, 23.976 / 24, 23.976 / 25, 24 / 25, 0.5, 1.5, 2.5])
    ratio = np.where(rng.random(n) < 0.5, grid[rng.integers(0, len(grid), n)], rng.uniform(0.9, 1.1, n))
    best_offset = rng.integers(-(1 << 20), 1 << 20, n)
    apply = np.where(rng.random(n) < 0.5, 0.0, rng.uniform(-100, 100, n))
    apply = np.where(rng.random(n) < 0.2, np.round(apply * 2e6) / 2e6, apply)        # half-microsecond shifts
    rec = np.zeros(n, IN_DT)
    rec["t"], rec["ratio"], rec["best_offset"], rec["apply"] = t, ratio, best_offset, apply
    rec["best_score"], rec["sample_rate"], rec["max_dev"] = 1.0, 100, 0.1
    got = _emul(rec)
    td = timedelta
    bad = 0
    for i in range(n):
        ti, ri, oi = float(t[i]), float(ratio[i]), int(best_offset[i]) / 100.0 + float(apply[i])
        scaled = td(seconds=ti * ri) // US
        shift = td(seconds=oi) // US
        if (got["scaled_us"][i] != scaled or got["shift_us"][i] != shift or got["synced_us"][i] != scaled + shift
                or got["offset_seconds"][i] != oi or got["status"][i] != so.WRITTEN | so.APPLIED | so.SUCCESSFUL):
            bad += 1
    assert bad == 0


def test_emulator_search_point_and_failures(built):
    rec = [_record(12.5, 1.0, 10, best_k=1, gss_ratio=g, has_gss=1) for g in (0.9, 1.1, 0.95, 0.8999999, 1.1000001,
                                                                              float("nan"))]
    rec += [_record(12.5, 1.0, 10, best_k=k) for k in (-1, -2, 1, 7)]   # no search: k == K fails too
    got = _emul(rec)
    assert [int(s) & so.FAILED != 0 for s in got["status"]] == [False] * 3 + [True] * 7
    assert [int(u) for u in got["synced_us"][3:]] == [12_500_000] * 7
    assert got["scale"][:3].tolist() == [0.9, 1.1, 0.95] and np.isnan(got["scale"][3:]).all()


# ---------------------------------------------------------------- ABI

def test_export_and_header_signature(built):
    from ffsubsync_b200 import _native
    hdr = open(os.path.join(ROOT, "include", "ffsubsync_b200.h")).read()
    m = re.search(r"int b2_apply_sync\((.*?)\);", hdr, re.S)
    assert m
    params = [p for p in re.sub(r"/\*.*?\*/", "", m.group(1)).split(",") if p.strip()]
    lib = _native.load()
    assert len(lib.b2_apply_sync.argtypes) == len(params) == 25
    assert "b2_apply_sync" in _native.EXPORTS
    for name, bit in (("WRITTEN", 1), ("APPLIED", 2), ("SUCCESSFUL", 4), ("FAILED", 8), ("SUPPRESSED", 16),
                      ("LOW_SCORE", 32), ("LOW_OFFSET", 64), ("LOW_FRAMERATE", 128)):
        assert re.search(r"B2_SYNC_%s = %d\b" % (name, bit), hdr), name
    # refused without a handle, before anything is read
    assert lib.b2_apply_sync(*([None] * 5 + [0] + [None] * 4 + [0, 100, 0.0, 0, 0.0, 30.0, 0.1, 0, 0.0]
                               + [None] * 5 + [0])) == -1
