"""CPU suite for the reference's chunk loop (oracle/chunk_oracle.py) and the library's energy / ZCR detector calls.

The reference calls the detector once per (2 fr // sr) * 10000 bytes it reads, and every call restarts the window grid.
For energy / ZCR that equals one call over the whole video only where a read is a whole number of windows; at
22.05 kHz (2 205 000 samples of 221) it is not, and the batched sync calls' planner (csrc/sync_plan.h) must cut the
videos into the reference's calls there and nowhere else."""
import numpy as np
import pytest

from oracle import chunk_oracle as co
from oracle import vad_oracle as vo
from sync_plan import plan

DIVIDING = [8000, 11025, 12000, 16000, 24000, 32000, 44100, 48000, 96000]


def _video(fr, seconds, seed):
    """Seeded PCM of runs of silence, voiced speech and loud hiss, with a loud ragged tail."""
    fpw = vo.frames_per_window(fr, 100)
    rng = np.random.RandomState(seed)
    n = int(seconds * fr)
    cls = np.repeat(rng.choice(3, -(-n // fpw) // 7 + 1, p=[0.45, 0.4, 0.15]), 7)[: -(-n // fpw)]
    return vo.synth_pcm(cls.astype(np.uint8), fpw, seed)[:n]


@pytest.mark.parametrize("fr", DIVIDING)
def test_chunk_loop_is_one_call_where_reads_divide_into_windows(fr):
    pcm = _video(fr, 230.5, fr % 101)
    for label in (0.0, 0.3):
        one = vo.energy_zcr_detect(pcm, 100, fr, label)
        assert np.array_equal(co.chunk_loop("energy_zcr", pcm, fr, 100, label), one)


def test_chunk_loop_differs_from_one_call_at_22050():
    """The premise: at 22.05 kHz each 100 s call ends in an 83-sample partial window and the next starts a new grid,
    so a 250 s video has one frame more, and its frames after the first call are shifted."""
    fr = 22050
    pcm = _video(fr, 250.0, 7)
    one = vo.energy_zcr_detect(pcm, 100, fr, 0.0)
    loop = co.chunk_loop("energy_zcr", pcm, fr, 100, 0.0)
    assert co.read_samples(fr) == 2205000 and co.read_samples(fr) % 221 == 83
    assert len(one) == -(-len(pcm) // 221) and len(loop) == 2 * 9978 + -(-(len(pcm) - 2 * 2205000) // 221)
    assert len(loop) == len(one) + 1
    assert np.array_equal(loop[:9977], one[:9977]) and loop[9977] == 0.0
    assert np.count_nonzero(loop[: len(one)] != one) > 100


@pytest.mark.parametrize("fr", DIVIDING + [22050])
def test_num_windows_and_call_samples(fr):
    from ffsubsync_b200 import _native
    lib = _native.load()
    fpw = vo.frames_per_window(fr, 100)
    call = lib.b2_vad_call_samples(fr, 100)
    assert call == (co.read_samples(fr) if fr == 22050 else 0)
    for n in (0, 1, fpw - 1, fpw, co.read_samples(fr) - 1, co.read_samples(fr), co.read_samples(fr) + 1,
              2 * co.read_samples(fr) + fpw // 2, int(2.5 * co.read_samples(fr))):
        pcm_len = len(co.chunk_loop("energy_zcr", np.zeros(n, np.int16), fr))
        assert lib.b2_vad_num_windows(n, fr, 100) == pcm_len, n


# ---------------------------------------------------------------- the planner's tables

def _req(fr, lens, **over):
    pcm_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    V = len(lens)
    req = dict(pcm_off=pcm_off, track_video=np.arange(V, dtype=np.int32), cue_start=np.tile([1.0], V),
               cue_end=np.tile([2.0], V), cue_off=np.arange(V + 1), ratios=[1.0], energy_threshold=100000,
               frame_rate=fr, lane=1)
    req.update(over)
    return req


def test_plan_energy_chunk_table_at_22050():
    """Videos of 0, 1, a call - 1, a call, a call + 1 and 2.5 calls: one table entry per call from each video's start,
    the chunk loop's frames per call, no tail floor read, and floats (never packed words) for the lane test."""
    fr, C = 22050, 2205000
    lens = [0, 1, C - 1, C, C + 1, 5 * C // 2]
    p = plan(**_req(fr, lens))
    assert p["status"] == 0, p["err"]
    assert p["call"].tolist() == [C, 1]
    calls = [[]] + [[n] if n <= C else [C] * (n // C) + ([n % C] if n % C else []) for n in lens[1:]]
    assert np.diff(p["ch_pcm"]).tolist() == [x for c in calls for x in c]
    assert np.diff(p["ch_first"]).tolist() == [len(c) for c in calls]
    assert np.diff(p["ch_out"]).tolist() == [-(-x // 221) for c in calls for x in c]
    assert np.diff(p["ref_off"]).tolist() == [sum(-(-x // 221) for x in c) for c in calls]
    for v, n in enumerate(lens):
        assert p["ref_off"][v + 1] - p["ref_off"][v] == len(co.chunk_loop("energy_zcr", np.zeros(n, np.int16), fr))


@pytest.mark.parametrize("fr", [16000, 48000, 8000, 44100])
def test_plan_keeps_one_entry_per_video_where_calls_divide(fr):
    fpw = vo.frames_per_window(fr, 100)
    C = co.read_samples(fr)
    lens = [0, C + 1, 5 * C // 2, 3 * fpw]
    p = plan(**_req(fr, lens))
    assert p["status"] == 0, p["err"]
    assert p["call"].tolist() == [0, 0] and p["ch_pcm"].size == 0 and p["ch_first"].size == 0
    assert np.diff(p["ref_off"]).tolist() == [-(-n // fpw) for n in lens]


def test_plan_auditok_call_is_its_chunk():
    p = plan(**_req(22050, [1000, 5000], detector=1, chunk_samples=3000))
    assert p["status"] == 0, p["err"]
    assert p["call"].tolist() == [3000, 1] and np.diff(p["ch_pcm"]).tolist() == [1000, 3000, 2000]
