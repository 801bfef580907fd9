"""CPU suite for the batched sync calls' host planner (csrc/sync_plan.h): the sub-batch cuts of the pipeline and
the status every bad argument gets, checked on the planner the five b2_sync_* entry points run before they launch
anything (the GPU suites check the same statuses through a handle)."""
import numpy as np
import pytest

from sync_plan import plan

GRID = [0.96, 1.0, 1.04]
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1


def _tracks(n_videos=4, per_video=(1, 2, 0, 3), samples=16000 * 30, **over):
    """A valid b2_sync_tracks request: video v has per_video[v] tracks, each of three cues."""
    tv = np.repeat(np.arange(n_videos), per_video).astype(np.int32)
    T = len(tv)
    starts = np.tile([1.0, 5.0, 9.5], T)
    req = dict(pcm_off=np.arange(n_videos + 1) * samples, track_video=tv, cue_start=starts, cue_end=starts + 2.0,
               cue_off=np.arange(T + 1) * 3, ratios=GRID, energy_threshold=100000)
    req.update(over)
    return req


def _ok(p):
    assert p["status"] == 0, p["err"]
    return p


# ---------------------------------------------------------------- sub-batch cuts

def test_small_batches_and_the_group_kernel_stay_unpipelined():
    p = _ok(plan(**_tracks(lane=1)))
    assert p["n_sub"].tolist() == [1, 0] and p["cut"].tolist() == [0, 4]
    V = 120
    p = _ok(plan(**_tracks(V, [1] * V, 1600, lane=0)))   # 120 tracks, not lane-eligible
    assert p["n_sub"].tolist() == [1, 0]


def test_default_cuts_are_a_third_of_the_tracks_each():
    V = 120
    p = _ok(plan(**_tracks(V, [1] * V, 1600, lane=1)))
    assert p["n_sub"].tolist() == [3, (132 * 54 + 50) // 100]
    assert p["cut"].tolist() == [0, 40, 80, 120]   # one track per video: T*i/3 exactly
    p = _ok(plan(**_tracks(V, [1] * V, 1600, lane=1, sm_count=114)))
    assert p["n_sub"][1] == (114 * 54 + 50) // 100


@pytest.mark.parametrize("n_sub", [2, 3, 5, 7])
def test_cuts_balance_tracks_and_leave_no_sub_batch_empty(n_sub):
    rng = np.random.RandomState(n_sub)
    per = rng.randint(0, 5, 40)
    per[[0, 17, 18, 19, 39]] = 0                  # videos without tracks, leading and trailing ones included
    p = _ok(plan(**_tracks(40, per, 1600, subbatches=str(n_sub), vad_sms="50")))
    cut, trk = p["cut"], p["trk_off"]
    T = int(per.sum())
    assert cut[0] == 0 and cut[-1] == 40 and np.all(np.diff(cut) > 0)
    assert p["n_sub"].tolist() == [len(cut) - 1, 50]
    assert np.all(np.diff(trk[cut]) > 0)          # every sub-batch holds at least one track
    for v in cut[1:-1]:   # a cut is the first video whose tracks start at or after T*i/n_sub for some i
        assert any(trk[v - 1] < T * i // n_sub <= trk[v] for i in range(1, n_sub))
    assert trk[-1] == T and np.array_equal(trk, np.concatenate([[0], np.cumsum(per)]))


def test_cut_knobs_are_clamped():
    p = _ok(plan(**_tracks(subbatches="1000", vad_sms="-4")))
    assert p["n_sub"][1] == 0 and p["cut"].tolist() == [0, 1, 2, 4]   # T = 6 tracks, no empty sub-batch
    p = _ok(plan(**_tracks(subbatches="0", vad_sms="999")))
    assert p["n_sub"].tolist() == [1, 132]


def test_videos_without_tracks():
    assert _ok(plan(**_tracks(4, [0, 0, 0, 0], subbatches="3")))["cut"].size == 0   # T == 0: nothing to plan
    p = _ok(plan(**_tracks(5, [0, 3, 0, 0, 0], subbatches="3")))
    assert p["cut"].tolist() == [0, 5]         # three tracks of one video: one sub-batch
    assert p["ref_off"].tolist() == (np.arange(6) * 3000).tolist()


# ---------------------------------------------------------------- bad arguments (status, message)

def _status(**req):
    p = plan(**req)
    return p["status"], p["err"]


def test_tracks_bad_arguments():
    c = _tracks()
    tv = c["track_video"]
    for bad in (tv[[1, 0, 2, 3, 4, 5]], np.r_[tv[:-1], 4], np.r_[-1, tv[1:]]):   # decreasing, == V, negative
        st, err = _status(**dict(c, track_video=bad))
        assert st == -1 and "track_video" in err
    pcm_off = c["pcm_off"].copy()
    pcm_off[1] = pcm_off[2] + 1
    assert _status(**dict(c, pcm_off=pcm_off)) == (-1, "sync_tracks: pcm_off not monotone")
    cue_off = c["cue_off"].copy()
    cue_off[1] = cue_off[2] + 1
    assert _status(**dict(c, cue_off=cue_off))[0] == -1
    assert _status(**dict(c, outputs=0)) == (-1, "sync_tracks: null output")
    assert _status(**dict(c, ratios=[])) == (-1, "sync_tracks: bad arguments")
    assert _status(**dict(c, sample_rate=0))[0] == -1
    ends = c["cue_end"].copy()
    ends[4] = np.nan
    st, err = _status(**dict(c, cue_end=ends))
    assert st == -1 and "cue end time" in err and "index 4" in err
    st, err = _status(**dict(c, ratios=[1.0, -1.0]))
    assert st == -1 and "ratio is not a finite positive number" in err
    st, err = _status(**dict(c, start_seconds=np.inf))
    assert st == -1 and "start_seconds" in err


def test_sync_batch_names_itself():
    c = _tracks(3, [1, 1, 1], who="sync_batch")
    c.pop("track_video")
    assert _ok(plan(**c))["trk_off"].tolist() == [0, 1, 2, 3]
    st, err = _status(**dict(c, cue_start=np.r_[1e300, c["cue_start"][1:]]))
    assert st == -1 and err.startswith("sync_batch: cue start time") and "index 0" in err


def _subs(**over):
    """A valid b2_sync_tracks_subs request: videos 0 and 2 take subtitle references, 1 and 3 audio."""
    c = _tracks(who="sync_tracks_subs", pcm_off=[0, 0, 16000 * 30, 16000 * 30, 16000 * 60])
    ref_start = np.array([1.0, 4.0, 8.0, 2.0, 3.0])
    c.update(ref_is_subs=[1, 0, 1, 0], ref_cue_start=ref_start, ref_cue_end=ref_start + 1.5,
             ref_cue_off=[0, 3, 3, 5, 5])
    c.update(over)
    return c


def test_subs_ref_tables():
    p = _ok(plan(**_subs()))
    assert p["sub_video"].tolist() == [0, 2]
    # a subtitle reference is int(max_end * sample_rate) + 2 frames long, an audio one ceil(n / fpw)
    assert np.diff(p["ref_off"]).tolist() == [int(9.5 * 100) + 2, 3000, int(4.5 * 100) + 2, 3000]
    assert p["audio_samples"][0] == 16000 * 60
    p = _ok(plan(**_subs(detector=1, chunk_samples=320000)))   # auditok: one empty chunk per subtitle video
    assert np.diff(p["ch_pcm"]).tolist() == [0, 320000, 160000, 0, 320000, 160000]
    assert p["ch_first"].tolist() == [0, 1, 3, 4, 6] and p["tok_first"].tolist() == [0, 0, 2, 2, 4]
    assert np.diff(p["ref_off"]).tolist() == [952, 3000, 452, 3000]
    # the tokenizer's chunks are the audio videos' ranges, the subtitle references' ranges left out
    assert p["tok_off"].tolist() == [952, 952 + 2000, 952 + 3000 + 452, 952 + 3000 + 452 + 2000]
    assert (p["tok_end"] - p["tok_off"]).tolist() == [2000, 1000, 2000, 1000]


def test_subs_ref_bad_arguments():
    c = _subs()
    st, err = _status(**dict(c, ref_is_subs=[1, 1, 1, 0]))
    assert st == -1 and "non-empty PCM range" in err
    st, err = _status(**dict(c, ref_cue_off=[0, 3, 2, 5, 5]))
    assert st == -1 and "not monotone" in err
    for bad in (np.nan, np.inf, 1e300):
        rs = c["ref_cue_start"].copy()
        rs[4] = bad
        st, err = _status(**dict(c, ref_cue_start=rs))
        assert st == -1 and "reference cue start" in err and "index 4" in err
    re_ = c["ref_cue_end"].copy()
    re_[3] = np.nan
    st, err = _status(**dict(c, ref_cue_end=re_))
    assert st == -1 and "index 3" in err
    st, err = _status(**dict(c, ref_is_subs=[1, 0, 0, 0]))         # cues for a video without a subtitle reference
    assert st == -1 and "ref_is_subs[2] = 0" in err
    st, err = _status(**dict(c, pcm=0))
    assert st == -1 and "null pcm with 960000 samples" in err
    assert _ok(plan(**_subs(pcm=0, pcm_off=[0] * 5, ref_is_subs=[1, 1, 1, 1], ref_cue_off=[0, 3, 4, 5, 5])))
    # references of both kinds at a non-zero label: three levels, so no search
    st, err = _status(**dict(c, label=0.3, gss=1))
    assert st == -6 and "0.3" in err and err.startswith("sync_tracks_subs")
    assert _ok(plan(**dict(c, gss=1)))["two_level"]
    p = _ok(plan(**dict(c, label=0.3, ref_is_subs=[1, 0, 1, 0])))
    assert not p["two_level"] and abs(p["ref_label"] - 0.3) < 1e-7


def test_auditok_bad_arguments():
    c = _tracks(who="sync_tracks_auditok", detector=1, chunk_samples=320 * 5000)
    assert _status(**dict(c, frame_rate=99))[0] == -6
    for kw in (dict(max_length=0), dict(min_length=0.0), dict(min_length=600.0), dict(max_continuous_silence=500.0),
               dict(chunk_samples=-1)):
        assert _status(**dict(c, **kw)) == (-1, "sync_tracks_auditok: bad tokenizer parameters"), kw
    st, err = _status(**dict(c, auditok_label=0.3, gss=1))
    assert st == -6 and "0.3" in err
    assert _ok(plan(**dict(c, auditok_label=0.0, gss=1)))["two_level"]


def test_gss_envelope():
    c = _tracks(who="sync_tracks_gss", gss=1)
    for mos in (INT64_MIN, 16385, 10 ** 9, -1, 1 << 62, INT64_MAX, INT64_MIN + 1):
        st, err = _status(**dict(c, max_offset_samples=mos))
        assert st == -6 and "max_offset_samples" in err, mos
    st, err = _status(**dict(c, label=float("nan")))
    assert st == -6 and "non_speech_label" in err
    n = 16385
    st, err = _status(**dict(c, cue_start=np.arange(n) * 0.02, cue_end=np.arange(n) * 0.02 + 0.01,
                             cue_off=[0, n] + [n] * 5))
    assert st == -6 and "16384" in err
    _ok(plan(**dict(c, max_offset_samples=16384)))
    # b2_sync_tracks_gss always searches: a null gss_ratio is checked after the envelope and the other outputs
    assert _status(**dict(c, gss_ratio=0)) == (-1, "sync_tracks_gss: null gss_ratio")
    assert _status(**dict(c, gss_ratio=0, outputs=0)) == (-1, "sync_tracks_gss: null output")
    assert _status(**dict(c, gss_ratio=0, max_offset_samples=16385))[0] == -6
    assert _status(**dict(c, gss_ratio=0, max_offset_samples=16385, track_video=[], cue_off=[0]))[0] == -6
    assert _status(**dict(c, gss_ratio=0, track_video=[], cue_off=[0]))[0] == 0
    # the cue times are checked at the search interval's upper end too
    ends = c["cue_end"].copy()
    ends[7] = 9007199254.740992 / 1.05
    st, err = _status(**dict(c, cue_end=ends))
    assert st == -1 and "at ratio 1.1: cue end time" in err and "index 7" in err
    assert _ok(plan(**dict(c, gss=0, cue_end=ends)))
