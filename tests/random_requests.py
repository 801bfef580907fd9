"""Seeded random requests of the batched sync calls, shared by tests/test_plan_random_cpu.py (the host planner through
plan_emul) and tests/test_gpu_random_requests.py (every output of a call against the composed oracles).

draw(seed) picks one request with every field drawn on its own and weighted towards the edges the planner cuts at:
lengths around window multiples, shorter than one window, across the 100 s chunk edge and empty; videos without
tracks at either end and in a row; tracks without cues, with every cue past the reference and with keep masks; K of
1, 2, 5 and 7; one-offset windows; both memspaces; B2_SUBBATCHES of 1, 2, 3 and 5 with the aligner, reference format,
raster and VAD knobs.  On about one seed in eight (one in two on the split tiled knob set) max_offset_samples is
N - S for a job whose padded length N is at least 2 S + 1: the reference's mask then wraps and leaves that job a
one-offset window.  The request holds no PCM: test_gpu_random_requests makes it from the seed."""
import numpy as np

from oracle import aligner_oracle as ao
from oracle import pgs_oracle as po
from oracle import raster_oracle as ro
from oracle import segment_oracle as so
from oracle import vad_oracle as vo

ENTRIES = ["batch", "tracks", "gss", "auditok", "subs", "pgs", "sig", "seg"]
# the kinds of reference each entry point takes
KINDS = {"batch": ["audio"], "tracks": ["audio"], "gss": ["audio"], "auditok": ["audio"],
         "subs": ["audio", "subs"], "pgs": ["audio", "subs", "pgs"], "sig": ["audio", "subs", "pgs", "sig"],
         "seg": ["audio", "subs", "pgs", "sig", "seg"]}
# every B2_SUBBATCHES value beside an aligner path, the reference format, the raster, the split and the VAD layout
KNOBS = [
    dict(B2_SUBBATCHES="1"),
    dict(B2_SUBBATCHES="2", B2_ALIGN_PATH="runs"),
    dict(B2_SUBBATCHES="3", B2_ALIGN_PATH="tiled", B2_REF_PACKED="0"),
    dict(B2_SUBBATCHES="5", B2_ALIGN_PATH="big", B2_BIG_WS_MB="64"),
    dict(B2_SUBBATCHES="2", B2_ALIGN_PATH="tiled", B2_ALIGN_SPLIT="5", B2_FUSED_RASTER="0"),
    dict(B2_SUBBATCHES="3", B2_VAD_LAYOUT="group", B2_ALIGN_SPLIT="1"),
    dict(B2_SUBBATCHES="5", B2_VAD_SMS="8", B2_ALIGN_PATH="runs"),
]
RATES = [8000, 16000, 48000]
# ratios of the bench grid (levels 1 and float32(1 / r)) and two below level 1 that a power of two holds exactly
RATIOS = [1.0, 24 / 23.976, 25 / 23.976, 25 / 24.0, 23.976 / 24, 23.976 / 25, 24 / 25.0, 2.0, 4.0]
# non_speech_label values whose levels keep every score a float64-exact sum (no 0.3: its scores round)
LABELS = [0.0, 1.0, -0.5]
MOS_NONE = None
SR = 100                                       # frames per second of every signal
GSS_MAX_MOS = 16384                            # the search's envelope: windows of at most 2 * 16384 offsets
WHO = {"batch": "sync_batch", "tracks": "sync_tracks", "gss": "sync_tracks_gss", "auditok": "sync_tracks_auditok",
       "subs": "sync_tracks_subs", "pgs": "sync_tracks_pgs", "sig": "sync_tracks_sig", "seg": "sync_tracks_seg"}
INT64_MIN = -(1 << 63)


def chunk_samples(fr):
    """The reference's read: (2 fr // 100) * 5000 samples, 100 s."""
    return (2 * fr // 100) * 5000


def _pick(rng, xs, p=None):
    return xs[int(rng.choice(len(xs), p=p))]


def _length(rng, fr, allow_zero=True):
    """Samples of one audio video: around window multiples, sub-window, around the 100 s chunk edge, or empty."""
    fpw = fr // SR
    kind = rng.randint(8)
    if kind == 0 and allow_zero:
        return 0
    if kind <= 1:
        return int(rng.randint(1, fpw))                                 # shorter than one window
    if kind == 2:                                                       # across the 100 s chunk edge
        return chunk_samples(fr) + int(rng.choice([-fpw - 1, -fpw, -1, 0, 1, fpw, fpw + 1, 7 * fpw + 3]))
    w = int(rng.choice([1, 2, 31, 32, 33, 500, 3000, 6000]) if kind < 6 else rng.randint(2, 9000))
    return max(1, w * fpw + int(rng.choice([-fpw, -1, 0, 1, fpw, fpw // 2])))


def _cues(rng, dur, seed):
    """One track's cue list and keep mask: a synthetic list shifted by a few seconds, none, or all past the end."""
    kind = rng.randint(10)
    if kind == 0:
        return np.zeros(0), np.zeros(0)
    st, en = ro.synthetic_cues(seed, max(dur, 12.0) + rng.uniform(-5, 5))
    if kind == 1:                                                       # every cue past the reference
        off = dur + rng.uniform(1, 20)
        return np.round(st[:8] + off, 3), np.round(en[:8] + off, 3)
    d = rng.randint(-300, 300) / 100.0
    ok = st + d >= 0
    return np.round(st[ok] + d, 3), np.round(en[ok] + d, 3)


def _tracks_per_video(rng, V, entry):
    if entry == "batch":
        return [1] * V
    per = rng.randint(0, 5, V)
    if rng.rand() < 0.7:                                               # zero-track videos at the ends and in a row
        for v in {0, V - 1, V // 2, min(V - 1, V // 2 + 1)}:
            if rng.rand() < 0.6:
                per[v] = 0
    if per.sum() == 0:
        per[rng.randint(V)] = 1
    return [int(x) for x in per]


def window(req):
    """Samples per detector window: int(fr / sr + 0.5) for energy / ZCR, fr // sr for auditok's blocks."""
    return req["fr"] // SR if req["detector"] == "auditok" else vo.frames_per_window(req["fr"], SR)


def detector_call(req, n):
    """Samples per detector call over an audio video of n samples: auditok's chunk_samples (0: one call), energy /
    ZCR's 100 s read where that is not a whole number of windows (one call elsewhere: the frames are the same)."""
    if req["detector"] == "auditok":
        return req["chunk"] if req["chunk"] > 0 else max(n, 1)
    call = chunk_samples(req["fr"])
    return call if call % window(req) else max(n, 1)


def ref_length(req, d):
    """The reference length of video d by its kind's oracle (the detector's chunk loop for audio)."""
    if d["kind"] == "audio":
        n, step, w = d["n"], detector_call(req, d["n"]), window(req)
        return sum(-(-min(step, n - i) // w) for i in range(0, n, step))
    if d["kind"] == "subs":
        return len(ro.rasterize(d["starts"], d["ends"], None, SR, 0.0, 1.0)[0])
    if d["kind"] == "pgs":
        return po.pgs_length(max(d["ends"]), SR)
    if d["kind"] == "sig":
        return len(d["x"])
    return so.length(d["total"], SR)


def _one_offset_mos(req):
    """max_offset_samples N - S of the first job (track, ratio) with N >= 2 S + 1, or None: the mask's wrap leaves
    that job the single offset -S (aligner_oracle.surviving_index_range)."""
    for t in req["tracks"]:
        R = ref_length(req, req["videos"][t["video"]])
        for r in req["ratios"]:
            S = len(ro.rasterize(t["starts"], t["ends"], None, SR, 0.0, r)[0])
            N = ao.padded_length(R, S)
            if R > 0 and N >= 2 * S + 1 and (req["entry"] != "gss" or N - S <= GSS_MAX_MOS):
                return N - S
    return None


def draw(seed, rates=RATES):
    """One request (a dict) for seed: entry point, videos, tracks, grid, window, label, memspace and knob set.  rates:
    the frame rates to draw from."""
    rng = np.random.RandomState(seed)
    entry = ENTRIES[seed % len(ENTRIES)] if seed < 2 * len(ENTRIES) else _pick(rng, ENTRIES)
    fr = _pick(rng, rates)
    fpw = fr // SR
    V = int(rng.choice([1, 2, 3, 5, 8, 13, 40], p=[0.1, 0.15, 0.2, 0.2, 0.15, 0.12, 0.08]))
    big = V >= 13
    kinds = KINDS[entry]
    videos = []
    for v in range(V):
        kind = _pick(rng, kinds)
        d = dict(kind=kind)
        if kind == "audio" or kind == "seg":
            n = _length(rng, fr)
            if big:   # many videos: keep the call small
                n = min(n, int(rng.randint(1, 40)) * 100 * fpw + int(rng.randint(0, fpw)))
            d["n"] = n
        dur = d["n"] / fr if "n" in d else rng.uniform(5, 150)
        if kind == "subs":
            st, en = ro.synthetic_cues(seed * 100 + v, dur) if rng.rand() < 0.85 else (np.zeros(0), np.zeros(0))
            d.update(starts=st, ends=en, keep=(rng.rand(len(st)) < 0.8).astype(np.uint8))
        elif kind == "pgs":
            st, en = ro.synthetic_cues(seed * 100 + v + 50, dur)
            if len(st) == 0:
                st, en = np.array([1.0]), np.array([2.5])
            d.update(starts=st + 0.004, ends=en + 0.006)
        elif kind == "sig":
            n = int(rng.choice([0, 1, 31, 32, 33, int(dur * SR)]))
            d["x"] = rng.choice([0.0, 0.25, 1.0], n).astype(np.float64)
        elif kind == "seg":
            total = d["n"] / fr
            starts = sorted(set(int(s) for s in rng.randint(0, int(total) + 3, rng.randint(0, 4))))
            lo = [min(d["n"], s * fr) for s in starts]
            hi = [min(d["n"], a + int(rng.choice([1, 10, 30])) * fr) for a in lo]
            d.update(total=total, starts=starts, lo=lo, hi=hi)
        d["dur"] = dur
        videos.append(d)
    per = _tracks_per_video(rng, V, entry)
    tracks = []
    for v, m in enumerate(per):
        for i in range(m):
            st, en = _cues(rng, videos[v]["dur"], seed * 1000 + 7 * v + i)
            tracks.append(dict(video=v, starts=st, ends=en))
    K = int(rng.choice([1, 2, 5, 7]))
    ratios = [1.0] if K == 1 and rng.rand() < 0.5 else [float(_pick(rng, RATIOS)) for _ in range(K)]
    gss = entry == "gss"
    mos = _pick(rng, [MOS_NONE, 0, 1, 6000, 10 ** 6])
    if gss:
        mos = _pick(rng, [0, 1, 6000, GSS_MAX_MOS])
    label = 0.0 if gss else float(_pick(rng, LABELS))
    req = dict(seed=seed, entry=entry, fr=fr, videos=videos, tracks=tracks, ratios=ratios, mos=mos, label=label,
               memspace=_pick(rng, ["host", "device"]), knobs=KNOBS[rng.randint(len(KNOBS))],
               detector="auditok" if entry == "auditok" or (entry in ("subs", "pgs", "sig", "seg") and rng.rand() < 0.3)
               else "energy_zcr",
               chunk=_pick(rng, [0, chunk_samples(fr), 333 * fpw + 7]), keep_tracks=rng.rand() < 0.4,
               keep_seed=seed + 17)
    if rng.rand() < (0.5 if "B2_ALIGN_SPLIT" in req["knobs"] and req["knobs"].get("B2_ALIGN_PATH") == "tiled" else 0.12):
        one = _one_offset_mos(req)
        req["mos"] = req["mos"] if one is None else one
    return req


def plan_request(req, a):
    """The plan_emul fields (tests/sync_plan.py) of request req, host tables a = arrays(req)."""
    e = req["entry"]
    p = dict(who=WHO[e], pcm_off=a["pcm_off"], cue_start=a["cue_start"], cue_end=a["cue_end"], cue_off=a["cue_off"],
             ratios=req["ratios"], frame_rate=req["fr"], sample_rate=SR, label=req["label"],
             auditok_label=req["label"], energy_threshold=100000, chunk_samples=req["chunk"], all=1,
             detector=int(req["detector"] == "auditok"), gss=int(e == "gss"),
             max_offset_samples=INT64_MIN if req["mos"] is None else req["mos"],
             subbatches=req["knobs"]["B2_SUBBATCHES"], vad_sms=req["knobs"].get("B2_VAD_SMS"))
    if e != "batch":
        p["track_video"] = a["track_video"]
    for k in ("ref_is_subs", "ref_cue_start", "ref_cue_end", "ref_cue_off", "ref_is_pgs", "pgs_start", "pgs_end",
              "pgs_off", "ref_is_sig", "sig_off", "seg_video", "seg_total", "seg_off", "seg_start", "seg_lo", "seg_hi"):
        if a.get(k) is not None:
            p[k] = a[k]
    return p


def arrays(req):
    """The call's host tables of request req (no PCM): pcm_off, track_video, cue arrays (cue_keep or None) and every
    reference table, with None where the entry point has no such argument."""
    vids, trk = req["videos"], req["tracks"]
    V = len(vids)
    n = [d.get("n", 0) if d["kind"] in ("audio", "seg") else 0 for d in vids]
    cat = lambda xs, dt: np.concatenate([np.asarray(x, dt) for x in xs]).astype(dt) if xs else np.zeros(0, dt)  # noqa
    off = lambda xs: np.concatenate([[0], np.cumsum([len(x) for x in xs])]).astype(np.int64)  # noqa: E731
    cs, ce = [t["starts"] for t in trk], [t["ends"] for t in trk]
    a = dict(pcm_off=off([np.zeros(k) for k in n]), track_video=np.array([t["video"] for t in trk], np.int32),
             cue_start=cat(cs, np.float64), cue_end=cat(ce, np.float64), cue_off=off(cs))
    nc = int(a["cue_off"][-1])
    a["cue_keep"] = (np.random.RandomState(req["keep_seed"]).rand(nc) < 0.85).astype(np.uint8) \
        if req["keep_tracks"] else None
    kinds = KINDS[req["entry"]]
    sel = lambda k, key: [d[key] if d["kind"] == k else [] for d in vids]   # noqa: E731
    if "subs" in kinds:
        a.update(ref_is_subs=np.array([d["kind"] == "subs" for d in vids], np.uint8),
                 ref_cue_start=cat(sel("subs", "starts"), np.float64), ref_cue_end=cat(sel("subs", "ends"), np.float64),
                 ref_cue_keep=cat(sel("subs", "keep"), np.uint8), ref_cue_off=off(sel("subs", "starts")))
    if "pgs" in kinds:
        a.update(ref_is_pgs=np.array([d["kind"] == "pgs" for d in vids], np.uint8),
                 pgs_start=cat(sel("pgs", "starts"), np.float64), pgs_end=cat(sel("pgs", "ends"), np.float64),
                 pgs_off=off(sel("pgs", "starts")))
    if "sig" in kinds:
        a.update(ref_is_sig=np.array([d["kind"] == "sig" for d in vids], np.uint8), x=cat(sel("sig", "x"), np.float64),
                 sig_off=off(sel("sig", "x")))
    if "seg" in kinds:
        sv = [v for v in range(V) if vids[v]["kind"] == "seg"]
        a.update(seg_video=np.array(sv, np.int32), seg_total=np.array([vids[v]["total"] for v in sv], np.float64),
                 seg_off=off([vids[v]["starts"] for v in sv]),
                 seg_start=cat([vids[v]["starts"] for v in sv], np.int64),
                 seg_lo=cat([vids[v]["lo"] for v in sv], np.int64), seg_hi=cat([vids[v]["hi"] for v in sv], np.int64))
    return a


def summary(req):
    """One line per request: what a failure report prints so that the seed replays it."""
    kinds = "".join(d["kind"][0] for d in req["videos"])
    per = np.bincount([t["video"] for t in req["tracks"]], minlength=len(req["videos"])).tolist()
    return ("seed=%d entry=%s fr=%d V=%d kinds=%s tracks=%s lens=%s K=%d ratios=%s mos=%s label=%s det=%s chunk=%d "
            "memspace=%s knobs=%s keep=%s" % (
                req["seed"], req["entry"], req["fr"], len(req["videos"]), kinds, per,
                [d.get("n", -1) for d in req["videos"]], len(req["ratios"]), ["%.5g" % r for r in req["ratios"]],
                req["mos"], req["label"], req["detector"], req["chunk"], req["memspace"], req["knobs"],
                req["keep_tracks"]))
