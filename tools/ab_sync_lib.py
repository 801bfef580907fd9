"""A/B check of two builds of the library on the batched sync calls: every output bit for bit and the number of
kernel launches of every call must agree.

    python tools/ab_sync_lib.py OLD.so [NEW.so]      (NEW defaults to the tree's ffsubsync_b200/_lib build)

Runs the seeded corpora of tests/test_gpu_subs_ref.py (subtitle and audio references mixed, several tracks per
video) and a one-track-per-video corpus through b2_sync_batch, b2_sync_tracks, b2_sync_tracks_gss,
b2_sync_tracks_auditok (grid and search) and b2_sync_tracks_subs (both detectors, grid and search), on B2_HOST,
B2_DEVICE and two chained B2_DEVICE_RESIDENT calls, under B2_SUBBATCHES=1 and 3 and fused and unfused raster.
Needs an H100.  Prints one line per configuration and exits non-zero on the first difference."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "golden")]

import torch  # noqa: E402

from ffsubsync_b200 import _native  # noqa: E402
from test_gpu_subs_ref import _corpus  # noqa: E402

GRID = [1.0, 24 / 23.976, 25 / 24.0, 23.976 / 24, 24 / 25.0]
MOS, THR, FR = 6000, 100000, 16000
CHUNK = (2 * FR // 100) * 5000


def handle_for(path):
    _native._lib, _native.LIB_PATH = None, path
    h = _native.Handle(0)
    _native._lib = None
    return h


def corpora():
    mixed = _corpus([(60.0 + 7 * (v % 5), v % 4 == 1, [(GRID[(v + i) % 5], 37 * v - 11 * i) for i in range(1 + v % 3)])
                     for v in range(40)], FR, seed0=5)
    pairs = _corpus([(70.0 + 3 * (v % 7), False, [(GRID[v % 5], 23 * v - 300)]) for v in range(36)], FR, seed0=9)
    return mixed, pairs


def calls(c):
    """(name, method, positional args, keyword args) of every call kind on corpus c."""
    tv, common = c["track_video"], (c["cue_start"], c["cue_end"], None, c["cue_off"], GRID, 0.0, MOS)
    energy = (FR, 100, 0.0, THR, -1, -1)
    out = []
    if len(tv) == len(c["pcm_off"]) - 1 and not c["is_subs"].any():
        out.append(("sync_batch", "sync_batch", (c["pcm_off"],) + energy + common, {}))
    if not c["is_subs"].any():
        out += [("sync_tracks", "sync_tracks", (c["pcm_off"], tv) + energy + common, {}),
                ("sync_tracks_gss", "sync_tracks_gss", (c["pcm_off"], tv) + energy + common, dict(want_evals=True)),
                ("auditok", "sync_tracks_auditok", (c["pcm_off"], tv, FR, 100, 0.0) + common + (CHUNK,), {}),
                ("auditok_search", "sync_tracks_auditok", (c["pcm_off"], tv, FR, 100, 0.0) + common + (CHUNK,),
                 dict(gss=True, want_evals=True))]
    refs = (c["is_subs"], c["ref_start"], c["ref_end"], c["ref_keep"], c["ref_off"])
    for det in (_native.B2_DETECTOR_ENERGY_ZCR, _native.B2_DETECTOR_AUDITOK):
        for gss in (False, True):
            out.append(("subs_%d%s" % (det, "_search" if gss else ""), "sync_tracks_subs",
                        (c["pcm_off"], tv, FR, 100, 0.0) + refs + common,
                        dict(detector=det, energy_threshold=THR, chunk_samples=CHUNK, gss=gss, want_evals=gss)))
    return out


def run(h, c, name, method, args, kw, memspace):
    """One call (two chained calls for B2_DEVICE_RESIDENT); returns (outputs as bytes, launch count delta)."""
    T, K = len(c["track_video"]), len(GRID)
    gss = name.endswith("gss") or kw.get("gss", False)
    cols = K + 1 if gss else K
    n0 = h.launch_count
    if memspace == _native.B2_HOST:
        r = getattr(h, method)(c["pcm"], *args, want_all=True, memspace=memspace, **kw)
        res = [np.asarray(x).tobytes() for x in r if x is not None]
        return res, h.launch_count - n0
    dev = torch.device("cuda", 0)
    pcm = torch.from_numpy(c["pcm"]).to(dev) if len(c["pcm"]) else None
    res = []
    for _ in range(2 if memspace == _native.B2_DEVICE_RESIDENT else 1):
        o = dict(best_score=torch.full((T,), -7.0, dtype=torch.float64, device=dev),
                 best_offset=torch.full((T,), -7, dtype=torch.int32, device=dev),
                 best_k=torch.full((T,), -7, dtype=torch.int32, device=dev),
                 all_score=torch.full((T * cols,), -7.0, dtype=torch.float64, device=dev),
                 all_offset=torch.full((T * cols,), -7, dtype=torch.int32, device=dev))
        if gss:
            o.update(gss_ratio=torch.full((T,), -7.0, dtype=torch.float64, device=dev),
                     gss_evals=torch.full((T * _native.GSS_EVALS,), -7.0, dtype=torch.float64, device=dev))
        kw2 = {k: v for k, v in kw.items() if k != "want_evals"}
        torch.cuda.synchronize()
        getattr(h, method)(pcm.data_ptr() if pcm is not None else None, *args, memspace=memspace,
                           **{k: v.data_ptr() for k, v in o.items()}, **kw2)
        h.synchronize()
        res += [v.cpu().numpy().tobytes() for v in o.values()]
    return res, h.launch_count - n0


def main():
    old_path = sys.argv[1]
    new_path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "ffsubsync_b200", "_lib", "libffsubsync_b200.so")
    ha, hb = handle_for(old_path), handle_for(new_path)
    n_calls = 0
    for c in corpora():
        for sub in ("1", "3"):
            for fused in ("1", "0"):
                os.environ["B2_SUBBATCHES"], os.environ["B2_FUSED_RASTER"] = sub, fused
                for name, method, args, kw in calls(c):
                    for ms in (_native.B2_HOST, _native.B2_DEVICE, _native.B2_DEVICE_RESIDENT):
                        ra, la = run(ha, c, name, method, args, kw, ms)
                        rb, lb = run(hb, c, name, method, args, kw, ms)
                        where = "%s memspace=%d B2_SUBBATCHES=%s B2_FUSED_RASTER=%s" % (name, ms, sub, fused)
                        if la != lb:
                            sys.exit("launch counts differ: %d vs %d (%s)" % (la, lb, where))
                        if len(ra) != len(rb) or any(x != y for x, y in zip(ra, rb)):
                            sys.exit("outputs differ (%s)" % where)
                        n_calls += 1
                print("ab: T=%d B2_SUBBATCHES=%s B2_FUSED_RASTER=%s: %d call kinds equal"
                      % (len(c["track_video"]), sub, fused, len(calls(c))), flush=True)
    print("ab ok: %d configurations, every output and launch count equal" % n_calls)


if __name__ == "__main__":
    main()
