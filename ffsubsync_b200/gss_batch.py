"""Batched golden-section search over the framerate ratio (the reference's ``--gss`` mode).

Per pair the reference runs ``gss(opt_func, 0.9, 1.1)`` (ffsubsync/aligners.py:111-129,
ffsubsync/golden_section_search.py:15-74): 17 strictly sequential evaluations of
``-score(ratio)``, each one = SubtitleScaler(ratio) + SubtitleSpeechTransformer + FFTAligner, and
only the LAST evaluation is recorded as the candidate.  The sequence of ratios depends on the
scores, so the 17 rounds stay sequential - but every round is one rasterise + one align launch
for ALL pairs (per-pair ratios), with the reference signals resident on the device.

The interval bookkeeping below is the reference's, vectorised over pairs with numpy; it yields
bit-identical ratios (same float64 operations in the same order).
"""
import math
from typing import NamedTuple, Optional

import numpy as np

from . import _native
from .aligners import MAX_FRAMERATE_RATIO, MIN_FRAMERATE_RATIO
from .golden_section_search import invphi, invphi2


class GssResult(NamedTuple):
    score: np.ndarray      # float64[B]  score of the last evaluation
    offset: np.ndarray     # int32[B]
    ratio: np.ndarray      # float64[B]  ratio of the last evaluation
    evals: np.ndarray      # float64[B, n_evals]  every ratio evaluated, in order
    status: np.ndarray     # int32[B]   B2_ALIGN_* flags of the last evaluation


def gss_align_batch(ref, ref_off, cue_start, cue_end, cue_off, cue_keep=None,
                    max_offset_samples: Optional[int] = None, sample_rate: int = 100,
                    start_seconds: float = 0.0, lo: float = MIN_FRAMERATE_RATIO,
                    hi: float = MAX_FRAMERATE_RATIO, tol: float = 1e-4, handle=None) -> GssResult:
    """ref: float32 reference speech signals of B pairs back to back - a numpy array (uploaded once)
    or a CUDA torch tensor; ref_off: [B+1].  Cues as in ``BatchSynchronizer`` (host arrays)."""
    import torch

    handle = handle or _native.get_handle()
    ref_off = np.ascontiguousarray(ref_off, dtype=np.int64)
    cue_off = np.ascontiguousarray(cue_off, dtype=np.int64)
    B = len(ref_off) - 1
    if isinstance(ref, np.ndarray):
        ref = torch.from_numpy(np.ascontiguousarray(ref, dtype=np.float32)).cuda()
    dev = ref.device
    score_d = torch.empty(2 * B, dtype=torch.float64, device=dev)
    offset_d = torch.empty(2 * B, dtype=torch.int32, device=dev)
    status_d = torch.empty(2 * B, dtype=torch.int32, device=dev)

    def evaluate(ratios: np.ndarray):
        """ratios: float64[B, k] (k = 1 or 2) -> (scores[B, k], offsets[B, k], status[B, k])"""
        k = ratios.shape[1]
        flat = np.ascontiguousarray(ratios.reshape(-1))
        lengths = handle.rasterize_lengths(cue_end, cue_off, flat, k, True, sample_rate)
        sub_off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
        sub = torch.empty(int(sub_off[-1]), dtype=torch.float32, device=dev)
        handle.rasterize(cue_start, cue_end, cue_keep, cue_off, flat, k, True, sample_rate, start_seconds,
                         out=sub.data_ptr(), out_off=sub_off, memspace=_native.B2_DEVICE)
        handle.align_batch(ref.data_ptr(), ref_off, sub.data_ptr(), sub_off, B, k, max_offset_samples,
                           score=score_d.data_ptr(), offset=offset_d.data_ptr(), status=status_d.data_ptr(),
                           memspace=_native.B2_DEVICE)
        handle.synchronize()
        n = B * k
        return (score_d[:n].cpu().numpy().reshape(B, k).copy(), offset_d[:n].cpu().numpy().reshape(B, k).copy(),
                status_d[:n].cpu().numpy().reshape(B, k).copy())

    # ---- golden_section_search.gss, one lane per pair ------------------------------------------
    a = np.full(B, min(lo, hi), dtype=np.float64)
    b = np.full(B, max(lo, hi), dtype=np.float64)
    h = b - a
    if B == 0 or h[0] <= tol:
        z = np.zeros(B)
        return GssResult(z, z.astype(np.int32), a, np.zeros((B, 0)), z.astype(np.int32))
    n = int(math.ceil(math.log(tol / h[0]) / math.log(invphi)))
    c = a + invphi2 * h
    d = a + invphi * h
    evals = [c.copy(), d.copy()]
    s, o, st = evaluate(np.stack([c, d], axis=1))
    yc, yd = -s[:, 0], -s[:, 1]
    last = (s[:, 1].copy(), o[:, 1].copy(), d.copy(), st[:, 1].copy())   # n == 1: both flagged, d is appended last
    for k in range(n - 1):
        left = yc < yd                      # shrink towards a: new point c
        h = invphi * h
        b = np.where(left, d, b)
        a_new = np.where(left, a, c)
        d_l, yd_l = c, yc                   # left branch:  d <- c, yd <- yc, c <- a + invphi2*h
        c_r, yc_r = d, yd                   # right branch: c <- d, yc <- yd, d <- a + invphi*h
        a = a_new
        new_c = a + invphi2 * h
        new_d = a + invphi * h
        x = np.where(left, new_c, new_d)    # the one new evaluation of this iteration, per pair
        evals.append(x.copy())
        s, o, st = evaluate(x[:, None])
        y = -s[:, 0]
        c = np.where(left, new_c, c_r)
        d = np.where(left, d_l, new_d)
        yc = np.where(left, y, yc_r)
        yd = np.where(left, yd_l, y)
        if k == n - 2:
            last = (s[:, 0].copy(), o[:, 0].copy(), x.copy(), st[:, 0].copy())
    return GssResult(last[0], last[1].astype(np.int32), last[2], np.stack(evals, axis=1), last[3].astype(np.int32))


def combine_gss(best_score, best_offset, best_k, gss: GssResult, K: int, max_offset_samples: Optional[int],
                all_score=None, all_offset=None):
    """MaxScoreAligner.transform (ffsubsync/aligners.py:154-167) over the candidates [grid, GSS] of every
    track, given the grid's reduced result (b2_sync_tracks) and the search's last evaluation: the GSS candidate
    is number K, last in list order, so it wins only with a strictly higher score; it goes through the same
    |offset| filter, and a track whose reference is empty (status B2_ALIGN_EMPTY) keeps the grid's answer
    and gets ratio NaN.  all_*: the grid's [T*K] per-ratio results, returned as [T*(K+1)] with column K the
    candidate.  Returns (best_score, best_offset, best_k, gss_ratio, all_score, all_offset) as numpy arrays."""
    bs = np.array(best_score, dtype=np.float64)
    bo = np.array(best_offset, dtype=np.int32)
    bk = np.array(best_k, dtype=np.int32)
    T = len(bk)
    live = (np.asarray(gss.status) & _native.ALIGN_EMPTY) == 0
    ok = live if max_offset_samples is None else live & (np.abs(gss.offset.astype(np.int64)) <= max_offset_samples)
    win = ok & ((bk < 0) | (gss.score > bs))
    bs[win], bo[win], bk[win] = gss.score[win], gss.offset[win], K
    ratio = np.where(live, gss.ratio, np.nan)
    a_s = a_o = None
    if all_score is not None:
        a_s = np.concatenate([np.asarray(all_score, np.float64).reshape(T, K), gss.score[:, None]], axis=1).reshape(-1)
    if all_offset is not None:
        a_o = np.concatenate([np.asarray(all_offset, np.int32).reshape(T, K),
                              gss.offset.astype(np.int32)[:, None]], axis=1).reshape(-1)
    return bs, bo, bk, ratio, a_s, a_o
