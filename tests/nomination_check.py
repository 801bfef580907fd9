"""The aligner's nomination stage of one call, checked against a float64 correlation at every offset.

Shared by tests/test_gpu_nomination.py and tests/test_gpu_bigfft_roundoff.py.  b2_capture_nominations exposes the
fp32 window, (maximum, tau) and the candidate count of every (pair, ratio) job; check_jobs compares them with the
exact correlation of the signals the kernels were given (DESIGN.md section 4, "Round-off bound")."""
import numpy as np
import scipy.fft

from oracle import aligner_oracle as ao

K_CAND = 32
U = 2.0 ** -24


class Exact:
    """float64 correlation of a (ref, sub) pair, computed once per pair of signals.  full[o mod N] =
    sum_j s'[j] r'[j + o] with x' = 2 x - 1 and N = ao.padded_length(R, S): the sequence oracle/aligner_oracle
    .correlation calls ``convolve``, read at index N - 1 - S - o, computed with real transforms."""

    def __init__(self):
        self.memo = {}
        self.spec = {}

    def _full(self, ref, sub):
        key = (id(ref), id(sub))
        if key not in self.memo:
            N = ao.padded_length(len(ref), len(sub))
            rk = (id(ref), N)
            if rk not in self.spec:   # the reference spectrum is shared by the ratios / subtitles of a pair
                self.spec[rk] = (scipy.fft.rfft(2.0 * np.asarray(ref, np.float64) - 1.0, N, workers=-1), ref)
            s = scipy.fft.rfft(2.0 * np.asarray(sub, np.float64) - 1.0, N, workers=-1)
            full = scipy.fft.irfft(np.conj(s) * self.spec[rk][0], N, workers=-1)
            if binary(ref) and binary(sub):
                full = np.round(full)          # +-1 products: the exact scores are integers
            self.memo[key] = (full, float(np.sqrt(np.sum(full * full))), ref, sub)   # arrays kept alive: ids are keys
        return self.memo[key]

    def window(self, ref, sub, w0, n):
        full = self._full(ref, sub)[0]
        o = w0 + np.arange(n)
        # aligners.py:47; offsets where the signals do not overlap score exactly 0 (no FFT round-off)
        return np.where((o > -len(sub)) & (o < len(ref)), full[o % len(full)], 0.0)

    def tau(self, ref, sub):
        """The bound the kernels evaluate in fp32, in float64: u (512 sqrt(Es Er) + 192 ||c||_2), the energies of
        2 x - 1 over each signal, ||c||_2 over the whole N-length output of the exact correlation."""
        es = float(np.sum((2.0 * np.asarray(sub, np.float64) - 1.0) ** 2))
        er = float(np.sum((2.0 * np.asarray(ref, np.float64) - 1.0) ** 2))
        return U * (512.0 * np.sqrt(es * er) + 192.0 * self._full(ref, sub)[1])


def binary(x):
    return bool(np.all((x == 0) | (x == 1)))


def norm(x):
    return float(np.sqrt(np.sum((2.0 * np.asarray(x, np.float64) - 1.0) ** 2)))


def check_jobs(cap, sigs, mos, exact, key, worst=None, out=None, winner_only=False, K=1):
    """sigs[j] = (ref, sub) float64 arrays of global job j as the kernels saw them; out = (score, offset,
    status) per job (None in winner-only calls).  Records the worst max |fp32 - exact| / tau under worst[key].
    Returns per job (fp32 maximum, tau, (w0, n, fp32 scores) or None, max |fp32 - exact| or None)."""
    stats = []
    for j, (ref, sub) in enumerate(sigs):
        w0, n = (int(v) for v in cap["win"][j])
        mx, tau = (np.float32(v) for v in cap["stat"][j])
        cand = int(cap["cand"][j])
        o_lo, o_hi = ao.offset_range(len(ref), len(sub), mos)
        where = (key, j, len(ref), len(sub), mos)
        if o_lo > o_hi:
            assert n == 0 and cand == 0 and mx == -np.inf, where
            stats.append((mx, tau, None, None))
            continue
        assert (w0, n) == (o_lo, o_hi - o_lo + 1), where
        f = cap["scores"][j, :n]
        assert mx == f.max(), where
        ex = exact.window(ref, sub, w0, n)
        err = float(np.abs(f.astype(np.float64) - ex).max())
        assert err <= float(tau), (where, err, float(tau))
        if worst is not None:
            worst[key] = max(worst.get(key, (0.0,)), (err / float(tau), "N=%d" % ao.padded_length(len(ref), len(sub)),
                                                      "R=%d S=%d" % (len(ref), len(sub)), "mos=%s" % mos))
        cut = np.float32(mx - tau)           # float32 subtraction, as the selection kernels do
        hits = np.flatnonzero(f >= cut)
        if cand != -1:
            assert cand == len(hits), (where, cand, len(hits))
        if out is not None:
            score, offset, status = (None if a is None else a[j] for a in out)
            assert cand != -1, where
            if status is not None:           # b2_sync_batch does not return the per-ratio status
                assert bool(status & 4) == (cand > K_CAND), (where, status, cand)
            top = hits[::-1][:K_CAND]        # largest offsets first
            best = ex[top].max()
            m = int(offset) - w0
            assert m in set(top.tolist()), (where, int(offset))
            tol = 1e-9 * (norm(ref) * norm(sub) + 1.0)
            assert ex[m] >= best - tol and abs(float(score) - ex[m]) <= tol, (where, float(score), ex[m], best)
            if binary(ref) and binary(sub):   # integer scores: the tie rule is checkable exactly
                assert m == int(top[np.flatnonzero(ex[top] == best)[0]]), where
        stats.append((mx, tau, (w0, n, f), err))
    if winner_only:
        _check_approx(cap, stats, mos, K, key)
    return stats


def _check_approx(cap, stats, mos, K, key):
    """Winner-only pruning: cand == -1 exactly when max + tau < max_k (max_k - tau_k) and no surviving
    offset of the pair exceeds the mask width (no_prune)."""
    for b in range(len(stats) // K):
        js = range(b * K, b * K + K)
        floor = max(np.float32(stats[j][0] - stats[j][1]) for j in js)
        no_prune = mos is not None and any(
            stats[j][2] is not None and max(abs(stats[j][2][0]), abs(stats[j][2][0] + stats[j][2][1] - 1)) > mos
            for j in js)
        for j in js:
            mx, tau, w, _ = stats[j]
            if w is None:
                continue
            want = (not no_prune) and np.float32(mx + tau) < floor
            assert (int(cap["cand"][j]) == -1) == want, (key, b, j, float(mx), float(tau), float(floor))
