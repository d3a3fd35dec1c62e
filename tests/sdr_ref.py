"""float64 numpy / scipy restatement of the BSS Eval v3 SDR of fsnplus_b200.metrics.sdr (DESIGN.md §3.21) for one source, written
from the published algorithm (Vincent, Gribonval and Févotte, "Performance measurement in blind audio source separation", 2006)
the way mir_eval's bss_eval_sources computes it: a 512-tap distortion filter, FFT correlations, a dense solve and an FFT
convolution.

For a reference r and an estimate e of N samples, zero-extended, and F = 512:
    R[k] = sum_n r[n] r[n + k],  D[k] = sum_n r[n] e[n + k]           (k = 0 .. 511)
    G c = D with G[i][j] = R[|i - j|]                                   (symmetric Toeplitz, positive definite for r != 0)
    P[n] = sum_k c[k] r[n - k]  (n = 0 .. N + 510),  e' = e followed by 511 zeros
    SDR = 10 log10(sum P^2 / sum (e' - P)^2)                            (+inf for a zero denominator)

Conventions pinned here and on the device: a silent reference or a silent estimate scores NaN (mir_eval raises there).  Scores above
100 dB (est = ref, or very short clips) measure rounding noise, and two correct restatements can differ there by many dB.

``sdr`` is the reference procedure; ``sdr_direct`` restates it with direct sums, a Levinson solve (``levinson``, the recursion the
device runs) and a direct convolution, and is the check that both are the same quantity.
"""
import numpy as np
from scipy.signal import fftconvolve

FLEN = 512
HIGH_DB = 100.0


def _inputs(ref, est):
    r = np.asarray(ref, np.float64).ravel()
    e = np.asarray(est, np.float64).ravel()
    if r.size != e.size or r.size == 0:
        raise ValueError(f"ref has {r.size} samples and est {e.size}; both must have the same, nonzero length")
    return r, e


def _score(P, e):
    ep = np.zeros(P.size)
    ep[:e.size] = e
    num, den = np.sum(P * P), np.sum((ep - P) ** 2)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(10 * np.log10(num / den)) if den > 0 else (float("inf") if num > 0 else float("nan"))


def sdr(ref, est):
    """SDR in dB of est against ref: FFT correlations, np.linalg.solve on the 512 x 512 Toeplitz matrix, fftconvolve."""
    r, e = _inputs(ref, est)
    if not r.any() or not e.any():
        return float("nan")
    n = r.size
    nfft = int(2 ** np.ceil(np.log2(n + FLEN - 1)))
    rf = np.fft.rfft(r, nfft)
    R = np.fft.irfft(rf * np.conj(rf), nfft)[:FLEN]
    D = np.fft.irfft(np.conj(rf) * np.fft.rfft(e, nfft), nfft)[:FLEN]
    idx = np.arange(FLEN)
    G = R[np.abs(idx[:, None] - idx[None, :])]
    c = np.linalg.solve(G, D)
    P = fftconvolve(c, r)[:n + FLEN - 1]
    return _score(P, e)


def correlations(r, e):
    """R[k] = sum_n r[n] r[n + k] and D[k] = sum_n r[n] e[n + k], k = 0 .. 511, by direct sums."""
    n = r.size
    R = np.zeros(FLEN)
    D = np.zeros(FLEN)
    for k in range(min(FLEN, n)):
        R[k] = np.dot(r[:n - k], r[k:])
        D[k] = np.dot(r[:n - k], e[k:])
    return R, D


def levinson(R, D):
    """Solve G c = D, G[i][j] = R[|i - j|], by Levinson's recursion: Durbin's prediction-error filter a (G_m a = E_m e_0) grown
    one order per step, and the solution x of the leading m x m system corrected by E_{m+1}^-1 (D_m - eps) times the reversed filter.
    Returns None where R[0] == 0 or a prediction error E_m becomes <= 0 or non-finite (a numerically singular reference)."""
    n = R.size
    if not R[0] > 0:
        return None
    a = np.zeros(n)
    a[0] = 1.0
    x = np.zeros(n)
    x[0] = D[0] / R[0]
    E = R[0]
    for m in range(1, n):
        rr = R[m:0:-1]                                   # R[m - j], j = 0 .. m - 1
        delta = np.dot(a[:m], rr)
        eps = np.dot(x[:m], rr)
        kappa = -delta / E
        a[:m + 1] = a[:m + 1] + kappa * a[m::-1]         # [a; 0] + kappa [0; reversed a]
        E = E + kappa * delta
        if not (E > 0 and np.isfinite(E)):
            return None
        x[:m + 1] += (D[m] - eps) / E * a[m::-1]
    return x


def sdr_direct(ref, est):
    """The same SDR from direct-sum correlations, ``levinson`` and a direct convolution."""
    r, e = _inputs(ref, est)
    if not r.any() or not e.any():
        return float("nan")
    R, D = correlations(r, e)
    c = levinson(R, D)
    if c is None:
        return float("nan")
    P = np.convolve(c, r)[:r.size + FLEN - 1]
    return _score(P, e)
