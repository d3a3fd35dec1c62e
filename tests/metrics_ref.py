"""float64 numpy / scipy restatement of the two metrics of fsnplus_b200.metrics (DESIGN.md §3.20), written from the published
algorithms: SI-SDR (Le Roux et al., "SDR - half-baked or well done?", 2019) and the classic STOI (Taal et al., 2011) with the
conventions of pystoi 0.3.3, which the reference's scorer calls as stoi(x, y, fs, extended=False).

Conventions pinned here (pystoi releases differ on them):
- every frame loop runs ``range(0, n - 256, 128)``: a signal of n samples has ceil((n - 256) / 128) frames when n > 256, else none;
- the compacted signal of K kept frames is their overlap-add, (K - 1) * 128 + 256 samples long, so it has K - 1 STFT frames;
- a clip with fewer than 30 STFT frames scores 1e-5, and so does a clip with no frame at all (pystoi raises there).
"""
from math import gcd

import numpy as np
from scipy.signal import resample_poly

FS = 10000
N_FRAME = 256
HOP = 128
NFFT = 512
NUM_BANDS = 15
MIN_FREQ = 150
N_SEG = 30
BETA = -15.0
DYN_RANGE = 40
EPS = np.finfo(np.float64).eps
SHORT_SCORE = 1e-5

#: [lo, hi) rfft bins of the 15 one-third-octave bands at 10 kHz / 512 points
BANDS = ((7, 9), (9, 11), (11, 14), (14, 17), (17, 22), (22, 27), (27, 34), (34, 43), (43, 55), (55, 69), (69, 87), (87, 109),
         (109, 138), (138, 174), (174, 219))


def si_sdr(ref, est):
    """10 log10(|a r|^2 / |e - a r|^2), a = <r, e> / <r, r>, in float64."""
    r = np.asarray(ref, np.float64)
    e = np.asarray(est, np.float64)
    a = np.dot(r, e) / np.dot(r, r)
    proj = a * r
    noise = e - proj
    return float(10 * np.log10(np.sum(proj ** 2) / np.sum(noise ** 2)))


def thirdoct_bins(fs=FS, nfft=NFFT, num_bands=NUM_BANDS, min_freq=MIN_FREQ):
    """Each band's [lo, hi) bins: its edges min_freq 2^((2k -+ 1) / 6) rounded to the nearest rfft bin."""
    f = np.linspace(0, fs, nfft + 1)[:nfft // 2 + 1]
    k = np.arange(num_bands, dtype=np.float64)
    lo = min_freq * np.power(2.0, (2 * k - 1) / 6)
    hi = min_freq * np.power(2.0, (2 * k + 1) / 6)
    return tuple((int(np.argmin((f - a) ** 2)), int(np.argmin((f - b) ** 2))) for a, b in zip(lo, hi))


def rates(fs):
    """(p, q): resampling fs to 10 kHz is up p, down q."""
    g = gcd(FS, int(fs))
    return FS // g, int(fs) // g


def resample_filter(fs):
    """The Octave-compatible anti-aliasing filter pystoi's resample_oct builds for 10 kHz / fs: a Kaiser-windowed sinc with 60 dB
    rejection, cut off at 1 / (2 max(p, q)) and rolled off over a tenth of that; normalised to unit sum."""
    p, q = rates(fs)
    cutoff = 1.0 / (2 * max(p, q))
    roll_off = cutoff / 10
    rejection_db = 60.0
    half = int(np.ceil((rejection_db - 8) / (28.714 * roll_off)))
    t = np.arange(-half, half + 1)
    ideal = 2 * p * cutoff * np.sinc(2 * cutoff * t)
    beta = 0.1102 * (rejection_db - 8.7)
    h = np.kaiser(2 * half + 1, beta) * ideal
    return h / np.sum(h)


def resampled_length(n, fs):
    p, q = rates(fs)
    return n if p == q else -(-n * p // q)


def resample(x, fs):
    """x (fs) at 10 kHz, as scipy.signal.resample_poly(x, p, q, window=resample_filter(fs)) in float64."""
    x = np.asarray(x, np.float64)
    if int(fs) == FS:
        return x.copy()
    p, q = rates(fs)
    return resample_poly(x, p, q, window=resample_filter(fs))


def resample_direct(x, fs, m):
    """Output samples m of resample(x, fs) from the polyphase sum the device evaluates: y[m] = sum_j x[j] p h[(Nh - 1) / 2 + m q - j p]."""
    x = np.asarray(x, np.float64)
    p, q = rates(fs)
    h = resample_filter(fs) * p
    half = (h.size - 1) // 2
    out = np.zeros(len(m))
    for i, mm in enumerate(m):
        c = half + mm * q
        j = np.arange(max(0, -(-(c - h.size + 1) // p)), min(x.size - 1, c // p) + 1)
        out[i] = np.dot(x[j], h[c - j * p])
    return out


def window():
    """np.hanning(258)[1:-1]: the 256-point frame window."""
    return np.hanning(N_FRAME + 2)[1:-1]


def num_frames(n):
    """Frames of range(0, n - 256, 128)."""
    return len(range(0, n - N_FRAME, HOP))


def frames(x):
    w = window()
    return np.array([w * x[i:i + N_FRAME] for i in range(0, len(x) - N_FRAME, HOP)]).reshape(-1, N_FRAME)


def frame_energies(xr):
    """20 log10(|windowed frame| + EPS) of every frame of the 10 kHz signal xr."""
    return 20 * np.log10(np.linalg.norm(frames(xr), axis=1) + EPS)


def kept_frames(xr):
    """(energies, threshold, mask): a frame is kept when max_energy - 40 - energy < 0."""
    e = frame_energies(xr)
    if e.size == 0:
        return e, None, np.zeros(0, bool)
    thr = np.max(e) - DYN_RANGE
    return e, thr, (thr - e) < 0


def overlap_add(fr):
    k = fr.shape[0]
    out = np.zeros((k - 1) * HOP + N_FRAME if k else 0)
    for i in range(k):
        out[i * HOP:i * HOP + N_FRAME] += fr[i]
    return out


def remove_silent_frames(xr, yr):
    _, _, mask = kept_frames(xr)
    return overlap_add(frames(xr)[mask]), overlap_add(frames(yr)[mask])


def stft(x):
    """[frames, 257] rfft of the windowed 256-sample frames, zero-padded to 512 points."""
    return np.fft.rfft(frames(x), n=NFFT, axis=1)


def band_envelopes(x):
    """[15, frames]: sqrt of each band's summed |X|^2."""
    p = np.abs(stft(x)) ** 2
    return np.sqrt(np.stack([p[:, lo:hi].sum(axis=1) for lo, hi in BANDS]))


def stoi_envelopes(x, y, fs):
    """Band envelopes of x and y after resampling and silent-frame removal (the per-segment stage's input)."""
    xs, ys = remove_silent_frames(resample(x, fs), resample(y, fs))
    return band_envelopes(xs), band_envelopes(ys)


def stoi(x, y, fs):
    """Classic STOI of the estimate y against the reference x at fs Hz."""
    xr, yr = resample(x, fs), resample(y, fs)
    if num_frames(xr.size) == 0:
        return SHORT_SCORE
    xs, ys = remove_silent_frames(xr, yr)
    X, Y = band_envelopes(xs), band_envelopes(ys)
    if X.shape[1] < N_SEG:
        return SHORT_SCORE
    xseg = np.array([X[:, m - N_SEG:m] for m in range(N_SEG, X.shape[1] + 1)])
    yseg = np.array([Y[:, m - N_SEG:m] for m in range(N_SEG, Y.shape[1] + 1)])
    norm = np.linalg.norm(xseg, axis=2, keepdims=True) / (np.linalg.norm(yseg, axis=2, keepdims=True) + EPS)
    yp = np.minimum(yseg * norm, xseg * (1 + 10 ** (-BETA / 20)))
    yp = yp - np.mean(yp, axis=2, keepdims=True)
    xc = xseg - np.mean(xseg, axis=2, keepdims=True)
    yp /= np.linalg.norm(yp, axis=2, keepdims=True) + EPS
    xc /= np.linalg.norm(xc, axis=2, keepdims=True) + EPS
    return float(np.sum(yp * xc) / (xc.shape[0] * xc.shape[1]))


def threshold_margin(x, fs):
    """The smallest |energy - threshold| over the frames of x, in dB (inf without frames): a fixture whose margin is below the
    rounding of an fp32 resampler could flip a keep / drop decision, and its test would then check a tie-break, not arithmetic."""
    e, thr, _ = kept_frames(resample(x, fs))
    return float(np.min(np.abs(e - thr))) if e.size else float("inf")
