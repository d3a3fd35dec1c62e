"""fp64 truth and single-precision emulation of the audio transforms around the model: the offline STFT (audio_stft_kernel), the cIRM
product (apply_cirm_kernel, apply_cirm_planar_kernel, the fused heads) and the overlap-add synthesis (audio_istft_kernel), each from
the kernels' own input, with the weighting that makes every frame, sample and bin count, and the planted faults the rule must catch.

* stft_truth / stft_emulate: np.fft.rfft of the windowed frames of one clip, frame j = stream_ref.frame_index(j, hop, L_b) (reflected
  at 0 and at the clip's own end), T_b = L_b // hop + 1 frames; the emulation is the fp32 window product through scipy.fft's fp32 FFT.
  Weight (stft_weights): each frame's errors over the L2 norm of its windowed samples, the natural scale of an FFT's rounding.  A
  frame of digital silence has no scale: the kernel must give exactly 0 there.
* cirm_truth / cirm_emulate: O.decompress_cIRM of the fp32 mask, the attenuation floor of include/fsnplus_b200.h (a decompressed mask
  whose magnitude is below lam is raised to lam keeping its phase, a zero mask becomes (lam, 0)), then M X; the emulation clamps at
  9.9f and runs fsn_common.cuh's decompress_cirm / limit_mask and the product in fp32.  Weight: each element over |X| (|M| + 10):
  the product rounds relative to |M| |X|, and the decompression -10 log((10 - m) / (10 + m)) rounds its quotient to fp32 before the
  log, an absolute error of about 10 eps in each mask component whatever |M| is (eps = 2^-23).  Over |M| |X| alone that error of a
  component near 0 beside a larger one reaches 2e-4 of the element in the emulation itself, and the bound with it.
* istft_truth / istft_emulate: irfft (which drops the DC and Nyquist imaginary parts), the window, overlap-add and division by the
  two-frame envelope w^2(i + hop) + w^2(i), or by w^2(i + hop) alone for the last L_b mod hop samples; the emulation uses the fp32
  tables audio_tables rounds from double.  Weight: each sample times its envelope, i.e. the overlap-add sum before the division, so
  the interior and the one-frame end share one bound.

The rule is sb_rnn_ref.compare(got, want, emu, factor) on the weighted arrays.  STFT_FAULTS, ISTFT_FAULTS and CIRM_FAULTS plant the
bugs it must catch (test_audio_xforms_cpu.py).  The case lists the GPU file runs are built here, so that the CPU file can assert the
edges they reach.
"""
import numpy as np

import stream_ref
from oracle import fsn_oracle as O

F32 = np.float32
AUDIO_RUN_POINTS = 2048                   # k_audio.cu: frames (analysis) / output hops (synthesis) per CTA = 2048 / hop
N_FFTS = (64, 128, 256, 512, 1024)        # every n_fft the audio calls take (num_freqs 33 .. 513)
CIRM_ABS = 10.0                           # decompress_cirm's absolute rounding, in units of eps (see the module docstring)
LIM_F32 = F32(9.9)

STFT_FAULTS = ("run_early", "reflect_row", "right_reflect", "last_frame_zero")
ISTFT_FAULTS = ("env_at_end", "inv_last_shift", "dc_nyq_imag", "run_last_one_frame", "tail_window", "emit_m0")
CIRM_FAULTS = ("nyquist_conj", "limit_first", "mask_swap", "product_conj", "ring_next")


def run_frames(hop):
    """R: the frames of one analysis CTA and the output hops of one synthesis CTA (launch_audio_stft / launch_audio_istft)"""
    return AUDIO_RUN_POINTS // hop


def frames_of(Lb, hop):
    return Lb // hop + 1


# ---- tables ---------------------------------------------------------------------------------------------------------------------------
def tables(n_fft):
    """(window, two-frame envelope [hop], one-frame envelope [hop]) in fp64"""
    H = n_fft // 2
    w = O.hann_periodic(n_fft)
    return w, w[:H] ** 2 + w[H:] ** 2, w[H:] ** 2


def tables_f32(n_fft):
    """audio_tables: the window, 1 / envelope and 1 / one-frame envelope, each computed in double and rounded to float"""
    w, env, last = tables(n_fft)
    return w.astype(F32), (1.0 / env).astype(F32), (1.0 / last).astype(F32)


# ---- analysis -------------------------------------------------------------------------------------------------------------------------
def _index(j, hop, Lb, L, fault):
    if fault == "reflect_row":                                     # reflected at the row length L instead of the clip's L_b
        return stream_ref.frame_index(j, hop, L)
    return stream_ref.frame_index(j, hop, Lb, "right_reflect" if fault == "right_reflect" else None)


def stft_truth(row, Lb, hop):
    """row: the clip's row (at least L_b samples) -> (X [F, T_b] complex128, frame norms [T_b]): rfft of the windowed frames, fp64"""
    x = np.asarray(row, np.float64)
    w = O.hann_periodic(2 * hop)
    fr = np.stack([x[stream_ref.frame_index(j, hop, Lb)] for j in range(frames_of(Lb, hop))]) * w
    return np.fft.rfft(fr, axis=1).T, np.linalg.norm(fr, axis=1)


def stft_emulate(row, Lb, hop, fault=None):
    """The same in single precision (fp32 window product, scipy.fft's fp32 rfft) -> [F, T_b] complex128.  fault: one of STFT_FAULTS
      run_early:       frame t0 of every analysis run but the first (t0 = k R) is staged one hop early (frame t0 - 1's samples);
      reflect_row:     the right reflection at the row length L (len(row)) instead of the clip's L_b;
      right_reflect:   2 L_b - 1 - p instead of 2 (L_b - 1) - p;
      last_frame_zero: the clip's last frame T_b - 1 is zero."""
    import scipy.fft
    x = np.asarray(row, F32)
    w = O.hann_periodic(2 * hop).astype(F32)
    Tb, R = frames_of(Lb, hop), run_frames(hop)
    idx = [_index(j - 1 if fault == "run_early" and j and j % R == 0 else j, hop, Lb, len(x), fault) for j in range(Tb)]
    X = scipy.fft.rfft((x[np.stack(idx)] * w).astype(F32), axis=1).T.astype(np.complex128)
    if fault == "last_frame_zero":
        X[:, Tb - 1] = 0
    return X


def stft_weights(norms):
    """[T_b] weights of each frame's errors: 1 / the L2 norm of its windowed samples; 0 where the frame is digital silence"""
    n = np.asarray(norms, np.float64)
    return np.where(n > 0, 1.0 / np.where(n > 0, n, 1.0), 0.0)


def stft_arrays(got_re, got_im, X, emu, norms):
    """(got, want, emu) weighted per frame for the rule, real and imaginary parts side by side, silent frames left out; and the
    largest |got| on the silent frames (must be 0)"""
    s = stft_weights(norms)
    live = s > 0
    g = np.concatenate([np.asarray(got_re, np.float64), np.asarray(got_im, np.float64)]) * s
    want = np.concatenate([X.real, X.imag]) * s
    e = np.concatenate([emu.real, emu.imag]) * s
    silent = max(float(np.abs(got_re[:, ~live]).max(initial=0)), float(np.abs(got_im[:, ~live]).max(initial=0)))
    return g[:, live], want[:, live], e[:, live], silent


# ---- the cIRM product -----------------------------------------------------------------------------------------------------------------
def _limit(m0, m1, lam, dt):
    """limit_mask in arithmetic dt: |M| below lam raised to lam with M's phase, a zero M to (lam, 0)"""
    a2 = (m0 * m0 + m1 * m1).astype(dt)
    low = a2 < (lam * lam).astype(dt)
    s = np.where(a2 > 0, (lam / np.sqrt(np.where(a2 > 0, a2, 1)).astype(dt)).astype(dt), 1).astype(dt)
    n0 = np.where(low, np.where(a2 > 0, m0 * s, lam), m0).astype(dt)
    n1 = np.where(low, np.where(a2 > 0, m1 * s, 0), m1).astype(dt)
    return n0, n1


def _lam(lam, shape):
    """lam: None, a float or [B] (clips / slots on axis 0 of shape) -> broadcastable array or None"""
    if lam is None:
        return None
    lam = np.asarray(lam, np.float64)
    return lam.reshape((-1,) + (1,) * (len(shape) - 1)) if lam.ndim else lam


def cirm_truth(mask, X, lam=None):
    """mask [B, 2, ...] (the kernel's fp32 values), X [B, ...] complex, lam None or [B] (the fp32 floors the kernel reads) ->
    (E complex128, weight scale |X| (|M| + 10)) in fp64"""
    m = O.decompress_cIRM(np.asarray(mask, np.float64))
    m0, m1 = m[:, 0], m[:, 1]
    lm = _lam(lam, m0.shape)
    if lm is not None:
        m0, m1 = _limit(m0, m1, np.broadcast_to(lm, m0.shape), np.float64)
    X = np.asarray(X, np.complex128)
    M = m0 + 1j * m1
    return M * X, np.abs(X) * (np.abs(M) + CIRM_ABS)


def decompress_f32(v):
    """fsn_common.cuh decompress_cirm: the clamp at 9.9f, then -10 logf((10 - v) / (10 + v)), in fp32"""
    v = np.asarray(v, F32)
    v = np.where(v >= LIM_F32, LIM_F32, np.where(v <= -LIM_F32, -LIM_F32, v)).astype(F32)
    with np.errstate(divide="ignore"):
        return (F32(-10.0) * np.log(((F32(10.0) - v) / (F32(10.0) + v)).astype(F32))).astype(F32)


def cirm_emulate(mask, X, lam=None, fault=None):
    """The kernels' fp32 arithmetic -> complex128.  fault: one of CIRM_FAULTS
      nyquist_conj: the Nyquist bin (axis 1 = F of X, last bin) of the product conjugated;
      limit_first:  the floor applied to the compressed mask, before decompression;
      mask_swap:    the two mask channels swapped;
      product_conj: conj(M X);
      ring_next:    the streaming synthesis reads the spectrum ring at (m + 1) % R: frame m is multiplied by the spectrum of frame m + 1
                    (X's last axis is the frame; the last frame keeps its own)."""
    mask = np.asarray(mask, F32)
    c0, c1 = (mask[:, 1], mask[:, 0]) if fault == "mask_swap" else (mask[:, 0], mask[:, 1])
    lm = _lam(lam, c0.shape)
    lm = None if lm is None else np.broadcast_to(lm.astype(F32), c0.shape)
    if lm is not None and fault == "limit_first":
        c0, c1 = _limit(c0, c1, lm, F32)
    m0, m1 = decompress_f32(c0), decompress_f32(c1)
    if lm is not None and fault != "limit_first":
        m0, m1 = _limit(m0, m1, lm, F32)
    X = np.asarray(X, np.complex64)
    if fault == "ring_next":
        X = np.concatenate([X[..., 1:], X[..., -1:]], axis=-1)
    xr, xi = X.real.astype(F32), X.imag.astype(F32)
    E = ((m0 * xr - m1 * xi).astype(F32) + 1j * (m1 * xr + m0 * xi).astype(F32)).astype(np.complex128)
    if fault == "product_conj":
        E = np.conj(E)
    if fault == "nyquist_conj":
        E[:, -1] = np.conj(E[:, -1])
    return E


def cirm_arrays(got, E, emu, scale):
    """(got, want, emu) weighted per element, real and imaginary parts, for the rule; elements with scale 0 left out; and the largest
    |got| on those (must be 0)"""
    s = np.asarray(scale, np.float64)
    live = s > 0
    w = 1.0 / np.where(live, s, 1.0)
    got = np.asarray(got, np.complex128)
    pack = lambda z: np.concatenate([(z.real * w)[live], (z.imag * w)[live]])
    return pack(got), pack(E), pack(emu), float(np.abs(got[~live]).max(initial=0))


# ---- synthesis ------------------------------------------------------------------------------------------------------------------------
def envelope(Lb, hop):
    """[L_b]: the overlap-add envelope of each output sample, w^2(i + hop) + w^2(i), and w^2(i + hop) for the last L_b mod hop"""
    _, env, last = tables(2 * hop)
    n = np.arange(Lb)
    q, k = n // hop, n % hop
    return np.where(q + 1 < frames_of(Lb, hop), env[k], last[k])


def istft_truth(E, Lb, hop):
    """E [F, >= T_b] (the kernel's enhanced spectrum) -> y [L_b] fp64: torch.istft(length = L_b) of frames 0 .. T_b - 1"""
    N, Tb = 2 * hop, frames_of(Lb, hop)
    w = O.hann_periodic(N)
    fr = np.fft.irfft(np.asarray(E, np.complex128)[:, :Tb].T, n=N, axis=1) * w
    y = np.zeros(hop * (Tb + 1))
    for t in range(Tb):
        y[t * hop:t * hop + N] += fr[t]
    return y[hop:hop + Lb] / envelope(Lb, hop)


def istft_emulate(E, Lb, hop, fault=None):
    """audio_istft_kernel's arithmetic: the DC / Nyquist imaginary parts dropped, scipy.fft's fp32 irfft, the fp32 window and tables
    -> [L_b] float64.  fault: one of ISTFT_FAULTS
      env_at_end:         the last L_b mod hop samples divided by the two-frame envelope (inv_env) instead of inv_last;
      inv_last_shift:     inv_last read one sample shifted (k + 1);
      dc_nyq_imag:        the DC and Nyquist imaginary parts not dropped (the inverse split then folds them into the even / odd samples);
      run_last_one_frame: the last hop of every synthesis run (q mod R = R - 1) treated as one-frame, w(i + hop) y_q / w^2(i + hop);
      tail_window:        the one-frame end windowed with w[i] instead of w[hop + i];
      emit_m0:            frame 0's first half emitted as a hop of its own (everything one hop late)."""
    import scipy.fft
    N, Tb, R = 2 * hop, frames_of(Lb, hop), run_frames(hop)
    w, inv_env, inv_last = tables_f32(N)
    E = np.asarray(E, np.complex64)[:, :Tb].copy()
    dcn = E[[0, hop]].imag.astype(np.float64)
    E[[0, hop]] = E[[0, hop]].real
    fr = scipy.fft.irfft(E.T, n=N, axis=1).astype(F32)                 # [T_b, N]
    if fault == "dc_nyq_imag":                                          # y[2n] -= (b + d) / N, y[2n + 1] += (b - d) / N
        b, d = dcn[0], dcn[1]
        fr[:, 0::2] -= ((b + d) / N).astype(F32)[:, None]
        fr[:, 1::2] += ((b - d) / N).astype(F32)[:, None]
    hi = (fr[:, hop:] * w[hop:]).astype(F32)
    lo = (fr[:, :hop] * w[:hop]).astype(F32)
    if fault == "tail_window":
        tw = (fr[:, hop:] * w[:hop]).astype(F32)
    n = np.arange(Lb)
    q, k = n // hop, n % hop
    inner = q + 1 < Tb
    qn = np.minimum(q + 1, Tb - 1)
    y = np.where(inner, ((hi[q, k] + lo[qn, k]).astype(F32) * inv_env[k]).astype(F32), (hi[q, k] * inv_last[k]).astype(F32))
    if fault == "env_at_end":
        y = np.where(inner, y, (hi[q, k] * inv_env[k]).astype(F32))
    elif fault == "inv_last_shift":
        y = np.where(inner, y, (hi[q, k] * inv_last[np.minimum(k + 1, hop - 1)]).astype(F32))
    elif fault == "run_last_one_frame":
        y = np.where(q % R == R - 1, (hi[q, k] * inv_last[k]).astype(F32), y)
    elif fault == "tail_window":
        y = np.where(inner, y, (tw[q, k] * inv_last[k]).astype(F32))
    elif fault == "emit_m0":
        y = np.concatenate([(lo[0] * inv_env).astype(F32), y])[:Lb]
    return y.astype(np.float64)


def istft_arrays(got, want, emu, Lb, hop):
    """(got, want, emu) of one clip, each sample times its envelope (the overlap-add sum before the division)"""
    env = envelope(Lb, hop)
    return tuple(np.asarray(a, np.float64)[:Lb] * env for a in (got, want, emu))


# ---- cases ----------------------------------------------------------------------------------------------------------------------------
def residues(hop):
    """the L mod hop classes every length list covers: 0, 1, hop / 2, hop - 1"""
    return (0, 1, hop // 2, hop - 1)


def short_lengths(n_fft):
    """the shortest clips: hop + 1, hop + 2, n_fft - 1, n_fft, n_fft + 1"""
    hop = n_fft // 2
    return [hop + 1, hop + 2, n_fft - 1, n_fft, n_fft + 1]


def run_lengths(n_fft, runs=(1, 2)):
    """lengths q hop + r with q around the k-th run boundary (q in k R - 2 .. k R + 1, k in runs) and r in residues(hop): T_b = q + 1
    and ceil(L_b / hop) = q + (r > 0) then fall on both sides of each boundary"""
    hop = n_fft // 2
    R = run_frames(hop)
    return [q * hop + r for k in runs for q in range(k * R - 2, k * R + 2) for r in residues(hop)]


def long_length(n_fft):
    """one clip of more than three analysis and synthesis runs"""
    hop = n_fft // 2
    return (3 * run_frames(hop) + 5) * hop + hop // 2 + 3


def offline_lengths(n_fft):
    """every clip length of the per-n_fft ragged batch of the GPU file"""
    return short_lengths(n_fft) + run_lengths(n_fft) + [long_length(n_fft)]


def boundaries_hit(lengths, hop):
    """{(kind, k, side)}: the run boundaries k R (k >= 1) that the frame counts T_b (kind "stft") and the output hop counts
    ceil(L_b / hop) (kind "istft") reach from below (side -1: count = k R - 1 .. the last run is short by one), exactly (0) and from above
    (+1: one frame or hop into the next run)"""
    R = run_frames(hop)
    hit = set()
    for L in lengths:
        for kind, cnt in (("stft", frames_of(L, hop)), ("istft", -(-L // hop))):
            for k in range(1, cnt // R + 2):
                d = cnt - k * R
                if d in (-1, 0, 1):
                    hit.add((kind, k, d))
    return hit


def speech(n, seed, level=1.0):
    """n samples of synthetic noisy speech at `level` times its usual amplitude, float32 (generated at >= 1000 samples: the
    generator's envelope smoothing needs them)"""
    return (O.synth_clips(1, num_samples=max(n, 1000), seed0=seed)[0, :n] * level).astype(F32)


def with_silence(n, seed):
    """speech with digital silence over [n / 3, n / 2) and over its last quarter: whole frames of exact zeros"""
    x = speech(n, seed)
    x[n // 3:n // 2] = 0
    x[3 * n // 4:] = 0
    return x
