"""fp64 truth and emulation of one streaming step call (fsn_stream_step / _step_slots / _step_chunk), from the kernels' own input and
carried state, and the decoder of a saved session's payload.

A call of K frames runs, per slot: the cumulative norm (stream_norm_kernel) -> fb_in; the full-band LSTM / GRU from the carried
(h_fb, c_fb) -> fb_out; the sub-band pack (stream_pack_frame_kernel / stream_pack_kernel / stream_pack_wide_kernel) of the magnitude
and fb_out with its own running sums -> the fp16 sub-band input; the sub-band LSTM / GRU from the carried (h_sb, c_sb) -> mask column k
of frame n_b + k - look_ahead.  Each stage is checked from what the kernels fed it (get_stage, the saved payloads), so an error is
charged to the stage that made it:

* norm_truth / norm_emulate: the reference's cumulative norm (oracle NORMS) of the session's frames since its START, which is causal,
  so the offline norm of the whole session is the truth of every streamed frame; the emulation sums in fp64, casts the scale to fp32
  and applies fmaf.  norm_sums: the fp64 sums the payload's cum_in must hold.
* sb_truth / sb_emulate: the unfold of (magnitude, fb_out) with reflect at both bin edges, cumulative-normalised over every frame of
  the session (fp64); the emulation is the kernels' fp32 fmaf, the +-65504 clamp and the fp16 rounding.  sb_sums: cum_sb's fp64 sums.
* The recurrences: sb_rnn_ref.truth / emulate with state= (the payload before the call) and return_state=True (compared with the
  payload after it).
* decode: a payload [stride] uint8 -> its six model segments, at the offsets of fsn_stream_state_layout (DESIGN.md §3.11).

NORM_FAULTS and PACK_FAULTS plant the bugs the rule must catch (test_stream_step_cpu.py); the recurrences' faults are planted in the
state they start from.
"""
import numpy as np

from oracle import fsn_oracle as O

F32 = np.float32
EPS = 1.1920928955078125e-07

NORM_FAULTS = ("no_restart", "count_n", "held_advances")
PACK_FAULTS = ("top_replicate", "window_restart")


# ---- payload ------------------------------------------------------------------------------------------------------------------------
def segments(F, L, Hfb, Hsb):
    """[(name, shape, dtype)] of the model segments in payload order: cum_in, cum_sb (fp64 sum and sum of squares), then the
    full band's and the sub band's h (fp16) and c (fp32; GRU: the fp32 h)"""
    return [("cum_in", (2,), np.float64), ("cum_sb", (F, 2), np.float64), ("h_fb", (L, Hfb), np.float16), ("c_fb", (L, Hfb), np.float32),
            ("h_sb", (L, F, Hsb), np.float16), ("c_sb", (L, F, Hsb), np.float32)]


def offsets(F, L, Hfb, Hsb):
    """each segment's byte offset (16-byte aligned, in order) and the end of the last one"""
    off, o = [], 0
    for _, shape, dt in segments(F, L, Hfb, Hsb):
        off.append(o)
        o += (int(np.prod(shape)) * np.dtype(dt).itemsize + 15) // 16 * 16
    return off, o


def decode(payload, F, L, Hfb, Hsb):
    """one session's payload (bytes, uint8 array or tensor) -> {name: array} of the model segments (float64 copies)"""
    raw = np.frombuffer(np.ascontiguousarray(np.asarray(payload, np.uint8)).tobytes(), np.uint8)
    off, _ = offsets(F, L, Hfb, Hsb)
    out = {}
    for o, (name, shape, dt) in zip(off, segments(F, L, Hfb, Hsb)):
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        out[name] = np.frombuffer(raw[o:o + n].tobytes(), dt).reshape(shape).astype(np.float64)
    return out


# ---- the cumulative norm --------------------------------------------------------------------------------------------------------------
def norm_truth(x, kind):
    """x [F, N]: the session's frames since its START -> the reference's cumulative norm [F, N], float64"""
    return O.NORMS[kind](np.asarray(x, np.float64)[None, None])[0, 0]


def _scale(s, q, cnt, kind):
    cm = s / cnt
    if kind == "cumulative_laplace_norm":
        return (1.0 / (cm + EPS)).astype(F32), np.zeros_like(cm, dtype=F32)
    inv = 1.0 / np.sqrt((q - 2.0 * cm * s) / cnt + cm * cm + EPS)
    return inv.astype(F32), (-cm * inv).astype(F32)


def norm_sums(x):
    """fp64 running (sum, sum of squares) over F after every frame of x [F, N]: [N, 2]"""
    x = np.asarray(x, F32).astype(np.float64)
    return np.stack([np.cumsum(x.sum(0)), np.cumsum((x * x).sum(0))], axis=1)


def norm_emulate(x, kind, fault=None, fault_at=0, carry=None):
    """stream_norm_kernel over x [F, N] (float32, the session's frames): fp64 running sums, the scale cast to fp32, fmaf.  fault:
      no_restart:    the sums carry `carry` (fp64 (sum, sum of squares) of a previous session) instead of restarting at START;
      count_n:       the count is F n instead of F (n + 1) (frame 0 at F, where F n would divide by zero);
      held_advances: a held tick before frame fault_at adds that frame's values to the sums once more."""
    x = np.asarray(x, F32)
    F, N = x.shape
    sq = norm_sums(x)
    if fault == "no_restart":
        sq = sq + np.asarray(carry, np.float64)[None, :]
    if fault == "held_advances":
        xf = x[:, fault_at].astype(np.float64)
        sq[fault_at:] += np.array([xf.sum(), (xf * xf).sum()])[None, :]
    n = np.arange(N, dtype=np.float64)
    cnt = F * (np.maximum(n, 1.0) if fault == "count_n" else n + 1.0)
    sa, sb = _scale(sq[:, 0], sq[:, 1], cnt, kind)
    return fma32(x, sa[None, :], sb[None, :])


def fma32(a, b, c):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


# ---- the sub-band pack ----------------------------------------------------------------------------------------------------------------
def _reflect(p, F, fault=None):
    p = np.abs(p)
    r = np.where(p > F - 1, 2 * (F - 1) - p, p)
    if fault == "top_replicate":                                         # the top bin's neighbour replicated instead of reflected
        r = np.where(p > F - 1, F - 1, r)
    return r


def unfold(mag, fb, Ns, Nf, fault=None):
    """mag, fb [F, N] -> [F, I, N]: the 2 Ns + 1 magnitude neighbours, then the 2 Nf + 1 full-band neighbours of every bin"""
    F = mag.shape[0]
    f = np.arange(F)
    ch = [mag[_reflect(f + i - Ns, F, fault)] for i in range(2 * Ns + 1)] + [fb[_reflect(f + j - Nf, F, fault)] for j in range(2 * Nf + 1)]
    return np.stack(ch, axis=1)


def sb_truth(mag, fb, Ns, Nf, kind):
    """the normalised sub-band input [F, I, N] (float64) of the session's frames mag, fb [F, N] (the kernels' own values)"""
    x = unfold(np.asarray(mag, np.float64), np.asarray(fb, np.float64), Ns, Nf)
    return O.NORMS[kind](x[None])[0]


def sb_sums(mag, fb, Ns, Nf):
    """cum_sb after the last frame: [F, 2] fp64 (sum, sum of squares) over the channels and every frame"""
    x = unfold(np.asarray(mag, F32), np.asarray(fb, F32), Ns, Nf).astype(np.float64)
    return np.stack([x.sum((1, 2)), (x * x).sum((1, 2))], axis=1)


def sb_emulate(mag, fb, Ns, Nf, kind, fault=None, fault_at=0):
    """the packers' fp16 values [F, I, N] (as float64): fp64 running sums per bin over the channels, the scale cast to fp32, fmaf, the
    +-65504 clamp and the fp16 rounding.  fault: top_replicate (see _reflect); window_restart: the sums restart at frame fault_at, as a
    window k0 > 0 that took itself for the session's first."""
    x = unfold(np.asarray(mag, F32), np.asarray(fb, F32), Ns, Nf, fault)
    F, I, N = x.shape
    xd = x.astype(np.float64)
    s, q = np.cumsum(xd.sum(1), axis=1), np.cumsum((xd * xd).sum(1), axis=1)
    n = np.arange(N, dtype=np.float64)
    cnt = I * (n + 1.0)
    if fault == "window_restart" and 0 < fault_at < N:                  # the count still runs from the session's START
        s[:, fault_at:] -= s[:, fault_at - 1:fault_at]
        q[:, fault_at:] -= q[:, fault_at - 1:fault_at]
    sa, sb = _scale(s, q, cnt, kind)
    y = np.clip(fma32(x, sa[:, None, :], sb[:, None, :]), -65504.0, 65504.0)
    return y.astype(np.float16).astype(np.float64)


# ---- the audio calls' analysis -----------------------------------------------------------------------------------------------------------
AUDIO_FAULTS = ("right_reflect",)


def frame_index(j, hop, L, fault=None):
    """the sample positions of STFT frame j (torch.stft center=True, reflect): [hop (j - 1), hop (j + 1)) reflected at 0 and, with
    L > 0 (the session's length, known after its FLUSH), at L - 1.  fault right_reflect: 2 L - 1 - p instead of 2 (L - 1) - p."""
    p = np.abs(np.arange(hop * (j - 1), hop * (j + 1)))
    if L:
        p = np.where(p >= L, (2 * L - 1 if fault == "right_reflect" else 2 * (L - 1)) - p, p)
    return p


def stft_mag_truth(x, j0, n, hop, L):
    """|rfft(window * frame j)| in fp64 of frames j0 .. j0 + n - 1 of the session's samples x: [F, n]; frames past the session's end
    (j > L / hop, L > 0) are zero frames"""
    w = O.hann_periodic(2 * hop)
    out = np.zeros((hop + 1, n))
    for i in range(n):
        j = j0 + i
        if not (L and j > L // hop):
            out[:, i] = np.abs(np.fft.rfft(np.asarray(x, np.float64)[frame_index(j, hop, L)] * w))
    return out


def stft_mag_emulate(x, j0, n, hop, L, fault=None):
    """the same in single precision: the fp32 windowed frame through scipy.fft.rfft (an fp32 FFT), |.| in fp32"""
    import scipy.fft
    w = O.hann_periodic(2 * hop).astype(F32)
    out = np.zeros((hop + 1, n), F32)
    for i in range(n):
        j = j0 + i
        if not (L and j > L // hop):
            out[:, i] = np.abs(scipy.fft.rfft((np.asarray(x, F32)[frame_index(j, hop, L, fault)] * w).astype(F32)))
    return out.astype(np.float64)
