"""numpy restatement of the reference FullSubNet+/FullSubNet inference forward.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).  Parity status: PINNED by
tests/golden/*.npz, generated from the imported reference by
tests/golden/make_golden.py.

Every function cites the reference file:line it follows (paths relative to
speech_enhance/ of the reference).  All arithmetic is plain numpy, float64 by
default (the "truth" the CUDA path is measured against, SURVEY.md 8c).

The arithmetic of the reference lives in PyTorch (nn.LSTM, nn.Conv1d,
nn.GroupNorm, nn.PReLU, nn.Linear, F.unfold, F.pad(reflect), torch.stft/istft;
torch is a third-party dependency, README pins "pytorch=1.7.1", this image has
2.11); the published definitions of those operators are restated here and
anchored on the reference's call sites.
"""
from __future__ import annotations

import numpy as np

# ----------------------------------------------------------------------------
# configs (config/inference.toml:30-44 and fullsubnet/model/fullsubnet.py:13-26)
# ----------------------------------------------------------------------------

TCN_HIDDEN = 512            # audio_zen/model/module/causal_conv.py:68 (hidden_channel default)
TCN_DILATIONS = (1, 2, 5, 9, 1, 2, 5, 9)   # audio_zen/model/module/sequence_model.py:47-58
GLN_EPS = 1e-8              # causal_conv.py:73,79
NORM_EPS = 1e-5             # audio_zen/model/base_model.py:223
EPSILON = float(np.finfo(np.float32).eps)   # audio_zen/constant.py:8


def default_plus_config():
    """config/inference.toml:30-44."""
    return dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2,
                sequence_model="LSTM", fb_output_activate_function="ReLU",
                sb_output_activate_function=False, channel_attention_model="TSSE",
                fb_model_hidden_size=512, sb_model_hidden_size=384, weight_init=False,
                norm_type="offline_laplace_norm", num_groups_in_drop_band=2,
                kersize=[3, 5, 10], subband_num=1)


def default_fsn_config():
    """fullsubnet/model/fullsubnet.py:124-136 (__main__ hyper-parameters)."""
    return dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2,
                sequence_model="LSTM", fb_output_activate_function="ReLU",
                sb_output_activate_function=False, fb_model_hidden_size=512,
                sb_model_hidden_size=384, weight_init=False,
                norm_type="offline_laplace_norm", num_groups_in_drop_band=2)


# ----------------------------------------------------------------------------
# deterministic parameters (numpy RNG, so fixtures do not depend on torch's RNG)
# ----------------------------------------------------------------------------

def _uni(rng, shape, bound):
    return rng.uniform(-bound, bound, size=shape).astype(np.float32)


def _lstm_params(rng, prefix, inp, hid, layers, out, scale=1.0, gates=4):
    """Keys/shapes of nn.LSTM (gates=4) / nn.GRU (gates=3) + nn.Linear as registered at sequence_model.py:32-46,74-79."""
    p = {}
    b = scale / np.sqrt(hid)
    for l in range(layers):
        k = inp if l == 0 else hid
        p[f"{prefix}.sequence_model.weight_ih_l{l}"] = _uni(rng, (gates * hid, k), b)
        p[f"{prefix}.sequence_model.weight_hh_l{l}"] = _uni(rng, (gates * hid, hid), b)
        p[f"{prefix}.sequence_model.bias_ih_l{l}"] = _uni(rng, (gates * hid,), b)
        p[f"{prefix}.sequence_model.bias_hh_l{l}"] = _uni(rng, (gates * hid,), b)
    p[f"{prefix}.fc_output_layer.weight"] = _uni(rng, (out, hid), 1 / np.sqrt(hid))
    p[f"{prefix}.fc_output_layer.bias"] = _uni(rng, (out,), 1 / np.sqrt(hid))
    return p


def _tcn_params(rng, prefix, nf):
    """Keys/shapes of 8 TCNBlocks + Linear (sequence_model.py:47-58,80-81; causal_conv.py:67-80)."""
    p = {}
    for i in range(8):
        q = f"{prefix}.sequence_model.{i}"
        p[f"{q}.conv1x1.weight"] = _uni(rng, (TCN_HIDDEN, nf, 1), 1 / np.sqrt(nf))
        p[f"{q}.conv1x1.bias"] = _uni(rng, (TCN_HIDDEN,), 1 / np.sqrt(nf))
        p[f"{q}.prelu1.weight"] = np.array([0.25 + 0.02 * i], np.float32)
        p[f"{q}.norm1.weight"] = (1 + 0.1 * rng.standard_normal(TCN_HIDDEN)).astype(np.float32)
        p[f"{q}.norm1.bias"] = (0.1 * rng.standard_normal(TCN_HIDDEN)).astype(np.float32)
        p[f"{q}.depthwise_conv.weight"] = _uni(rng, (TCN_HIDDEN, 1, 3), 1 / np.sqrt(3))
        p[f"{q}.depthwise_conv.bias"] = _uni(rng, (TCN_HIDDEN,), 1 / np.sqrt(3))
        p[f"{q}.prelu2.weight"] = np.array([0.2 + 0.01 * i], np.float32)
        p[f"{q}.norm2.weight"] = (1 + 0.1 * rng.standard_normal(TCN_HIDDEN)).astype(np.float32)
        p[f"{q}.norm2.bias"] = (0.1 * rng.standard_normal(TCN_HIDDEN)).astype(np.float32)
        p[f"{q}.sconv.weight"] = _uni(rng, (nf, TCN_HIDDEN, 1), 1 / np.sqrt(TCN_HIDDEN))
        p[f"{q}.sconv.bias"] = _uni(rng, (nf,), 1 / np.sqrt(TCN_HIDDEN))
    p[f"{prefix}.fc_output_layer.weight"] = _uni(rng, (nf, nf), 1 / np.sqrt(nf))
    p[f"{prefix}.fc_output_layer.bias"] = _uni(rng, (nf,), 1 / np.sqrt(nf))
    return p


def _tsse_params(rng, prefix, nc, kersize):
    """Keys/shapes of ChannelTimeSenseSELayer (attention_model.py:49-76)."""
    p = {}
    for name, k in zip(("smallConv1d", "middleConv1d", "largeConv1d"), kersize):
        p[f"{prefix}.{name}.0.weight"] = _uni(rng, (nc, 1, k), 1 / np.sqrt(k))
        p[f"{prefix}.{name}.0.bias"] = _uni(rng, (nc,), 1 / np.sqrt(k))
    p[f"{prefix}.feature_concate_fc.weight"] = _uni(rng, (1, 3), 1 / np.sqrt(3))
    p[f"{prefix}.feature_concate_fc.bias"] = _uni(rng, (1,), 1 / np.sqrt(3))
    p[f"{prefix}.fc1.weight"] = _uni(rng, (nc // 2, nc), 1 / np.sqrt(nc))
    p[f"{prefix}.fc1.bias"] = _uni(rng, (nc // 2,), 1 / np.sqrt(nc))
    p[f"{prefix}.fc2.weight"] = _uni(rng, (nc, nc // 2), 1 / np.sqrt(nc // 2))
    p[f"{prefix}.fc2.bias"] = _uni(rng, (nc,), 1 / np.sqrt(nc // 2))
    return p


def _attn_params(rng, prefix, nc, cfg):
    kind = cfg.get("channel_attention_model", "TSSE")
    if kind == "TSSE":
        return _tsse_params(rng, prefix, nc, cfg["kersize"])
    if kind == "ECA":                                            # attention_model.py:345
        return {f"{prefix}.conv.weight": _uni(rng, (1, 1, 3), 1 / np.sqrt(3))}
    return {f"{prefix}.fc1.weight": _uni(rng, (nc // 2, nc), 1 / np.sqrt(nc)), f"{prefix}.fc1.bias": _uni(rng, (nc // 2,), 1 / np.sqrt(nc)),
            f"{prefix}.fc2.weight": _uni(rng, (nc, nc // 2), 1 / np.sqrt(nc // 2)), f"{prefix}.fc2.bias": _uni(rng, (nc,), 1 / np.sqrt(nc // 2))}


def make_params_plus(cfg, seed=0, lstm_scale=1.0, num_layers=2):
    """state_dict of FullSubNet_Plus(**cfg) (fullsubnet_plus.py:52-110) with
    PyTorch-default-like scales; ``lstm_scale`` > 1 saturates gates like a
    trained net (SURVEY.md 8c stress variant)."""
    rng = np.random.default_rng(seed)
    nf = cfg["num_freqs"]
    p = {}
    for s in ("", "_real", "_imag"):
        p.update(_attn_params(rng, f"channel_attention{s}", nf, cfg))
    for s in ("", "_real", "_imag"):
        p.update(_tcn_params(rng, f"fb_model{s}", nf))
    isb = (2 * cfg["sb_num_neighbors"] + 1) + 3 * (2 * cfg["fb_num_neighbors"] + 1)
    gates = 3 if cfg.get("sequence_model", "LSTM") == "GRU" else 4
    p.update(_lstm_params(rng, "sb_model", isb, cfg["sb_model_hidden_size"], num_layers,
                          cfg.get("output_size", 2), lstm_scale, gates))
    return p


def make_params_fsn(cfg, seed=0, lstm_scale=1.0, num_layers=2):
    """state_dict of fullsubnet Model(**cfg) (fullsubnet.py:39-57)."""
    rng = np.random.default_rng(seed)
    nf = cfg["num_freqs"]
    p = {}
    gates = 3 if cfg.get("sequence_model", "LSTM") == "GRU" else 4
    p.update(_lstm_params(rng, "fb_model", nf, cfg["fb_model_hidden_size"], num_layers, nf, lstm_scale, gates))
    isb = (2 * cfg["sb_num_neighbors"] + 1) + (2 * cfg["fb_num_neighbors"] + 1)
    p.update(_lstm_params(rng, "sb_model", isb, cfg["sb_model_hidden_size"], num_layers, 2, lstm_scale, gates))
    return p


# ----------------------------------------------------------------------------
# synthetic clips + STFT/iSTFT (audio_zen/acoustics/feature.py:10-65)
# ----------------------------------------------------------------------------

def synth_clips(n, num_samples=48000, sr=16000, seed0=1000):
    """SURVEY.md 8d generator: harmonic 'speech' with syllabic envelope + white
    noise at SNR U[-5, 20] dB (config/train.toml:49), level -25 dBFS +-10
    (recipe of fullsubnet/dataset/dataset_train.py:130-182)."""
    out = np.zeros((n, num_samples), np.float32)
    t = np.arange(num_samples) / sr
    for i in range(n):
        rng = np.random.default_rng(seed0 + i)
        f0 = rng.uniform(100, 300)
        nh = int(rng.integers(3, 6))
        s = np.zeros(num_samples)
        for h in range(1, nh + 1):
            s += rng.uniform(0.3, 1.0) / h * np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 2 * np.pi))
        env = (np.sin(2 * np.pi * rng.uniform(3, 6) * t + rng.uniform(0, 2 * np.pi)) > -0.2).astype(np.float64)
        k = np.hanning(321); k /= k.sum()
        env = np.convolve(env, k, mode="same")
        s *= env
        s *= 0.1 / (np.abs(s).max() + 1e-9)
        snr = rng.uniform(-5, 20)
        noise = rng.standard_normal(num_samples)
        ps, pn = np.mean(s ** 2) + 1e-12, np.mean(noise ** 2)
        noise *= np.sqrt(ps / (pn * 10 ** (snr / 10)))
        y = s + noise
        level = rng.uniform(-35, -15)
        y *= 10 ** (level / 20) / (np.sqrt(np.mean(y ** 2)) + 1e-12)
        out[i] = np.clip(y, -0.99, 0.99).astype(np.float32)
    return out


def hann_periodic(n):
    return 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n) / n)


def stft(y, n_fft=512, hop=256, win=512, dtype=np.float64):
    """torch.stft(y, n_fft, hop, win, window=hann, center=True, reflect pad,
    return_complex=True) as called at feature.py:24-31.  y [B, L] -> [B, F, T] complex."""
    assert win == n_fft
    y = np.asarray(y, dtype)
    yp = np.pad(y, ((0, 0), (n_fft // 2, n_fft // 2)), mode="reflect")
    T = 1 + (yp.shape[1] - n_fft) // hop
    idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
    frames = yp[:, idx] * hann_periodic(n_fft).astype(dtype)       # [B, T, n_fft]
    return np.fft.rfft(frames, axis=-1).transpose(0, 2, 1)


def istft(X, n_fft=512, hop=256, win=512, length=None):
    """torch.istft(X, n_fft, hop, win, window=hann, length=length) (feature.py:58-65)."""
    B, F, T = X.shape
    w = hann_periodic(n_fft)
    frames = np.fft.irfft(X.transpose(0, 2, 1), n=n_fft, axis=-1) * w      # [B, T, n_fft]
    L = n_fft + hop * (T - 1)
    y = np.zeros((B, L)); env = np.zeros(L)
    for t in range(T):
        y[:, t * hop:t * hop + n_fft] += frames[:, t]
        env[t * hop:t * hop + n_fft] += w * w
    y = y[:, n_fft // 2:]; env = env[n_fft // 2:]
    if length is not None:
        y = y[:, :length]; env = env[:length]
    return y / np.where(env > 1e-11, env, 1.0)


def decompress_cIRM(mask, K=10, limit=9.9):
    """audio_zen/acoustics/mask.py:60-63."""
    mask = limit * (mask >= limit) - limit * (mask <= -limit) + mask * (np.abs(mask) < limit)
    return -K * np.log((K - mask) / (K + mask))


def enhance(noisy_complex, crm):
    """fullsubnet_plus/inferencer/inferencer.py:152-157. crm [B,2,F,T] -> complex [B,F,T]."""
    m = decompress_cIRM(crm)
    er = m[:, 0] * noisy_complex.real - m[:, 1] * noisy_complex.imag
    ei = m[:, 1] * noisy_complex.real + m[:, 0] * noisy_complex.imag
    return er + 1j * ei


# ----------------------------------------------------------------------------
# building blocks
# ----------------------------------------------------------------------------

def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def offline_laplace_norm(x):
    """base_model.py:210-225.  x [B, C, F, T]."""
    mu = x.mean(axis=(1, 2, 3), keepdims=True)
    return x / (mu + NORM_EPS)


def cumulative_laplace_norm(x):
    """base_model.py:227-258.  x [B, C, F, T]."""
    B, C, F, T = x.shape
    xr = x.reshape(B * C, F, T)
    csum = np.cumsum(xr.sum(axis=1), axis=-1)
    cnt = np.arange(F, F * T + 1, F, dtype=x.dtype).reshape(1, T)
    cmean = (csum / cnt).reshape(B * C, 1, T)
    return (xr / (cmean + EPSILON)).reshape(B, C, F, T)


def offline_gaussian_norm(x):
    """base_model.py:260-275 (torch.std is the unbiased estimator)."""
    mu = x.mean(axis=(1, 2, 3), keepdims=True)
    std = x.std(axis=(1, 2, 3), keepdims=True, ddof=1)
    return (x - mu) / (std + NORM_EPS)


def cumulative_layer_norm(x):
    """base_model.py:277-316."""
    B, C, F, T = x.shape
    xr = x.reshape(B * C, F, T)
    csum = np.cumsum(xr.sum(axis=1), axis=-1)
    cpow = np.cumsum((xr * xr).sum(axis=1), axis=-1)
    cnt = np.arange(F, F * T + 1, F, dtype=x.dtype).reshape(1, T)
    cmean = csum / cnt
    cvar = (cpow - 2 * cmean * csum) / cnt + cmean ** 2
    cstd = np.sqrt(cvar + EPSILON)
    return ((xr - cmean[:, None, :]) / cstd[:, None, :]).reshape(B, C, F, T)


NORMS = dict(offline_laplace_norm=offline_laplace_norm,
             cumulative_laplace_norm=cumulative_laplace_norm,
             offline_gaussian_norm=offline_gaussian_norm,
             cumulative_layer_norm=cumulative_layer_norm)   # base_model.py:318-330


def unfold(x, n):
    """base_model.py:15-47.  x [B, C, F, T] -> [B, F, C, 2n+1, T] (reflect pad on F)."""
    B, C, F, T = x.shape
    if n < 1:
        return x.transpose(0, 2, 1, 3).reshape(B, F, C, 1, T)
    xp = np.pad(x, ((0, 0), (0, 0), (n, n), (0, 0)), mode="reflect")
    idx = np.arange(F)[:, None] + np.arange(2 * n + 1)[None, :]     # [F, 2n+1]
    return xp[:, :, idx, :].transpose(0, 2, 1, 3, 4)


def tsse(x, p, prefix, kersize):
    """ChannelTimeSenseSELayer.forward (attention_model.py:78-98).  x [B, C, T]."""
    B, C, T = x.shape
    feats = []
    for name, k in zip(("smallConv1d", "middleConv1d", "largeConv1d"), kersize):
        w = p[f"{prefix}.{name}.0.weight"].astype(x.dtype)[:, 0, :]        # [C, k]
        b = p[f"{prefix}.{name}.0.bias"].astype(x.dtype)
        To = T - k + 1
        y = np.zeros((B, C, To), x.dtype)
        for j in range(k):                                                 # depthwise, no padding
            y += w[None, :, j, None] * x[:, :, j:j + To]
        y += b[None, :, None]
        feats.append(np.maximum(y.mean(axis=2), 0.0))                      # AdaptiveAvgPool1d(1) then ReLU
    feat = np.stack(feats, axis=2)                                         # [B, C, 3]
    wc = p[f"{prefix}.feature_concate_fc.weight"].astype(x.dtype)
    bc = p[f"{prefix}.feature_concate_fc.bias"].astype(x.dtype)
    sq = feat @ wc[0] + bc[0]                                              # [B, C]
    f1 = np.maximum(sq @ p[f"{prefix}.fc1.weight"].astype(x.dtype).T + p[f"{prefix}.fc1.bias"].astype(x.dtype), 0.0)
    f2 = sigmoid(f1 @ p[f"{prefix}.fc2.weight"].astype(x.dtype).T + p[f"{prefix}.fc2.bias"].astype(x.dtype))
    return x * f2[:, :, None]


def se_layer(x, p, prefix):
    """ChannelSELayer.forward (attention_model.py:25-40)."""
    sq = x.mean(axis=2)
    f1 = np.maximum(sq @ p[f"{prefix}.fc1.weight"].astype(x.dtype).T + p[f"{prefix}.fc1.bias"].astype(x.dtype), 0.0)
    g = sigmoid(f1 @ p[f"{prefix}.fc2.weight"].astype(x.dtype).T + p[f"{prefix}.fc2.bias"].astype(x.dtype))
    return x * g[:, :, None]


def cbam_layer(x, p, prefix):
    """ChannelCBAMLayer.forward (attention_model.py:317-334)."""
    w1, b1 = p[f"{prefix}.fc1.weight"].astype(x.dtype), p[f"{prefix}.fc1.bias"].astype(x.dtype)
    f1 = np.maximum(x.mean(axis=2) @ w1.T + b1, 0.0) + np.maximum(x.max(axis=2) @ w1.T + b1, 0.0)
    g = sigmoid(f1 @ p[f"{prefix}.fc2.weight"].astype(x.dtype).T + p[f"{prefix}.fc2.bias"].astype(x.dtype))
    return x * g[:, :, None]


def eca_layer(x, p, prefix):
    """ChannelECAlayer.forward (attention_model.py:349-359): conv1d over the channel axis, k = 3, zero padding 1, no bias."""
    w = p[f"{prefix}.conv.weight"].astype(x.dtype).reshape(-1)
    y = np.pad(x.mean(axis=2), ((0, 0), (1, 1)))
    g = sigmoid(w[0] * y[:, :-2] + w[1] * y[:, 1:-1] + w[2] * y[:, 2:])
    return x * g[:, :, None]


def channel_attention(x, p, prefix, cfg):
    """Dispatch of fullsubnet_plus.py:52-70."""
    kind = cfg.get("channel_attention_model", "TSSE")
    if kind == "TSSE":
        return tsse(x, p, prefix, cfg["kersize"])
    return {"SE": se_layer, "CBAM": cbam_layer, "ECA": eca_layer}[kind](x, p, prefix)


def prelu(x, a):
    return np.where(x >= 0, x, a * x)


def gln(x, g, b):
    """nn.GroupNorm(1, C, eps=1e-8): statistics over (C, T) per sample (causal_conv.py:73,79)."""
    mu = x.mean(axis=(1, 2), keepdims=True)
    var = x.var(axis=(1, 2), keepdims=True)
    return (x - mu) / np.sqrt(var + GLN_EPS) * g[None, :, None] + b[None, :, None]


def tcn_block(x, p, q, d, causal=False):
    """TCNBlock.forward with the skip connection (causal_conv.py:96-108).  x [B, C, T].  causal=False (what SequenceModel builds,
    sequence_model.py:47-58): symmetric zero padding d, taps t-d, t, t+d.  causal=True (causal_conv.py:74-75,104-105): padding 2d
    on both sides and the last 2d outputs chomped, i.e. taps t-2d, t-d, t."""
    dt = x.dtype
    w1 = p[f"{q}.conv1x1.weight"].astype(dt)[:, :, 0]
    y = np.einsum("oc,bct->bot", w1, x) + p[f"{q}.conv1x1.bias"].astype(dt)[None, :, None]
    y = gln(prelu(y, p[f"{q}.prelu1.weight"].astype(dt)[0]),
            p[f"{q}.norm1.weight"].astype(dt), p[f"{q}.norm1.bias"].astype(dt))
    T = y.shape[2]
    yp = np.pad(y, ((0, 0), (0, 0), (2 * d, 0) if causal else (d, d)))     # zeros; causal: left 2d (right pad + chomp cancel)
    wd = p[f"{q}.depthwise_conv.weight"].astype(dt)[:, 0, :]
    z = np.zeros_like(y)
    for j in range(3):
        z += wd[None, :, j, None] * yp[:, :, j * d:j * d + T]
    z += p[f"{q}.depthwise_conv.bias"].astype(dt)[None, :, None]
    z = gln(prelu(z, p[f"{q}.prelu2.weight"].astype(dt)[0]),
            p[f"{q}.norm2.weight"].astype(dt), p[f"{q}.norm2.bias"].astype(dt))
    w2 = p[f"{q}.sconv.weight"].astype(dt)[:, :, 0]
    o = np.einsum("oc,bct->bot", w2, z) + p[f"{q}.sconv.bias"].astype(dt)[None, :, None]
    return x + o


def activation(x, name):
    """sequence_model.py:84-93."""
    if not name:
        return x
    if name == "Tanh":
        return np.tanh(x)
    if name == "ReLU":
        return np.maximum(x, 0.0)
    if name == "ReLU6":
        return np.clip(x, 0.0, 6.0)
    raise NotImplementedError(name)


def seq_tcn(x, p, prefix, act, causal=False):
    """SequenceModel.forward, TCN branch (sequence_model.py:106-112).  x [B, F, T]."""
    for i, d in enumerate(TCN_DILATIONS):
        x = tcn_block(x, p, f"{prefix}.sequence_model.{i}", d, causal)
    x = np.maximum(x, 0.0)                                                  # nn.ReLU at sequence_model.py:57
    w = p[f"{prefix}.fc_output_layer.weight"].astype(x.dtype)
    b = p[f"{prefix}.fc_output_layer.bias"].astype(x.dtype)
    o = np.einsum("of,bft->bot", w, x) + b[None, :, None]                   # Linear over F on [B, T, F]
    return activation(o, act)


def lstm_stack(x, p, prefix, num_layers, return_all=False):
    """nn.LSTM(batch_first) as used at sequence_model.py:118: gate rows i,f,g,o;
    c_t = s(f) c + s(i) tanh(g); h_t = s(o) tanh(c_t); zero initial state.  x [N, T, I] -> [N, T, H]."""
    dt = x.dtype
    N, T, _ = x.shape
    inp = x
    for l in range(num_layers):
        # (per-step small GEMMs: one big [N*T, K] GEMM is an order of magnitude slower on this OpenBLAS build)
        wiT = np.ascontiguousarray(p[f"{prefix}.sequence_model.weight_ih_l{l}"].astype(dt).T)
        whT = np.ascontiguousarray(p[f"{prefix}.sequence_model.weight_hh_l{l}"].astype(dt).T)
        b = (p[f"{prefix}.sequence_model.bias_ih_l{l}"].astype(dt)
             + p[f"{prefix}.sequence_model.bias_hh_l{l}"].astype(dt))
        H = whT.shape[0]
        h = np.zeros((N, H), dt); c = np.zeros((N, H), dt)
        out = np.empty((N, T, H), dt)
        inp_t = np.ascontiguousarray(inp.transpose(1, 0, 2))                # [T, N, K]
        for t in range(T):
            g = inp_t[t] @ wiT + h @ whT + b
            i_, f_, g_, o_ = g[:, :H], g[:, H:2 * H], g[:, 2 * H:3 * H], g[:, 3 * H:]
            c = sigmoid(f_) * c + sigmoid(i_) * np.tanh(g_)
            h = sigmoid(o_) * np.tanh(c)
            out[:, t] = h
        inp = out
    return inp


def gru_stack(x, p, prefix, num_layers):
    """nn.GRU(batch_first) as built at sequence_model.py:39-46: gate rows r,z,n;
    n = tanh(W_in x + b_in + r (W_hn h + b_hn)); h_t = (1 - z) n + z h; zero initial state.  x [N, T, I] -> [N, T, H]."""
    dt = x.dtype
    N, T, _ = x.shape
    inp = x
    for l in range(num_layers):
        wiT = np.ascontiguousarray(p[f"{prefix}.sequence_model.weight_ih_l{l}"].astype(dt).T)
        whT = np.ascontiguousarray(p[f"{prefix}.sequence_model.weight_hh_l{l}"].astype(dt).T)
        bi = p[f"{prefix}.sequence_model.bias_ih_l{l}"].astype(dt)
        bh = p[f"{prefix}.sequence_model.bias_hh_l{l}"].astype(dt)
        H = whT.shape[0]
        h = np.zeros((N, H), dt)
        out = np.empty((N, T, H), dt)
        inp_t = np.ascontiguousarray(inp.transpose(1, 0, 2))
        for t in range(T):
            gi = inp_t[t] @ wiT + bi
            gh = h @ whT + bh
            r = sigmoid(gi[:, :H] + gh[:, :H])
            z = sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            n = np.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
            h = (1.0 - z) * n + z * h
            out[:, t] = h
        inp = out
    return inp


def seq_lstm(x, p, prefix, num_layers, act, kind="LSTM"):
    """SequenceModel.forward, LSTM / GRU branch (sequence_model.py:113-122).  x [N, I, T] -> [N, O, T]."""
    o = (gru_stack if kind == "GRU" else lstm_stack)(x.transpose(0, 2, 1), p, prefix, num_layers)
    w = p[f"{prefix}.fc_output_layer.weight"].astype(x.dtype)
    b = p[f"{prefix}.fc_output_layer.bias"].astype(x.dtype)
    o = activation(o @ w.T + b, act)
    return o.transpose(0, 2, 1)


# ----------------------------------------------------------------------------
# model forwards (eval path: drop_band bypassed, SURVEY.md 0.4)
# ----------------------------------------------------------------------------

def fullsubnet_plus_forward(p, cfg, mag, real, imag, dtype=np.float64, num_layers=2, stages=None):
    """FullSubNet_Plus.forward (fullsubnet_plus.py:122-209), one call per batch
    with every sample treated independently (== the reference called with B=1
    per sample).  Inputs [B, 1, F, T]; returns [B, 2, F, T].  ``stages`` (dict)
    receives the intermediate tensors the kernel-level tests compare against."""
    sub = cfg.get("subband_num", 1)
    # the reference forward itself raises for subband_num > 1 with TSSE / SE / CBAM (the real / imag attentions are built for
    # F // subband_num + 1 channels but applied to F, fullsubnet_plus.py:47-50,157-163); only the channel-agnostic ECA runs
    assert sub == 1 or cfg.get("channel_attention_model", "TSSE") == "ECA"
    la, ns, nfb = cfg["look_ahead"], cfg["sb_num_neighbors"], cfg["fb_num_neighbors"]
    norm = NORMS[cfg["norm_type"]]
    pad = lambda x: np.pad(np.asarray(x, dtype), ((0, 0), (0, 0), (0, 0), (0, la)))     # :137-139
    mag, real, imag = pad(mag), pad(real), pad(imag)
    B, C, F, T = mag.shape
    assert C == 1
    fb_in, fb_out = [], []
    for x, s in ((mag, ""), (real, "_real"), (imag, "_imag")):
        if sub > 1 and s == "":                                                         # :146-153, mag branch only
            pn = sub - F % sub                                                          # (a whole extra group when F % sub == 0)
            xi = np.pad(norm(x), ((0, 0), (0, 0), (0, pn), (0, 0)), mode="reflect").reshape(B, (F + pn) // sub, T * sub)
            xi = channel_attention(xi, p, "channel_attention", cfg).reshape(B, F + pn, T)[:, :F]
        else:
            xi = norm(x).reshape(B, F, T)                                               # :144,157,162
            xi = channel_attention(xi, p, f"channel_attention{s}", cfg)                     # :145,158,163
        fb_in.append(xi)
        fb_out.append(seq_tcn(xi, p, f"fb_model{s}", cfg["fb_output_activate_function"], cfg.get("causal_tcn", False))
                      .reshape(B, 1, F, T))                                             # :154,159,164
    unf = [unfold(o, nfb).reshape(B, F, 2 * nfb + 1, T) for o in fb_out]                 # :167-179
    mag_unf = unfold(fb_in[0].reshape(B, 1, F, T), ns).reshape(B, F, 2 * ns + 1, T)      # :182-185
    sb_in = norm(np.concatenate([mag_unf] + unf, axis=2))                                # :188-189
    if stages is not None:
        stages.update(fb_in=np.stack(fb_in), fb_out=np.stack([o[:, 0] for o in fb_out]), sb_in=sb_in)
    Isb = sb_in.shape[2]
    m = seq_lstm(sb_in.reshape(B * F, Isb, T), p, "sb_model", num_layers,
                 cfg["sb_output_activate_function"], cfg.get("sequence_model", "LSTM"))  # :205
    O = m.shape[1]
    m = m.reshape(B, F, O, T).transpose(0, 2, 1, 3)                                      # :206
    return np.ascontiguousarray(m[:, :, :, la:])                                         # :208


def fullsubnet_forward(p, cfg, mag, dtype=np.float64, num_layers=2, stages=None):
    """fullsubnet Model.forward (fullsubnet.py:68-118), eval path, per-sample semantics."""
    la, ns, nfb = cfg["look_ahead"], cfg["sb_num_neighbors"], cfg["fb_num_neighbors"]
    norm = NORMS[cfg["norm_type"]]
    mag = np.pad(np.asarray(mag, dtype), ((0, 0), (0, 0), (0, 0), (0, la)))              # :81
    B, C, F, T = mag.shape
    assert C == 1
    fb_in = norm(mag).reshape(B, F, T)                                                   # :86
    fb_out = seq_lstm(fb_in, p, "fb_model", num_layers,
                      cfg["fb_output_activate_function"], cfg.get("sequence_model", "LSTM")).reshape(B, 1, F, T)   # :87
    fb_unf = unfold(fb_out, nfb).reshape(B, F, 2 * nfb + 1, T)                           # :90-91
    mag_unf = unfold(mag, ns).reshape(B, F, 2 * ns + 1, T)                               # :94-95 (raw mag)
    sb_in = norm(np.concatenate([mag_unf, fb_unf], axis=2))                              # :98-99
    if stages is not None:
        stages.update(fb_in=fb_in, fb_out=fb_out[:, 0], sb_in=sb_in)
    Isb = sb_in.shape[2]
    m = seq_lstm(sb_in.reshape(B * F, Isb, T), p, "sb_model", num_layers,
                 cfg["sb_output_activate_function"], cfg.get("sequence_model", "LSTM"))  # :114
    m = m.reshape(B, F, 2, T).transpose(0, 2, 1, 3)                                      # :115
    return np.ascontiguousarray(m[:, :, :, la:])                                         # :117


def rel_l2(y, ref):
    y = np.asarray(y, np.float64); ref = np.asarray(ref, np.float64)
    return float(np.linalg.norm(y - ref) / (np.linalg.norm(ref) + 1e-300))


# ----------------------------------------------------------------------------
# algorithmic work (SURVEY.md 8d formula)
# ----------------------------------------------------------------------------

def flops_plus(cfg, T_in, num_layers=2):
    F = cfg["num_freqs"]; Tp = T_in + cfg["look_ahead"]
    H = cfg["sb_model_hidden_size"]
    I = (2 * cfg["sb_num_neighbors"] + 1) + 3 * (2 * cfg["fb_num_neighbors"] + 1)
    O = cfg.get("output_size", 2)
    sb = Tp * F * (2 * 4 * H * (I + H) + (num_layers - 1) * 2 * 4 * H * 2 * H + 2 * H * O)
    tcn = 3 * Tp * (8 * (2 * 2 * F * TCN_HIDDEN + 2 * 3 * TCN_HIDDEN) + 2 * F * F)
    ts = 3 * (2 * F * sum(cfg["kersize"]) * Tp + 4 * F * (F // 2))
    return dict(subband=sb, fullband=tcn, tsse=ts, total=sb + tcn + ts)


def flops_fsn(cfg, T_in, num_layers=2):
    F = cfg["num_freqs"]; Tp = T_in + cfg["look_ahead"]
    H = cfg["sb_model_hidden_size"]; Hf = cfg["fb_model_hidden_size"]
    I = (2 * cfg["sb_num_neighbors"] + 1) + (2 * cfg["fb_num_neighbors"] + 1)
    sb = Tp * F * (2 * 4 * H * (I + H) + (num_layers - 1) * 2 * 4 * H * 2 * H + 2 * H * 2)
    fb = Tp * (2 * 4 * Hf * (F + Hf) + (num_layers - 1) * 2 * 4 * Hf * 2 * Hf + 2 * Hf * F)
    return dict(subband=sb, fullband=fb, tsse=0, total=sb + fb)
