"""Test infrastructure for FullSubNet+ with a TCN sub-band model (sequence_model = "TCN", reference fullsubnet_plus.py:45,102-110).

The pinned oracles (oracle/fsn_oracle.py, oracle/torch_port.py) cover the LSTM / GRU sub-band models; this module adds the TCN one on
top of their building blocks, without changing them:
  * make_params       -- state_dict of FullSubNet_Plus(sequence_model="TCN"): fsn_oracle's attention and full-band draws, then the
                         sub-band TCN's 8 blocks of hidden width 512 over Isb channels and Linear(Isb -> output_size);
  * forward           -- numpy fp64 forward (fullsubnet_plus.py:122-209 with SequenceModel("TCN") as the sub-band model);
  * flops             -- the sub-band TCN's algorithmic work per clip;
  * TcnPort           -- the CPU torch port with the sub-band TCN, run in chunks of sequences.
Pinned by tests/golden/plus_{small,default}_sbTCN.npz, generated from the unmodified reference by
tests/golden/make_golden_sbtcn.py.  Line references are to speech_enhance/ of the reference.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import fsn_oracle as O
from oracle.torch_port import TorchPort

HIDDEN = O.TCN_HIDDEN


def isb(cfg):
    return (2 * cfg["sb_num_neighbors"] + 1) + 3 * (2 * cfg["fb_num_neighbors"] + 1)


def make_params(cfg, seed=0, scale=1.0):
    """state_dict of FullSubNet_Plus(**cfg, sequence_model="TCN") (fullsubnet_plus.py:52-110; sb_model_hidden_size and num_layers are
    unused, like in the reference).  ``scale`` multiplies the bounds of the sub-band TCN's two 1x1 convolutions (the analogue of
    fsn_oracle's ``lstm_scale`` stress variant)."""
    rng = np.random.default_rng(seed)
    nf = cfg["num_freqs"]
    p = {}
    for s in ("", "_real", "_imag"):
        p.update(O._attn_params(rng, f"channel_attention{s}", nf, cfg))
    for s in ("", "_real", "_imag"):
        p.update(O._tcn_params(rng, f"fb_model{s}", nf))
    c, out = isb(cfg), cfg.get("output_size", 2)
    for i in range(8):                                       # keys / shapes of TCNBlock, causal_conv.py:67-80
        q = f"sb_model.sequence_model.{i}"
        p[f"{q}.conv1x1.weight"] = O._uni(rng, (HIDDEN, c, 1), scale / np.sqrt(c))
        p[f"{q}.conv1x1.bias"] = O._uni(rng, (HIDDEN,), scale / np.sqrt(c))
        p[f"{q}.prelu1.weight"] = np.array([0.25 + 0.02 * i], np.float32)
        p[f"{q}.norm1.weight"] = (1 + 0.1 * rng.standard_normal(HIDDEN)).astype(np.float32)
        p[f"{q}.norm1.bias"] = (0.1 * rng.standard_normal(HIDDEN)).astype(np.float32)
        p[f"{q}.depthwise_conv.weight"] = O._uni(rng, (HIDDEN, 1, 3), 1 / np.sqrt(3))
        p[f"{q}.depthwise_conv.bias"] = O._uni(rng, (HIDDEN,), 1 / np.sqrt(3))
        p[f"{q}.prelu2.weight"] = np.array([0.2 + 0.01 * i], np.float32)
        p[f"{q}.norm2.weight"] = (1 + 0.1 * rng.standard_normal(HIDDEN)).astype(np.float32)
        p[f"{q}.norm2.bias"] = (0.1 * rng.standard_normal(HIDDEN)).astype(np.float32)
        p[f"{q}.sconv.weight"] = O._uni(rng, (c, HIDDEN, 1), scale / np.sqrt(HIDDEN))
        p[f"{q}.sconv.bias"] = O._uni(rng, (c,), scale / np.sqrt(HIDDEN))
    p["sb_model.fc_output_layer.weight"] = O._uni(rng, (out, c), 1 / np.sqrt(c))      # sequence_model.py:80-81
    p["sb_model.fc_output_layer.bias"] = O._uni(rng, (out,), 1 / np.sqrt(c))
    return p


def forward(p, cfg, mag, real, imag, dtype=np.float64, stages=None):
    """FullSubNet_Plus.forward (fullsubnet_plus.py:122-209) with the sub-band TCN, every sample independent.  Inputs [B, 1, F, T];
    returns [B, O, F, T].  The front end is fsn_oracle's; the sub-band model is SequenceModel("TCN") (sequence_model.py:106-112),
    never causal (SequenceModel does not pass ``causal``).  ``stages`` receives fb_in, fb_out and sb_in."""
    sub = cfg.get("subband_num", 1)
    assert sub == 1 or cfg.get("channel_attention_model", "TSSE") == "ECA"
    la, ns, nfb = cfg["look_ahead"], cfg["sb_num_neighbors"], cfg["fb_num_neighbors"]
    norm = O.NORMS[cfg["norm_type"]]
    pad = lambda x: np.pad(np.asarray(x, dtype), ((0, 0), (0, 0), (0, 0), (0, la)))     # :137-139
    mag, real, imag = pad(mag), pad(real), pad(imag)
    B, _, Fq, T = mag.shape
    fb_in, fb_out = [], []
    for x, s in ((mag, ""), (real, "_real"), (imag, "_imag")):
        if sub > 1 and s == "":                                                         # :146-153, mag branch only
            pn = sub - Fq % sub
            xi = np.pad(norm(x), ((0, 0), (0, 0), (0, pn), (0, 0)), mode="reflect").reshape(B, (Fq + pn) // sub, T * sub)
            xi = O.channel_attention(xi, p, "channel_attention", cfg).reshape(B, Fq + pn, T)[:, :Fq]
        else:
            xi = O.channel_attention(norm(x).reshape(B, Fq, T), p, f"channel_attention{s}", cfg)    # :144-145,157-163
        fb_in.append(xi)
        fb_out.append(O.seq_tcn(xi, p, f"fb_model{s}", cfg["fb_output_activate_function"], cfg.get("causal_tcn", False))
                      .reshape(B, 1, Fq, T))                                            # :154,159,164
    unf = [O.unfold(o, nfb).reshape(B, Fq, 2 * nfb + 1, T) for o in fb_out]              # :167-179
    win = O.unfold(fb_in[0].reshape(B, 1, Fq, T), ns).reshape(B, Fq, 2 * ns + 1, T)       # :182-185
    sb_in = norm(np.concatenate([win] + unf, axis=2))                                    # :188-189
    if stages is not None:
        stages.update(fb_in=np.stack(fb_in), fb_out=np.stack([o[:, 0] for o in fb_out]), sb_in=sb_in)
    m = O.seq_tcn(sb_in.reshape(B * Fq, sb_in.shape[2], T), p, "sb_model", cfg["sb_output_activate_function"])   # :205
    m = m.reshape(B, Fq, -1, T).transpose(0, 2, 1, 3)                                    # :206
    return np.ascontiguousarray(m[:, :, :, la:])                                         # :208


def flops(cfg, T_in):
    """Algorithmic work of the sub-band TCN per clip: T' F [8 (2 * 2 Isb 512 + 2 * 3 * 512) + 2 Isb O]."""
    Tp = T_in + cfg["look_ahead"]
    c, o = isb(cfg), cfg.get("output_size", 2)
    return Tp * cfg["num_freqs"] * (8 * (2 * 2 * c * HIDDEN + 2 * 3 * HIDDEN) + 2 * c * o)


class TcnPort(TorchPort):
    """oracle.torch_port.TorchPort (the reference's ATen op sequence, one clip per call) with the sub-band TCN in place of the LSTM.
    The sub-band sequences are processed in chunks: each is independent (GroupNorm(1, 512) normalises each one on its own), and one
    fp32 hidden tensor of all of them is 512 / Isb times larger than the input."""

    def __init__(self, params, cfg, dtype=torch.float32, chunk=32):
        self.p = {k: torch.from_numpy(v).to(dtype) for k, v in params.items()}
        self.cfg, self.kind, self.L, self.dtype, self.lstm, self.chunk = cfg, "plus", 2, dtype, {}, chunk

    def _sb_tcn(self, x):                                    # sequence_model.py:106-112, causal_conv.py:96-108 (non-causal)
        p = self.p
        for i, d in enumerate(O.TCN_DILATIONS):
            q = f"sb_model.sequence_model.{i}"
            y = F.conv1d(x, p[f"{q}.conv1x1.weight"], p[f"{q}.conv1x1.bias"])
            y = F.group_norm(F.prelu(y, p[f"{q}.prelu1.weight"]), 1, p[f"{q}.norm1.weight"], p[f"{q}.norm1.bias"], 1e-8)
            y = F.conv1d(y, p[f"{q}.depthwise_conv.weight"], p[f"{q}.depthwise_conv.bias"], padding=d, dilation=d, groups=y.shape[1])
            y = F.group_norm(F.prelu(y, p[f"{q}.prelu2.weight"]), 1, p[f"{q}.norm2.weight"], p[f"{q}.norm2.bias"], 1e-8)
            x = x + F.conv1d(y, p[f"{q}.sconv.weight"], p[f"{q}.sconv.bias"])
        o = F.linear(F.relu(x).permute(0, 2, 1), p["sb_model.fc_output_layer.weight"], p["sb_model.fc_output_layer.bias"])
        return self.act(o, self.cfg["sb_output_activate_function"]).permute(0, 2, 1)

    def seq_lstm(self, x, pre, actname):                     # TorchPort.forward calls this for the sub-band model only (kind "plus")
        assert pre == "sb_model"
        return torch.cat([self._sb_tcn(x[i:i + self.chunk]) for i in range(0, x.shape[0], self.chunk)], dim=0).contiguous()
