"""PyTorch-CPU restatement of the reference forward, used ONLY as the timed CPU baseline.

TEST/BENCH INFRASTRUCTURE ONLY (see oracle/__init__.py).  The reference is pure Python on top of PyTorch and
may be absent where the benchmark runs (oracle/_ref/ is only made from a checkout of it), so bench.py's ``cpu_baseline`` leg and
``--impl reference`` arm time this port instead: it issues the SAME ATen operators the reference issues
(nn.LSTM, F.conv1d, F.group_norm, F.prelu, F.linear, F.pad(reflect) + F.unfold) in the same order, fp32,
one sample per call (the only batch size the reference inference supports, base_inferencer.py:65-69), with all
host threads.  Parity status: PINNED -- tests/test_oracle_golden.py checks it against the golden vectors
generated from the unmodified reference.  Line references are to speech_enhance/ of the reference.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

TCN_DILATIONS = (1, 2, 5, 9, 1, 2, 5, 9)


class TorchPort:
    def __init__(self, params, cfg, kind="plus", num_layers=2, dtype=torch.float32):
        self.p = {k: torch.from_numpy(v).to(dtype) for k, v in params.items()}
        self.cfg, self.kind, self.L, self.dtype = cfg, kind, num_layers, dtype
        self.lstm = {}
        for pre in (("sb_model",) if kind == "plus" else ("fb_model", "sb_model")):
            wi = self.p[f"{pre}.sequence_model.weight_ih_l0"]
            m = nn.LSTM(wi.shape[1], wi.shape[0] // 4, num_layers, batch_first=True).to(dtype)
            m.load_state_dict({k.split("sequence_model.")[1]: v for k, v in self.p.items()
                               if k.startswith(pre + ".sequence_model.")})
            self.lstm[pre] = m.eval()

    def norm(self, x):                              # base_model.py:318-330 (norm_wrapper) on [B, C, F, T]
        kind = self.cfg.get("norm_type", "offline_laplace_norm")
        if kind == "offline_laplace_norm":          # :210-225
            return x / (x.mean(dim=(1, 2, 3), keepdim=True) + 1e-5)
        if kind == "offline_gaussian_norm":         # :260-275
            return (x - x.mean(dim=(1, 2, 3), keepdim=True)) / (x.std(dim=(1, 2, 3), keepdim=True) + 1e-5)
        B, C, Fq, T = x.shape
        eps = torch.finfo(torch.float32).eps        # audio_zen/constant.py:8
        xr = x.reshape(B * C, Fq, T)
        cnt = torch.arange(Fq, Fq * T + 1, Fq, dtype=x.dtype).reshape(1, T)
        csum = torch.cumsum(xr.sum(dim=1), dim=-1)
        cmean = csum / cnt
        if kind == "cumulative_laplace_norm":       # :227-258
            return (xr / (cmean.reshape(B * C, 1, T) + eps)).reshape(B, C, Fq, T)
        if kind == "cumulative_layer_norm":         # :277-316
            cpow = torch.cumsum((xr * xr).sum(dim=1), dim=-1)
            cstd = torch.sqrt((cpow - 2 * cmean * csum) / cnt + cmean ** 2 + eps)
            return ((xr - cmean[:, None, :]) / cstd[:, None, :]).reshape(B, C, Fq, T)
        raise NotImplementedError(kind)

    @staticmethod
    def unfold(x, n):                               # base_model.py:15-47
        B, C, Fq, T = x.shape
        if n < 1:
            return x.permute(0, 2, 1, 3).reshape(B, Fq, C, 1, T)
        o = F.pad(x.reshape(B * C, 1, Fq, T), [0, 0, n, n], mode="reflect")
        o = F.unfold(o, (2 * n + 1, T))
        return o.reshape(B, C, 2 * n + 1, T, Fq).permute(0, 4, 1, 2, 3).contiguous()

    def tsse(self, x, pre):                         # attention_model.py:78-98
        p, C = self.p, x.shape[1]
        feats = [F.relu(F.conv1d(x, p[f"{pre}.{n}.0.weight"], p[f"{pre}.{n}.0.bias"], groups=C).mean(dim=2, keepdim=True))
                 for n in ("smallConv1d", "middleConv1d", "largeConv1d")]
        sq = F.linear(torch.cat(feats, dim=2), p[f"{pre}.feature_concate_fc.weight"], p[f"{pre}.feature_concate_fc.bias"])[..., 0]
        g = torch.sigmoid(F.linear(F.relu(F.linear(sq, p[f"{pre}.fc1.weight"], p[f"{pre}.fc1.bias"])),
                                   p[f"{pre}.fc2.weight"], p[f"{pre}.fc2.bias"]))
        return x * g[:, :, None]

    def tcn(self, x, pre):                          # sequence_model.py:106-112, causal_conv.py:96-108
        p = self.p
        for i, d in enumerate(TCN_DILATIONS):
            q = f"{pre}.sequence_model.{i}"
            y = F.conv1d(x, p[f"{q}.conv1x1.weight"], p[f"{q}.conv1x1.bias"])
            y = F.group_norm(F.prelu(y, p[f"{q}.prelu1.weight"]), 1, p[f"{q}.norm1.weight"], p[f"{q}.norm1.bias"], 1e-8)
            if self.cfg.get("causal_tcn", False):       # TCNBlock(causal=True): padding 2d, chomp 2d (causal_conv.py:74-75,104-105)
                y = F.conv1d(y, p[f"{q}.depthwise_conv.weight"], p[f"{q}.depthwise_conv.bias"], padding=2 * d, dilation=d, groups=y.shape[1])[:, :, :-2 * d]
            else:
                y = F.conv1d(y, p[f"{q}.depthwise_conv.weight"], p[f"{q}.depthwise_conv.bias"], padding=d, dilation=d, groups=y.shape[1])
            y = F.group_norm(F.prelu(y, p[f"{q}.prelu2.weight"]), 1, p[f"{q}.norm2.weight"], p[f"{q}.norm2.bias"], 1e-8)
            x = x + F.conv1d(y, p[f"{q}.sconv.weight"], p[f"{q}.sconv.bias"])
        o = F.linear(F.relu(x).permute(0, 2, 1), p[f"{pre}.fc_output_layer.weight"], p[f"{pre}.fc_output_layer.bias"])
        return self.act(o, self.cfg["fb_output_activate_function"]).permute(0, 2, 1)

    @staticmethod
    def act(o, name):                               # sequence_model.py:84-93
        return {None: o, False: o, "ReLU": F.relu(o), "Tanh": torch.tanh(o), "ReLU6": F.relu6(o)}[name]

    def seq_lstm(self, x, pre, actname):            # sequence_model.py:113-122
        xt = x.permute(0, 2, 1).contiguous()
        if xt.shape[1] <= 512:
            o, _ = self.lstm[pre](xt)
        else:                                       # long clips: same recurrence in time chunks with the state carried (ATen's CPU
            outs, st = [], None                     # LSTM slows down super-linearly with the sequence length)
            for t0 in range(0, xt.shape[1], 256):
                oc, st = self.lstm[pre](xt[:, t0:t0 + 256].contiguous(), st)
                outs.append(oc)
            o = torch.cat(outs, dim=1)
        o = self.act(F.linear(o, self.p[f"{pre}.fc_output_layer.weight"], self.p[f"{pre}.fc_output_layer.bias"]), actname)
        return o.permute(0, 2, 1).contiguous()

    @torch.no_grad()
    def forward(self, mag, real=None, imag=None):
        """One sample per call ([1, 1, F, T] tensors), like the reference inferencer."""
        c = self.cfg
        la, ns, nfb = c["look_ahead"], c["sb_num_neighbors"], c["fb_num_neighbors"]
        pad = lambda x: F.pad(x.to(self.dtype), [0, la])
        mag = pad(mag)
        B, _, Fq, T = mag.shape
        if self.kind == "plus":                     # fullsubnet_plus.py:122-209
            fb_in, outs = None, []
            for x, s in ((mag, ""), (pad(real), "_real"), (pad(imag), "_imag")):
                xi = self.tsse(self.norm(x).reshape(B, Fq, T), "channel_attention" + s)
                if s == "":
                    fb_in = xi
                outs.append(self.unfold(self.tcn(xi, "fb_model" + s).reshape(B, 1, Fq, T), nfb).reshape(B, Fq, 2 * nfb + 1, T))
            win = self.unfold(fb_in.reshape(B, 1, Fq, T), ns).reshape(B, Fq, 2 * ns + 1, T)
        else:                                       # fullsubnet.py:68-118
            fb = self.seq_lstm(self.norm(mag).reshape(B, Fq, T), "fb_model", c["fb_output_activate_function"]).reshape(B, 1, Fq, T)
            outs = [self.unfold(fb, nfb).reshape(B, Fq, 2 * nfb + 1, T)]
            win = self.unfold(mag, ns).reshape(B, Fq, 2 * ns + 1, T)
        sb = self.norm(torch.cat([win] + outs, dim=2))
        m = self.seq_lstm(sb.reshape(B * Fq, sb.shape[2], T), "sb_model", c["sb_output_activate_function"])
        m = m.reshape(B, Fq, -1, T).permute(0, 2, 1, 3).contiguous()
        return m[:, :, :, la:]
