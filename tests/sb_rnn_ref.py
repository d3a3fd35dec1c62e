"""fp64 references of the sub-band LSTM / GRU stage alone, and the element-wise rule the kernels are held to.

The stage is sb_model of the reference: nn.LSTM / nn.GRU (batch_first) -> Linear(H -> 2) -> output activation, the first
look_ahead frames dropped (sequence_model.py:113-122, fullsubnet_plus.py:200-208).  Both references read the model's own
state_dict (<prefix>.sequence_model.*, <prefix>.fc_output_layer.*), so the parameter packing is under test as well.  With
prefix="fb_model", head="fb" they check the full-band LSTM / GRU of fullsubnet.Model instead (fullsubnet.py:86-87): Linear(H -> F) +
fb_output_activate_function on every frame (conv1x1_tf32_kernel, k_front.cu), no look-ahead drop.

* truth():   torch.nn.LSTM / torch.nn.GRU in float64.
* emulate(): the same recurrence in float64, rounded where the kernels round: W_ih and W_hh to fp16, h to fp16 after every step,
             the input projection Gin of layers >= 1 to fp16 (the GEMM's fp16 output), the carried c (GRU: h) to fp32.  Its distance
             from truth() on the same elements is the error the kernels' number formats make unavoidable.  Full band: fb_pack
             (k_front.cu) rounds the fp32 input to fp16 first, Gin of the deeper layers stays in fp32 (k_lstm_ws.cu and lstm_mma_kernel
             accumulate it with the recurrent product), and the head reads the top layer's fp32 h (hseq), both operands rounded to
             tf32 (cvt.rna) by conv1x1_tf32_kernel.  ``fault`` plants one of
             the bugs the rule must catch (test_sb_recurrence_cpu.py).

Rule (compare()): err = |kernel - truth| per element; max err <= factor * (3 max |emulation - truth| + 1e-6 RMS), factor = 1 for
accurate gate math, FAST_FACTOR for fast math (tanh.approx, which the emulation does not model).
"""
import numpy as np
import torch

import tcn_ref

# Fast-math gates (tanh.approx, max rel. error 2^-11) on top of the fp16 rounding the emulation models: the accurate bound is
# multiplied by this factor.  Measured once on one H100 80GB HBM3 SXM (700 W power limit): the kernels' max err reached at most 1.15x
# the emulation's over every fast-math case of tests/test_gpu_sb_recurrence.py.
FAST_FACTOR = 1.5
ACCURATE_MULT = 3.0
FLOOR = 1e-6

FAULTS = ("swap_units", "c_reset", "h_lag", "row_c_drop", "gru_bias_fold")


def _act(y, act):
    if act in (None, False, "", "none"):
        return y
    if act == "ReLU":
        return torch.relu(y)
    if act == "Tanh":
        return torch.tanh(y)
    if act == "ReLU6":
        return torch.clamp(y, 0.0, 6.0)
    raise ValueError(act)


def _sd(sd, key, device):
    v = sd[key]
    v = v.detach().cpu() if isinstance(v, torch.Tensor) else torch.from_numpy(np.asarray(v))
    return v.to(device=device, dtype=torch.float64)


def num_layers(sd, prefix="sb_model"):
    return sum(1 for k in sd if k.startswith(f"{prefix}.sequence_model.weight_ih_l"))


def layers(sd, device="cpu", prefix="sb_model"):
    """[(w_ih, w_hh, b_ih, b_hh)] per layer, float64, reference (nn.LSTM / nn.GRU) layout."""
    p = f"{prefix}.sequence_model."
    return [tuple(_sd(sd, f"{p}{n}_l{l}", device) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
            for l in range(num_layers(sd, prefix))]


def _head(sd, y, look_ahead, act, device, prefix="sb_model", head="sb", tf32=False):
    """y: [N, Tp, H] -> act(Linear(y)), as [N, O, Tp - look_ahead] (head "sb": the first look_ahead frames dropped) or [N, O, Tp]
    (head "fb").  tf32: both operands rounded as cvt.rna.tf32 does (the full band's conv1x1_tf32_kernel)."""
    w, b = _sd(sd, f"{prefix}.fc_output_layer.weight", device), _sd(sd, f"{prefix}.fc_output_layer.bias", device)
    if head == "fb":
        look_ahead = 0
    elif head != "sb":
        raise ValueError(head)
    y = y[:, look_ahead:]
    if tf32:
        y, w = tcn_ref.round_tf32_away(y), tcn_ref.round_tf32_away(w)
    return _act(y @ w.T + b, act).permute(0, 2, 1).contiguous()


def truth(sd, kind, x, look_ahead, act, device="cpu", prefix="sb_model", head="sb", state=None, return_state=False):
    """x: [N, I, Tp] (any float type; the values are taken as they are) -> [N, O, Tp - look_ahead] float64 (head "fb": [N, O, Tp]).
    state: None (zero) or the initial (h, c) [L, N, H] of a carried session (GRU: c is the fp32 h, which the recurrence starts from);
    return_state: also return the final (h, c) [L, N, H] (GRU: both the final h)."""
    ls = layers(sd, device, prefix)
    I, H = ls[0][0].shape[1], ls[0][1].shape[1]
    rnn = getattr(torch.nn, kind)(I, H, len(ls), batch_first=True).to(device=device, dtype=torch.float64)
    with torch.no_grad():
        for l, (wi, wh, bi, bh) in enumerate(ls):
            for n, v in (("weight_ih", wi), ("weight_hh", wh), ("bias_ih", bi), ("bias_hh", bh)):
                getattr(rnn, f"{n}_l{l}").copy_(v)
        xin = torch.as_tensor(x).to(device=device, dtype=torch.float64).permute(0, 2, 1).contiguous()
        if state is None:
            y, hc = rnn(xin)
        else:
            h0, c0 = (torch.as_tensor(v).to(device=device, dtype=torch.float64).contiguous() for v in state[:2])
            y, hc = rnn(xin, c0 if kind == "GRU" else (h0, c0))
    out = _head(sd, y, look_ahead, act, device, prefix, head)
    if not return_state:
        return out
    return out, ((hc, hc) if kind == "GRU" else hc)


def emulate(sd, kind, x, look_ahead, act, device="cpu", dtype=torch.float64, fault=None, fault_t=32, fault_row=0, prefix="sb_model",
            head="sb", state=None, return_state=False):
    """The kernels' rounding in `dtype` arithmetic (see the module docstring); x, state and return_state as in truth(): state's h is
    the carried fp16 h, its c the carried fp32 c (GRU: fp32 h); an optional third entry [L, N, H] is h(t - 2) of the first frame
    (h_lag at fault_t = 0).  The final state is (fp16 h, fp32 c) per layer.  fault: None or one of FAULTS
      swap_units:    hidden units 3 and 5 (one 32-unit chunk) of layer 0 trade places after every step;
      c_reset:       c (GRU: the carried h) restarts from zero at step fault_t, as if a window boundary dropped it;
      h_lag:         step fault_t reads h(t - 2) instead of h(t - 1);
      row_c_drop:    row fault_row never carries its cell state (c(t - 1) read as zero);
      gru_bias_fold: GRU: b_hn added to the input pseudo-gate n_x instead of n_h, outside r's product."""
    f16 = lambda t: t.to(torch.float16).to(dtype)
    f32 = lambda t: t.to(torch.float32).to(dtype)
    gru = kind == "GRU"
    inp = torch.as_tensor(x).to(device=device, dtype=dtype).permute(2, 0, 1)          # [Tp, N, I]
    if head == "fb":
        inp = f16(inp)                                                                 # fb_pack: the fp32 input to fp16
    Tp, N = inp.shape[0], inp.shape[1]
    ls = layers(sd, device, prefix)
    hs, cs = [], []
    for l, (wi, wh, bi, bh) in enumerate(ls):
        H = wh.shape[1]
        wi16, wh16, bi, bh = f16(wi.to(dtype)), f16(wh.to(dtype)), bi.to(dtype), bh.to(dtype)
        gin = inp @ wi16.T                                                             # [Tp, N, G H]
        if l > 0 and head != "fb":                                                     # the full band's kernels keep Gin in fp32
            gin = f16(gin)
        h16 = torch.zeros(N, H, dtype=dtype, device=device)
        c = torch.zeros(N, H, dtype=dtype, device=device)                              # LSTM: c; GRU: h in fp32
        if state is not None:
            h16, c = (torch.as_tensor(v[l]).to(device=device, dtype=dtype).clone() for v in state[:2])
        hold = h16 if state is None or len(state) < 3 else torch.as_tensor(state[2][l]).to(device=device, dtype=dtype)   # h(t - 2)
        out, top = [], []
        for t in range(Tp):
            if fault == "c_reset" and t == fault_t:
                c = torch.zeros_like(c)
            if fault == "row_c_drop":
                c[fault_row] = 0
            hin = hold if (fault == "h_lag" and t == fault_t) else h16
            rec = hin @ wh16.T
            if gru:
                r = torch.sigmoid(gin[t, :, :H] + bi[:H] + rec[:, :H] + bh[:H])
                z = torch.sigmoid(gin[t, :, H:2 * H] + bi[H:2 * H] + rec[:, H:2 * H] + bh[H:2 * H])
                if fault == "gru_bias_fold":
                    n = torch.tanh(gin[t, :, 2 * H:] + bi[2 * H:] + bh[2 * H:] + r * rec[:, 2 * H:])
                else:
                    n = torch.tanh(gin[t, :, 2 * H:] + bi[2 * H:] + r * (rec[:, 2 * H:] + bh[2 * H:]))
                c = f32((1 - z) * n + z * c)
                h = c
            else:
                g = gin[t] + rec + bi + bh
                i, f, gg, o = g[:, :H], g[:, H:2 * H], g[:, 2 * H:3 * H], g[:, 3 * H:]
                c = f32(torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg))
                h = torch.sigmoid(o) * torch.tanh(c)
            hold, h16 = h16, f16(h)
            if fault == "swap_units" and l == 0:
                h16 = h16[:, [*range(3), 5, 4, 3, *range(6, H)]]
            out.append(h16)
            top.append(f32(h))
        hs.append(h16)
        cs.append(c)
        inp = torch.stack(out)
    if head == "fb":                                                                   # the head reads the top layer's fp32 h
        inp = torch.stack(top)
    y = _head(sd, inp.permute(1, 0, 2).to(torch.float64), look_ahead, act, device, prefix, head, tf32=head == "fb")
    return (y, (torch.stack(hs).to(torch.float64), torch.stack(cs).to(torch.float64))) if return_state else y


def sample_rows(nrows, seed=0, full_below=512):
    """Rows compared for a stage of nrows sequences: all of them up to full_below, else rows 0, 63, 64, 127, 128 and the last, the
    first and last row of every 64-row CTA, and 256 random rows."""
    if nrows <= full_below:
        return np.arange(nrows)
    s = {0, 63, 64, 127, 128, nrows - 1}
    for c0 in range(0, nrows, 64):
        s.update((c0, min(c0 + 63, nrows - 1)))
    s.update(np.random.default_rng(seed).choice(nrows, 256, replace=False).tolist())
    return np.array(sorted(s))


def compare(got, want, emu, factor, mask=None):
    """Element-wise errors of got against want (fp64 truth) on the elements mask selects (default: all), and the rule's bound
    factor * (3 max |emu - want| + 1e-6 RMS).  Returns a dict; ok = max err <= bound."""
    got, want, emu = (torch.as_tensor(a).to("cpu", torch.float64) for a in (got, want, emu))
    if mask is not None:
        got, want, emu = got[mask], want[mask], emu[mask]
    rms = float(want.pow(2).mean().sqrt()) if want.numel() else 0.0
    rms = rms if rms > 0 else 1.0
    err, eerr = float((got - want).abs().max()), float((emu - want).abs().max())
    bound = factor * (ACCURATE_MULT * eerr + FLOOR * rms)
    rel = float((got - want).norm() / max(float(want.norm()), 1e-300))
    return dict(err=err / rms, emu=eerr / rms, bound=bound / rms, rel=rel, ratio=err / max(eerr, 1e-300), ok=err <= bound,
                finite=bool(torch.isfinite(got).all()))
