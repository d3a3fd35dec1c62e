"""fp64 references of the TCN stage alone (the full-band models of FullSubNet+ and the sub-band TCN), and the faults the element-wise
rule of sb_rnn_ref.compare must catch in them.

The stage is SequenceModel's TCN branch (sequence_model.py:47-58,106-112; TCNBlock, causal_conv.py:67-108): eight blocks of 1x1 conv
(C -> 512) + PReLU + gLN, depth-wise conv (k = 3, dilations 1 2 5 9 1 2 5 9) + PReLU + gLN, 1x1 conv (512 -> C) + residual; then ReLU
and the head.  Both references read the model's own state_dict under `prefix` ("fb_model", "fb_model_real", "fb_model_imag" or
"sb_model"), so the host-side packing (pack_tcn_blocks, pack_tcn5, pack_sb_tcn in fsn_api.cu) is under test as well.

* truth():   the stage in float64, restating O.tcn_block / O.seq_tcn (test_full_band_cpu.py pins the two to 1e-12).  Each group
             (row of x) is its own clip of tlen[n] frames: gLN statistics, the depth-wise taps and the output cover those frames only.
* emulate(): the same computation rounded where the kernels round (k_gemm_tc5.cu, fsn_api.cu):
               - GEMM1 reads the fp32 residual stream through the tf32 tensor core, which truncates the 13 low mantissa bits; W1 is
                 rounded to tf32 on the host (to_tf32, round to nearest);
               - EPI5_PRELU_STATS: bias + PReLU in fp32, the gLN1 statistics from those values, then the hidden activation stored as
                 fp16(clamp(y * 2^-e, +-65504)), e from fp16_store_scale of max |x| over the group's stream entering the block;
               - dwconv_tm_kernel: the slab fp16 * (gamma rstd 2^e) + (beta - mean rstd gamma) in fp32, zero past the clip, the three
                 taps + bias + PReLU, the gLN2 statistics before the +-65504 clamp and the fp16 store;
               - EPI5_GLN_RES: W2' = fp16(W2 diag(gamma2)) (pack_tcn_blocks), s1 = sum of the rounded W2' and s2b = sum W2 beta2 + bias
                 in fp64 -> fp32, new stream = fp32(x + rstd (W2' y) - mean rstd s1 + s2b), zero past the clip;
               - full-band head (EPI5_OUT): relu(x) truncated to tf32 times the to_tf32-rounded Linear, + bias, activation;
                 sub-band head (EPI5_GLN_HEAD): relu(x) in fp32 times the fp32 Linear (pack_sb_tcn), + bias, activation, the first
                 look_ahead frames dropped.
             Its distance from truth() on the same elements is the error the kernels' number formats make unavoidable.  `fault` plants
             one of FAULTS (test_full_band_cpu.py shows each fails the rule by >= 10x).

Rule: sb_rnn_ref.compare, max |kernel - fp64| <= TCN_FACTOR * (3 max |emulation - fp64| + 1e-6 RMS).  TCN_FACTOR = 1: the TCN path has
no approximate transcendental (the head's tanh is the accurate tanhf).  Measured once on one H100 80GB HBM3 SXM at its 700 W power
limit over every case of tests/test_gpu_full_band.py: the kernels' max err was at most 1.28x the emulation's (T' = 18); the worst
case per stage and width is in DESIGN.md §2.
"""
import numpy as np
import torch

TCN_FACTOR = 1.0
DILATIONS = (1, 2, 5, 9, 1, 2, 5, 9)
HIDDEN = 512
GLN_EPS = 1e-8
DW_CHUNK = 256                                   # dwconv_tm_kernel's frame chunk (DW_TCH)

FAULTS = ("dilation", "causal_taps", "chunk_halo", "tile_stats", "gln_extent", "branch_param", "unscale_drop")


def _sd(sd, key, device):
    v = sd[key]
    v = v.detach().cpu() if isinstance(v, torch.Tensor) else torch.from_numpy(np.asarray(v))
    return v.to(device=device, dtype=torch.float64)


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


def _bits(t, fn):
    """fn applied to the fp32 bit pattern of t (as int32)"""
    return fn(t.to(torch.float32).contiguous().view(torch.int32)).view(torch.float32)


def trunc_tf32(t):
    """what the tf32 tensor core reads of an fp32 operand: the 13 low mantissa bits dropped"""
    return _bits(t, lambda u: u & -8192).to(t.dtype)


def round_tf32(t):
    """fsn_api.cu to_tf32: round to nearest even on the 13 dropped bits"""
    return _bits(t, lambda u: (u + 0xfff + ((u >> 13) & 1)) & -8192).to(t.dtype)


def round_tf32_away(t):
    """cvt.rna.tf32.f32 (conv1x1_tf32_kernel, k_front.cu): round to nearest, ties away from zero"""
    return _bits(t, lambda u: (u + 0x1000) & -8192).to(t.dtype)


def store_scale(amax):
    """fp16_store_scale (fsn_common.cuh): 2^-e with amax = m 2^e, m in [0.5, 1), e clamped to 0..126"""
    e = torch.frexp(torch.clamp(amax.to(torch.float32), max=3.0e38)).exponent.clamp(0, 126)
    return torch.pow(2.0, -e.to(torch.float64))


def _stats(y, v, n, centred):
    """mean and rstd of y over the valid frames v ([N, T, 1]) per group, n elements per group.  centred: the fp64 truth; otherwise the
    kernels' sum / sum-of-squares in fp64 (gln_mean_rstd, k_gemm_tc5.cu) with mean and rstd rounded to fp32."""
    s = (y * v).sum(dim=(1, 2))
    mean = s / n
    if centred:
        var = (((y - mean[:, None, None]) * v) ** 2).sum(dim=(1, 2)) / n
        return mean, 1.0 / torch.sqrt(var + GLN_EPS)
    var = ((y * v) ** 2).sum(dim=(1, 2)) / n - mean * mean
    rstd = 1.0 / torch.sqrt(var.clamp(min=0) + GLN_EPS)
    return mean.to(torch.float32).to(y.dtype), rstd.to(torch.float32).to(y.dtype)


def _run(sd, prefix, x, tlen, causal, head, act, look_ahead, device, dtype, rnd, fault=None, fault_blk=2):
    f16 = lambda t: t.clamp(-65504.0, 65504.0).to(torch.float16).to(dtype)
    f32 = lambda t: t.to(torch.float32).to(dtype)
    g = lambda k: _sd(sd, f"{prefix}.sequence_model.{k}", device).to(dtype)
    xs = torch.as_tensor(x).to(device=device, dtype=dtype).permute(0, 2, 1).contiguous()          # [N, T, C] time-major
    N, T, C = xs.shape
    tl = torch.full((N,), T, dtype=torch.int64, device=device) if tlen is None else torch.as_tensor(tlen, device=device).long()
    v = (torch.arange(T, device=device)[None, :] < tl[:, None]).to(dtype)[:, :, None]           # [N, T, 1]
    xs = xs * v
    n1 = (HIDDEN * tl).to(dtype)
    slope_pre = prefix.split("_")[0] + "_model" if fault == "branch_param" else prefix           # "fb_model_real" -> "fb_model"
    for blk, d in enumerate(DILATIONS):
        q = f"{blk}."
        if fault == "dilation" and blk == 2:
            d = 4
        w1, b1 = g(q + "conv1x1.weight")[:, :, 0], g(q + "conv1x1.bias")
        a1 = _sd(sd, f"{slope_pre}.sequence_model.{q}prelu1.weight", device).to(dtype)[0]
        a2 = _sd(sd, f"{slope_pre}.sequence_model.{q}prelu2.weight", device).to(dtype)[0]
        y = (trunc_tf32(xs) @ round_tf32(w1).T if rnd else xs @ w1.T) + b1
        y = torch.where(y >= 0, y, a1 * y) * v
        mean, rstd = _stats(y, v, n1, not rnd)
        gam, bet = g(q + "norm1.weight"), g(q + "norm1.bias")
        if rnd:
            sc = store_scale((xs.abs() * v).amax(dim=(1, 2)))[:, None, None].to(dtype)
            y16 = f16(y * sc)
            un = 1.0 if (fault == "unscale_drop" and blk == fault_blk) else 1.0 / sc
            gr = gam * rstd[:, None, None]
            slab = f32(y16 * f32(gr * un) + f32(bet - mean[:, None, None] * gr))
        else:
            slab = (y - mean[:, None, None]) * rstd[:, None, None] * gam + bet
        slab = slab * v
        wd, bd = g(q + "depthwise_conv.weight")[:, 0, :], g(q + "depthwise_conv.bias")
        cz = causal and not (fault == "causal_taps" and blk == fault_blk)
        offs = (-2 * d, -d, 0) if cz else (-d, 0, d)
        pad = torch.nn.functional.pad(slab, (0, 0, 2 * d, 2 * d))
        t = torch.arange(T, device=device)
        z = bd.expand(N, T, HIDDEN).clone()
        for j, o in enumerate(offs):
            tap = pad[:, 2 * d + o:2 * d + o + T]
            if fault == "chunk_halo":
                tap = tap * ((t + o) // DW_CHUNK == t // DW_CHUNK).to(dtype)[None, :, None]
            z = z + wd[:, j] * tap
        z = torch.where(z >= 0, z, a2 * z) * v
        n2 = (HIDDEN * torch.where(tl < T, torch.full_like(tl, T), tl)).to(dtype) if fault == "gln_extent" else n1
        mean2, rstd2 = _stats(z, v, n2, not rnd)
        mr, rr = mean2[:, None].expand(N, T).clone(), rstd2[:, None].expand(N, T).clone()
        if fault == "tile_stats":                    # a group starting inside a 128-row tile: its first row reads group n - 1's statistics
            for n in range(1, N):
                if (n * T) % 128:
                    mr[n, 0], rr[n, 0] = mean2[n - 1], rstd2[n - 1]
        mr, rr = mr[:, :, None], rr[:, :, None]
        w2, b2, g2, be2 = g(q + "sconv.weight")[:, :, 0], g(q + "sconv.bias"), g(q + "norm2.weight"), g(q + "norm2.bias")
        if rnd:
            w2h = f16(f32(w2 * g2))
            s1 = f32(w2h.to(torch.float64).sum(dim=1).to(dtype))
            s2b = f32((w2.to(torch.float64) @ be2.to(torch.float64) + b2.to(torch.float64)).to(dtype))
            o = rr * (f16(z) @ w2h.T) - mr * rr * s1 + s2b
            xs = f32(xs + o) * v
        else:
            xs = (xs + ((z - mr) * rr * g2 + be2) @ w2.T + b2) * v
    wfc, bfc = _sd(sd, f"{prefix}.fc_output_layer.weight", device).to(dtype), _sd(sd, f"{prefix}.fc_output_layer.bias", device).to(dtype)
    r = torch.relu(xs)
    if head == "fb":
        out = (trunc_tf32(r) @ round_tf32(wfc).T if rnd else r @ wfc.T) + bfc
        return _act(out, act).to(torch.float64).permute(0, 2, 1).contiguous()                   # [N, F, T]
    if head == "sb":
        return _act(r[:, look_ahead:] @ wfc.T + bfc, act).to(torch.float64).permute(0, 2, 1).contiguous()   # [N, O, T - la]
    raise ValueError(head)


def truth(sd, prefix, x, tlen, causal, head, act=None, look_ahead=0, device="cpu"):
    """x: [N, C, T'] (any float type; the values are taken as they are), tlen: [N] frames per group or None (all T').  head "fb":
    ReLU -> Linear(C -> C) -> act, [N, C, T'];  head "sb": ReLU -> Linear(C -> O) -> act without the first look_ahead frames,
    [N, O, T' - look_ahead].  float64; frames past a group's tlen are meaningless (the kernels' are compared as finite only)."""
    return _run(sd, prefix, x, tlen, causal, head, act, look_ahead, device, torch.float64, False)


def emulate(sd, prefix, x, tlen, causal, head, act=None, look_ahead=0, device="cpu", dtype=torch.float64, fault=None, fault_blk=2):
    """The kernels' rounding (module docstring) in `dtype` arithmetic; arguments as truth().  fault: None or one of FAULTS
      dilation:     block 2 uses dilation 4 instead of 5;
      causal_taps:  block fault_blk of a causal model reads t - d, t, t + d;
      chunk_halo:   taps that cross a 256-frame chunk boundary of the depth-wise kernel read zero;
      tile_stats:   the first row of a group that starts inside a 128-row tile takes the previous group's gLN2 mean / rstd;
      gln_extent:   a ragged group's gLN2 counts T' frames instead of its own tlen;
      branch_param: a real / imag branch uses the mag branch's ("fb_model") PReLU slopes;
      unscale_drop: block fault_blk's fp16 store scale is not undone before gLN1."""
    return _run(sd, prefix, x, tlen, causal, head, act, look_ahead, device, dtype, True, fault, fault_blk)


def distinct_slopes(sd, prefixes):
    """The parameter draws give every branch the same PReLU slopes; make them differ per branch and block (in place), so that a branch
    reading another's parameters is visible."""
    for k, pre in enumerate(prefixes):
        for blk in range(8):
            for j, name in enumerate(("prelu1", "prelu2")):
                sd[f"{pre}.sequence_model.{blk}.{name}.weight"] = np.array([0.05 + 0.15 * k + 0.03 * blk + 0.1 * j], np.float32)
    return sd
