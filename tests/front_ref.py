"""fp64 truth, float32 emulation and planted faults of the front end (k_front.cu), per clip over the clip's own extent.

Two stages:
  * fb_in: model input -> input norm (input_norm_kernel, or the utterance Laplace norm of the TSSE chain) -> channel attention
    (tsse_rowstats_kernel, tsse_norm_kernel, tsse_apply_kernel);
  * sub-band input: (fb_in[0] or the padded magnitude, fb_out) -> unfold -> norm (sb_rowsum_kernel, sb_stats_kernel, sb_pack_kernel /
    sb_pack_cum_kernel).  Its truth is computed from the forward's own fb_in / fb_out stages, so only the packer contributes error.

* fb_in_truth / sb_in_truth: float64, restated from oracle/fsn_oracle.py (the four NORMS, tsse, se_layer, cbam_layer, eca_layer, the
  subband_num > 1 ECA grouping, unfold), each clip b over frames[b] + look_ahead frames; zero past that extent.
* fb_in_emulate / sb_in_emulate: the kernels' float32 arithmetic in its order: lane-strided fp32 row sums (32 lanes, lane l summing
  frames l, l + 32, ... in order, then the xor-shuffle tree), fp64 utterance totals, the TSSE windowed sums as S - prefix - suffix from
  shuffle scans, per-frame fp32 column sums over F with an fp64 scan (cumulative norms), per-(sequence, frame) fp32 channel sums with
  an fp64 scan (sb_pack_cum_kernel), fp32 (v - mu) * inv for the offline sub-band norms.  ``fault`` plants one of FAULTS.
* decode_sb_img: the sub-band images (get_stage "sb_img") back to [B*F, Isb, T'] with its own restatement of SWIZZLE_128B (16-byte
  chunk k / 8 of row r stored at chunk (k / 8) ^ (r % 8), as TMA and wgmma define it).

The rule is sb_rnn_ref.compare with factor 1: no approximate transcendental takes part except __expf in the gates (max error
2 + floor(|1.16 x|) ulp), which for |x| < 1.7 is within 3 ulp of expf, below what 3 x the emulation's own error of the inputs covers.
"""
import numpy as np

from oracle import fsn_oracle as O

NORMS = tuple(O.NORMS)
F32 = np.float32
KMAX = 16
EPS_F32 = float(np.finfo(np.float32).eps)

FB_FAULTS = ("tsse_suffix", "mean_over_T", "ragged_batch_T", "eca_edge_self", "fc1_drop_last", "cbam_pad_ignored", "subband_reflect",
             "cum_count", "biased_std")
SB_FAULTS = ("sb_edge_replicate", "sb_fb_swap", "sb_biased_std", "sb_mean_over_T")
IMG_FAULTS = ("swizzle_hi",)
FAULTS = FB_FAULTS + SB_FAULTS + IMG_FAULTS


# ---- helpers ------------------------------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fmaf: a * b + c rounded once to float32 (the product of two floats is exact in float64)"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(F32)


def xor_tree(v):
    """warp_sum over the last axis (32 lanes): v += shfl_xor(v, o) for o = 16 .. 1; every lane ends with lane 0's value"""
    v = v.astype(F32)
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., idx ^ o]).astype(F32)
    return v[..., 0]


def lane_sum(x, sq=False):
    """The rowstats / rowsum warp's fp32 sum over the last axis: lane l adds frames l, l + 32, ... in order (fmaf(v, v, q) for sq)"""
    x = np.asarray(x, F32)
    n = x.shape[-1]
    pad = (-n) % 32
    xp = np.concatenate([x, np.zeros(x.shape[:-1] + (pad,), F32)], axis=-1).reshape(x.shape[:-1] + (-1, 32))
    acc = np.zeros(x.shape[:-1] + (32,), F32)
    for i in range(xp.shape[-2]):
        acc = fma32(xp[..., i, :], xp[..., i, :], acc) if sq else (acc + xp[..., i, :]).astype(F32)
    return xor_tree(acc)


def seq_sum(x, axis, sq=False):
    """fp32 sum in index order along ``axis`` (a single thread's loop; fmaf(v, v, q) for sq)"""
    x = np.moveaxis(np.asarray(x, F32), axis, 0)
    acc = np.zeros(x.shape[1:], F32)
    for v in x:
        acc = fma32(v, v, acc) if sq else (acc + v).astype(F32)
    return acc


def shfl_scan(v):
    """inclusive Hillis-Steele scan over the last axis (16 lanes) in fp32, as the rowstats warp's __shfl_up_sync loop"""
    v = v.astype(F32)
    for o in (1, 2, 4, 8):
        u = np.concatenate([np.zeros(v.shape[:-1] + (o,), F32), v[..., :-o]], axis=-1)
        v = (v + u).astype(F32)
    return v


def sigmoid32(y):
    return (F32(1.0) / (F32(1.0) + np.exp(-np.asarray(y, F32)).astype(F32))).astype(F32)


def _p(params, key, dt):
    return np.asarray(params[key], dt)


def clip_extents(B, Tp, la, frames):
    return [Tp] * B if frames is None else [int(n) + la for n in frames]


def branches(cfg, inputs):
    """(prefixes, input planes) of the model: FullSubNet+ has three branches (mag, real, imag), fullsubnet.Model one"""
    if len(inputs) == 3:
        return ("channel_attention", "channel_attention_real", "channel_attention_imag"), inputs
    return (None,), inputs


# ---- fb_in: truth -----------------------------------------------------------------------------------------------------------------
def fb_in_truth(params, cfg, inputs, frames=None):
    """float64 [nbranch, B, F, T'] fb_in of every clip over its own extent (zero past it).  inputs: (mag, real, imag) [B, 1, F, T] of
    FullSubNet+ or (mag,) of fullsubnet.Model; cfg: the model's configuration (channel_attention_model absent: no attention)."""
    la = cfg["look_ahead"]
    prefixes, planes = branches(cfg, inputs)
    B, _, F, T = planes[0].shape
    Tp = T + la
    norm = O.NORMS[cfg["norm_type"]]
    sub = cfg.get("subband_num", 1)
    out = np.zeros((len(planes), B, F, Tp))
    for b, Tpe in enumerate(clip_extents(B, Tp, la, frames)):
        for br, (pre, x) in enumerate(zip(prefixes, planes)):
            xb = np.zeros((1, 1, F, Tpe))
            xb[0, 0, :, :Tpe - la] = np.asarray(x[b, 0, :, :Tpe - la], np.float64)
            xn = norm(xb)
            if pre is None:
                y = xn[0, 0]
            elif sub > 1 and br == 0:                                    # fullsubnet_plus.py:146-153, mag branch only
                pn = sub - F % sub
                xi = np.pad(xn, ((0, 0), (0, 0), (0, pn), (0, 0)), mode="reflect").reshape(1, (F + pn) // sub, Tpe * sub)
                y = O.channel_attention(xi, params, pre, cfg).reshape(F + pn, Tpe)[:F]
            else:
                y = O.channel_attention(xn[0], params, pre, cfg)[0]
            out[br, b, :, :Tpe] = y
    return out


# ---- fb_in: emulation -------------------------------------------------------------------------------------------------------------
def _input_norm32(x, kind, F, Tpe, fault=None):
    """input_norm_kernel on one clip's padded plane x [F, Tpe] (float32): per-frame fp32 sums over F in bin order, fp64 scan"""
    cs, cq = seq_sum(x, 0), seq_sum(x, 0, sq=True)
    s, q = np.cumsum(cs.astype(np.float64)), np.cumsum(cq.astype(np.float64))
    if kind == "offline_gaussian_norm":
        n = float(F) * Tpe
        mu = s[-1] / n
        var = (q[-1] - n * mu * mu) / (n if fault == "biased_std" else n - 1.0)
        inv = 1.0 / (np.sqrt(max(var, 0.0)) + 1e-5)
        sa, sb = np.full(Tpe, inv), np.full(Tpe, -mu * inv)
    else:
        t = np.arange(Tpe, dtype=np.float64)
        cnt = float(F) * (t if fault == "cum_count" else t + 1)
        with np.errstate(divide="ignore", invalid="ignore"):
            cm = s / cnt
            if kind == "cumulative_laplace_norm":
                sa, sb = 1.0 / (cm + EPS_F32), np.zeros(Tpe)
            else:
                cv = (q - 2.0 * cm * s) / cnt + cm * cm
                inv = 1.0 / np.sqrt(cv + EPS_F32)
                sa, sb = inv, -cm * inv
    return fma32(x, sa.astype(F32)[None, :], sb.astype(F32)[None, :])


def _gate32(params, pre, cfg, x, Te, Tpe, inv, kind, sub, br, fault):
    """tsse_norm_kernel's per-channel gate of one (clip, branch): x [F, Tpe] float32 (zero past Te), inv its fp32 normaliser"""
    F = x.shape[0]
    S = lane_sum(x[:, :Te])
    rT = F32(1.0) / F32(Tpe)
    if kind == "TSSE":
        hv = np.zeros((F, KMAX), F32)
        n = min(KMAX, Te)
        hv[:, :n] = x[:, :n]
        tv = np.zeros((F, KMAX), F32)
        for j in range(KMAX):                                            # lane j: sample Tpe - 1 - j (zero in the look-ahead pad)
            t = Tpe - 1 - j
            if 0 <= t < Te:
                tv[:, j] = x[:, t]
        pfx = (shfl_scan(hv) - hv).astype(F32)
        sfx = (shfl_scan(tv) - tv).astype(F32)
        sfx = np.concatenate([sfx, np.zeros((F, 1), F32)], axis=1)       # index KMAX: what a k - j suffix index would reach at j = 0
        s = np.full(F, _p(params, f"{pre}.feature_concate_fc.bias", F32)[0], F32)
        cw = _p(params, f"{pre}.feature_concate_fc.weight", F32)[0]
        for i, (name, k) in enumerate(zip(("smallConv1d", "middleConv1d", "largeConv1d"), cfg["kersize"])):
            w = _p(params, f"{pre}.{name}.0.weight", F32)[:, 0, :]
            bias = _p(params, f"{pre}.{name}.0.bias", F32)
            rlen = F32(1.0) / F32(Tpe - k + 1)
            acc = np.zeros(F, F32)
            for j in range(k):
                m = k - j if fault == "tsse_suffix" else k - 1 - j
                wsum = ((S - pfx[:, j]).astype(F32) - sfx[:, m]).astype(F32)
                acc = fma32(w[:, j], wsum, acc)
            feat = np.maximum(fma32(acc, F32(inv * rlen), bias), F32(0))
            s = fma32(cw[i], feat, s)
        sq, mx = s, None
    else:
        sq = (S * inv).astype(F32) * rT
        sq = sq.astype(F32)
        if kind == "CBAM":
            big, small = x[:, :Te].max(axis=1), x[:, :Te].min(axis=1)
            mx = (big * inv if inv >= 0 else small * inv).astype(F32)
            if Tpe > Te and fault != "cbam_pad_ignored":
                mx = np.maximum(mx, F32(0))
    if kind == "ECA":
        w = _p(params, f"{pre}.conv.weight", F32).reshape(-1)
        if sub > 1 and br == 0:
            Cg = F // sub + 1
            sg = np.zeros(Cg, F32)
            for c in range(Cg):
                acc = F32(0)
                for j in range(sub):
                    f = c * sub + j
                    if f >= F:
                        f = 2 * F - 1 - f if fault == "subband_reflect" else 2 * F - 2 - f
                    acc = F32(acc + S[f])
                sg[c] = F32(F32(acc * inv) / F32(F32(Tpe) * F32(sub)))
            z = np.concatenate([[F32(0)], sg, [F32(0)]]).astype(F32)
            y = fma32(w[2], z[2:], fma32(w[1], z[1:-1], (w[0] * z[:-2]).astype(F32)))
            return sigmoid32(y)[np.arange(F) // sub]
        z = np.concatenate([[F32(0)], sq, [F32(0)]]).astype(F32)
        if fault == "eca_edge_self":
            z[0], z[-1] = sq[0], sq[-1]
        y = fma32(w[2], z[2:], fma32(w[1], z[1:-1], (w[0] * z[:-2]).astype(F32)))
        return sigmoid32(y)
    # fc1 -> ReLU (CBAM: on both squeezes, summed) -> fc2 -> sigmoid, lane-strided fmaf sums and the xor tree
    w1, b1 = _p(params, f"{pre}.fc1.weight", F32), _p(params, f"{pre}.fc1.bias", F32)
    w2, b2 = _p(params, f"{pre}.fc2.weight", F32), _p(params, f"{pre}.fc2.bias", F32)
    Cr = F // 2

    def dense(W, v):                                                     # [M, K] x [K] as the warps sum it
        M, K = W.shape
        acc = np.zeros((M, 32), F32)
        for c0 in range(0, K, 32):
            n = min(32, K - c0)
            acc[:, :n] = fma32(W[:, c0:c0 + n], v[None, c0:c0 + n], acc[:, :n])
        return xor_tree(acc)

    f1 = np.maximum((dense(w1, sq) + b1).astype(F32), F32(0))
    if kind == "CBAM":
        f1 = (f1 + np.maximum((dense(w1, mx) + b1).astype(F32), F32(0))).astype(F32)
    if fault == "fc1_drop_last" and Cr % 4:
        f1[Cr - 1] = 0
    return sigmoid32((dense(w2, f1) + b2).astype(F32))


def fb_in_emulate(params, cfg, inputs, frames=None, fault=None):
    """fb_in as the kernels compute it, float32 [nbranch, B, F, T'] (zero past each extent); fault: None or one of FB_FAULTS"""
    la = cfg["look_ahead"]
    prefixes, planes = branches(cfg, inputs)
    B, _, F, T = planes[0].shape
    Tp = T + la
    kind = cfg.get("channel_attention_model") if prefixes[0] is not None else None
    sub = cfg.get("subband_num", 1)
    nt = cfg["norm_type"]
    out = np.zeros((len(planes), B, F, Tp), F32)
    for b, Tpe in enumerate(clip_extents(B, Tp, la, frames)):
        if fault == "ragged_batch_T":
            Tpe_n = Tp                                                   # normalised over the batch's T'
        else:
            Tpe_n = Tpe
        for br, (pre, x) in enumerate(zip(prefixes, planes)):
            xp = np.zeros((F, Tpe), F32)
            xp[:, :Tpe - la] = np.asarray(x[b, 0, :, :Tpe - la], F32)
            if nt != "offline_laplace_norm":
                xp = _input_norm32(xp, nt, F, Tpe, fault)
                Te, inv = Tpe, F32(1.0)
            else:
                Te = Tpe - la
                tot = float(np.sum(lane_sum(xp[:, :Te]).astype(np.float64)))
                n = float(F) * ((Tpe_n - la) if fault == "mean_over_T" else Tpe_n)
                inv = F32(1.0 / (tot / n + 1e-5))
            if kind is None:
                scale = np.full(F, inv, F32)
            else:
                scale = (_gate32(params, pre, cfg, xp, Te, Tpe, inv, kind, sub, br, fault) * inv).astype(F32)
            out[br, b, :, :Tpe] = (xp * scale[:, None]).astype(F32)
    return out


# ---- sub-band input -----------------------------------------------------------------------------------------------------------------
def isb(cfg, nfb):
    return 2 * cfg["sb_num_neighbors"] + 1 + nfb * (2 * cfg["fb_num_neighbors"] + 1)


def _sources(win, fbs, b, Tpe):
    return np.asarray(win[b, :, :Tpe]), [np.asarray(o[b, :, :Tpe]) for o in fbs]


def sb_in_truth(cfg, win, fbs, frames=None):
    """float64 [B, F, Isb, T'] normalised sub-band input of every clip over its own extent (zero past it), and the utterance means
    [B] of the un-normalised input.  win: [B, F, T'] the window source (FullSubNet+: fb_in[0]; fullsubnet.Model: the padded magnitude),
    fbs: the full-band outputs [B, F, T'] (three or one), as the forward kept them."""
    B, F, Tp = win.shape
    la, Ns, Nf = cfg["look_ahead"], cfg["sb_num_neighbors"], cfg["fb_num_neighbors"]
    I = isb(cfg, len(fbs))
    out, mus = np.zeros((B, F, I, Tp)), np.zeros(B)
    for b, Tpe in enumerate(clip_extents(B, Tp, la, frames)):
        w, fo = _sources(win, fbs, b, Tpe)
        parts = [O.unfold(w.astype(np.float64)[None, None], Ns).reshape(1, F, 2 * Ns + 1, Tpe)]
        parts += [O.unfold(o.astype(np.float64)[None, None], Nf).reshape(1, F, 2 * Nf + 1, Tpe) for o in fo]
        x = np.concatenate(parts, axis=2)
        mus[b] = x.mean()
        out[b, :, :, :Tpe] = O.NORMS[cfg["norm_type"]](x)[0]
    return out, mus


def _reflect(p, F, fault=None):
    if fault == "sb_edge_replicate":
        return np.clip(p, 0, F - 1)
    p = np.abs(p)
    return np.where(p > F - 1, 2 * (F - 1) - p, p)


def sb_in_emulate(cfg, win, fbs, frames=None, fault=None):
    """The packers' float32 values [B, F, Isb, T'] (zero past each extent) and sb_stats_kernel's utterance means [B]; fault: None or
    one of SB_FAULTS"""
    B, F, Tp = win.shape
    la, Ns, Nf = cfg["look_ahead"], cfg["sb_num_neighbors"], cfg["fb_num_neighbors"]
    nfb = len(fbs)
    I = isb(cfg, nfb)
    nt = cfg["norm_type"]
    if fault == "sb_fb_swap" and nfb == 3:
        fbs = [fbs[0], fbs[2], fbs[1]]
    out, mus = np.zeros((B, F, I, Tp), F32), np.zeros(B, F32)
    for b, Tpe in enumerate(clip_extents(B, Tp, la, frames)):
        w, fo = _sources(win, fbs, b, Tpe)
        w, fo = np.asarray(w, F32), [np.asarray(o, F32) for o in fo]
        f = np.arange(F)
        chans = [w[_reflect(f + k - Ns, F, fault)] for k in range(2 * Ns + 1)]
        for o in fo:
            chans += [o[_reflect(f + j - Nf, F, fault)] for j in range(2 * Nf + 1)]
        x = np.stack(chans, axis=1)                                      # [F, I, Tpe] float32
        # sb_rowsum_kernel: lane-strided fp32 row sums of every source row; sb_stats_kernel: fp64 totals, each row counted as often as
        # it appears in some window
        srcs = [w] + fo
        rs = [lane_sum(s).astype(np.float64) for s in srcs]
        rq = [lane_sum(s, sq=True).astype(np.float64) for s in srcs]
        cnt = [np.bincount(_reflect(f[:, None] + np.arange(2 * n + 1)[None, :] - n, F).ravel(), minlength=F)
               for n in [Ns] + [Nf] * nfb]
        s = sum(float(np.dot(c, r)) for c, r in zip(cnt, rs))
        q = sum(float(np.dot(c, r)) for c, r in zip(cnt, rq))
        n = float(F) * I * ((Tpe - la) if fault == "sb_mean_over_T" else Tpe)
        mu = s / n
        mus[b] = mu
        if nt in ("offline_laplace_norm", "offline_gaussian_norm"):
            if nt == "offline_gaussian_norm":
                var = (q - n * mu * mu) / (n if fault == "sb_biased_std" else n - 1.0)
                sig = F32(np.sqrt(max(var, 0.0)))
                inv, sub = F32(1.0) / F32(sig + F32(1e-5)), F32(mu)
            else:
                inv, sub = F32(1.0) / F32(F32(mu) + F32(1e-5)), F32(0)
            y = ((x - sub).astype(F32) * inv).astype(F32)
        else:
            # sb_pack_cum_kernel: per (sequence, frame) fp32 sums over the I channels in channel order, fp64 scan over the frames
            cs, cq = seq_sum(x, 1), seq_sum(x, 1, sq=True)               # [F, Tpe]
            ds, dq = np.cumsum(cs.astype(np.float64), axis=1), np.cumsum(cq.astype(np.float64), axis=1)
            cnt = float(I) * (np.arange(Tpe) + 1.0)
            cm = ds / cnt
            if nt == "cumulative_laplace_norm":
                sc, sh = (1.0 / (cm + EPS_F32)).astype(F32), np.zeros_like(cm, dtype=F32)
            else:
                cv = (dq - 2.0 * cm * ds) / cnt + cm * cm
                iv = 1.0 / np.sqrt(cv + EPS_F32)
                sc, sh = iv.astype(F32), (-cm * iv).astype(F32)
            y = fma32(x, sc[:, None, :], sh[:, None, :])
        out[b, :, :, :Tpe] = y
    return out, mus


# ---- the fp16 sub-band images -------------------------------------------------------------------------------------------------------
def img_tiles(rows):
    """tiles of the images: ceil(rows / 128) rounded up to whole pairs (the clusters of the layer-wise kernel)"""
    return ((rows + 127) // 128 + 1) // 2 * 2


def img_bytes(rows, Tp, wide):
    return img_tiles(rows) * Tp * 128 * (256 if wide else 128)


def decode_sb_img(raw, rows, Tp, I, layout, fault=None):
    """raw: the bytes of get_stage("sb_img") (uint8) -> (values [rows, I, Tp] float16, every element of the buffer outside them:
    rows >= rows, channels >= I and the unused tail, as one flat float16 array).  layout: "sw128" (I <= 64), "wide_layerwise" or
    "wide_tm".  fault "swizzle_hi": decode with chunk (k / 8) ^ ((r >> 3) & 7)."""
    h = np.frombuffer(np.ascontiguousarray(raw).tobytes(), np.float16)
    npair = img_tiles(rows)
    used = np.zeros(h.shape, bool)
    if layout == "sw128":
        img = h.reshape(npair, Tp, 128, 8, 8)                             # [tile, t, r, physical chunk, half]
        r = np.arange(128)
        key = ((r >> 3) & 7) if fault == "swizzle_hi" else (r & 7)
        phys = np.arange(8)[None, :] ^ key[:, None]                      # [r, logical chunk] -> physical chunk
        vals = img[:, :, r[:, None], phys, :].reshape(npair, Tp, 128, 64)
        pos = np.arange(h.size).reshape(npair, Tp, 128, 8, 8)[:, :, r[:, None], phys, :].reshape(npair, Tp, 128, 64)
        vals = vals.transpose(0, 2, 3, 1).reshape(npair * 128, 64, Tp)
        pos = pos.transpose(0, 2, 3, 1).reshape(npair * 128, 64, Tp)
    elif layout == "wide_layerwise":
        vals = h.reshape(npair, Tp, 128, 128).transpose(0, 2, 3, 1).reshape(npair * 128, 128, Tp)
        pos = np.arange(h.size).reshape(npair, Tp, 128, 128).transpose(0, 2, 3, 1).reshape(npair * 128, 128, Tp)
    elif layout == "wide_tm":
        nt = (rows + 127) // 128
        n = Tp * nt * 128 * 128
        vals = h[:n].reshape(Tp, nt * 128, 128).transpose(1, 2, 0)
        pos = np.arange(n).reshape(Tp, nt * 128, 128).transpose(1, 2, 0)
    else:
        raise ValueError(layout)
    used[pos[:rows, :I].ravel()] = True
    return vals[:rows, :I], h[~used]


def encode_sw128(x):
    """[tiles * 128, 64, Tp] float16 -> the SWIZZLE_128B image bytes (what sb_pack_kernel's Fp16Img store writes); CPU tests only"""
    rows, _, Tp = x.shape
    img = np.zeros((rows // 128, Tp, 128, 8, 8), np.float16)
    v = x.reshape(rows // 128, 128, 8, 8, Tp).transpose(0, 4, 1, 2, 3)
    for r in range(128):
        img[:, :, r, np.arange(8) ^ (r & 7), :] = v[:, :, r]
    return img.view(np.uint8).ravel()


def fp16_spacing(x):
    """the spacing of fp16 numbers at |x| (2^-24 in the subnormal range)"""
    a = np.abs(np.asarray(x, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.exp2(e - 10)
