"""The front end (k_front.cu) against fp64, element by element: fb_in from the model input, and the sub-band input from the forward's
own fb_in / fb_out stages.

* fb_in (get_stage "fb_in"): input_norm_kernel (every norm but offline_laplace_norm), tsse_rowstats_kernel, tsse_norm_kernel and
  tsse_apply_kernel, per clip over frames[b] + look_ahead frames.  Truth and emulation: tests/front_ref.py.
* sub-band input: sb_rowsum_kernel, sb_stats_kernel and the packers.  The sub-band TCN keeps it in fp32 (get_stage "sb_in", Fp32Tm);
  the LSTM / GRU paths read fp16 images (get_stage "sb_img": Fp16Img's SWIZZLE_128B images, Fp16Wide's rows of 128 halves), decoded
  here with the test's own restatement of the swizzle (front_ref.decode_sb_img).  get_stage "sb_mu" is checked against the fp64 mean.
Rule (sb_rnn_ref.compare, factor 1): max |kernel - fp64| <= 3 max |emulation - fp64| + 1e-6 RMS; the fp16 images get one more fp16
spacing at |truth| per element, and values past the fp16 range must be exactly +-65504.  Everything past a clip's extent (frames,
channels >= Isb, rows >= B F, pad tiles) must be exactly zero; the model input past each clip's end is NaN.  One printed line per
case; the last test prints the worst case per stage and per width (DESIGN.md §2).  test_front_end_cpu.py checks that the case lists
reach the edges they claim.
"""
import time

import numpy as np
import pytest
import torch

import front_ref as FR
import sb_rnn_ref as R
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# ---- fb_in cases --------------------------------------------------------------------------------------------------------------------
FB_WIDTHS = [4, 5, 31, 32, 33, 63, 64, 65, 128, 129, 257, 513, 1025, 1548, 1549, 1550, 2048]   # 1548 / 1549: the gate kernel's old limit
TPRIME = [10, 11, 15, 16, 17, 31, 32, 33, 255, 256, 257, 1000]                   # 10: the largest default kersize; 256: rowstats chunk
KERSIZES = [((3, 5, 10), 40), ((1, 2, 16), 40), ((16, 16, 16), 16)]               # (16, 16, 16) at T' = 16: one window
ECA_SUB = [(2, 64), (2, 65), (3, 63), (3, 64), ("half", 64), ("half", 66)]        # (subband_num, F): divisible and not
ROWS_B = [1, 2, 3, 4, 5, 6, 7, 8]                                                  # 3 B 33 = 99 B: every residue mod 8
LONG_T = [14528, 14529, 20000]                                                     # input_norm_kernel's old shared-memory limit
HOUR_FRAMES = 60 * 60 * 16000 // 256 + 1                                          # a 60-minute 16 kHz clip at hop 256
RAGGED_TSSE = [8, 9, 12, 30]                                                       # extents from the TSSE minimum (10) up
RAGGED_SE = [1, 2, 5, 30]

# ---- sub-band input cases ------------------------------------------------------------------------------------------------------------
SB_TCN_NS = [0, 1, 3, 15]
SB_TCN_SHAPES = [(4, 3, 40), (33, 1, 40), (65, 3, 45), (33, 3, 33)]               # (F, Ns, T'): F = 4 at Ns 3, F and T' off 32
SB_IMG_ROWS = [(127, 1), (64, 2), (43, 3), (257, 1)]                               # (F, B): B F = 127, 128, 129, 257
SB_IMG_WIDE = [(66, 32, 0), (128, 63, 0), (64, 63, 0)]                             # (F, Ns, Nf) of fullsubnet.Model: Isb 66, 128; Ns = F - 1

WORST = {}


def _record(stage, width, label, r):
    for key in ((stage,), (stage, width)):
        if r["err"] >= WORST.get(key, (-1.0,))[0]:
            WORST[key] = (r["err"], r["ratio"], label)


def _line(label, r, extra=""):
    print(f"\n[{label}]{extra} max err/RMS {r['err']:.2e} emu {r['emu']:.2e} bound {r['bound']:.2e} ratio {r['ratio']:.2f} "
          f"rel-L2 {r['rel']:.2e}")


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _spectra(B, F, T, seed, kind="plain", scale=1.0):
    """(mag, real, imag) [B, 1, F, T] float32.  kind: "plain" (real / imag with small offsets), "zero_mean" (real / imag centred, so
    the utterance mean and the normaliser of those branches can be negative, and half of the real rows all positive), "constant"
    (every row constant)."""
    rng = np.random.default_rng(seed)
    real = rng.standard_normal((B, 1, F, T)) * 0.05 + 0.004
    imag = rng.standard_normal((B, 1, F, T)) * 0.05 - 0.003
    if kind == "zero_mean":
        real[:, :, ::2] = np.abs(real[:, :, ::2]) + 0.01                  # rows of one sign under a negative normaliser
        real[:, :, 1::2] = -np.abs(real[:, :, 1::2]) - 0.02
        imag -= imag.mean(axis=(1, 2, 3), keepdims=True) + 1e-3
    elif kind == "constant":
        real = np.broadcast_to(real[..., :1], real.shape).copy()
        imag = np.broadcast_to(imag[..., :1], imag.shape).copy()
    real, imag = real * scale, imag * scale
    mag = np.sqrt(real ** 2 + imag ** 2)
    return mag.astype(np.float32), real.astype(np.float32), imag.astype(np.float32)


def _nan_tails(planes, frames):
    if frames is None:
        return planes
    planes = tuple(x.copy() for x in planes)
    for b, n in enumerate(frames):
        for x in planes:
            x[b, :, :, n:] = np.nan
    return planes


def _plus(F, la=2, attn="TSSE", norm="offline_laplace_norm", kersize=(3, 5, 10), sub=1, seq="LSTM", Ns=None, Nf=0, hidden=64,
          impl="auto", seed=0):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    cfg.update(num_freqs=F, look_ahead=la, channel_attention_model=attn, norm_type=norm, kersize=list(kersize), subband_num=sub,
               sequence_model=seq, sb_num_neighbors=(1 if F < 16 else 3) if Ns is None else Ns, fb_num_neighbors=Nf,
               sb_model_hidden_size=hidden)
    params = O.make_params_plus(cfg, seed=seed) if seq != "TCN" else _sbtcn_params(cfg, seed)
    m = FullSubNet_Plus(**cfg, lstm_impl=impl) if seq != "TCN" else FullSubNet_Plus(**cfg)
    return _load(m, params), params, cfg


def _sbtcn_params(cfg, seed):
    import sbtcn_oracle as S
    return S.make_params(cfg, seed=seed)


def _fsn(F, la=2, norm="offline_laplace_norm", Ns=None, Nf=0, hidden=64, fb_hidden=64, impl="auto", seed=0, default=False, edit=None):
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    if not default:
        cfg.update(num_freqs=F, look_ahead=la, sb_num_neighbors=(1 if F < 16 else 3) if Ns is None else Ns, fb_num_neighbors=Nf,
                   sb_model_hidden_size=hidden, fb_model_hidden_size=fb_hidden)
    cfg.update(norm_type=norm)
    params = O.make_params_fsn(cfg, seed=seed)
    if edit:
        edit(params)
    return _load(Model(**cfg, lstm_impl=impl), params), params, cfg


def _load(m, params):
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    return m


def _run(m, planes, frames):
    with torch.no_grad():
        return m(*(_t(x) for x in _nan_tails(planes, frames)), frames=frames)


# ---- fb_in ----------------------------------------------------------------------------------------------------------------------------
def _fb_in_check(label, m, params, cfg, planes, frames=None, width=None, record=True):
    nbr = len(planes)
    B, _, F, T = planes[0].shape
    la = cfg["look_ahead"]
    Tp = T + la
    got = m.get_stage("fb_in", (nbr, B, F, Tp), DEV).cpu().double().numpy()
    acfg = cfg if nbr == 3 else {k: v for k, v in cfg.items() if k != "channel_attention_model"}
    want = FR.fb_in_truth(params, acfg, planes, frames)
    emu = FR.fb_in_emulate(params, acfg, planes, frames)
    ext = FR.clip_extents(B, Tp, la, frames)
    valid = np.arange(Tp)[None, None, None, :] < np.asarray(ext)[None, :, None, None]
    valid = np.broadcast_to(valid, got.shape)
    assert (got[~valid] == 0).all(), f"{label}: fb_in past a clip's extent is not zero"
    r = R.compare(torch.from_numpy(got), torch.from_numpy(want), torch.from_numpy(emu.astype(np.float64)), 1.0,
                  torch.from_numpy(np.ascontiguousarray(valid)))
    _line(label, r, f" F={F} B={B} T'={Tp} {cfg['norm_type']}:")
    if record:
        _record("fb_in", F if width is None else width, label, r)
    assert r["finite"], label
    assert r["ok"], (label, r)
    return r


def _fb_case(label, F, B, T, la=2, frames=None, spectra="plain", seed=0, width=None, record=True, **kw):
    m, params, cfg = _plus(F, la=la, seed=seed, **kw)
    planes = _spectra(B, F, T, seed + 1, spectra)
    _run(m, planes, frames)
    return _fb_in_check(label, m, params, cfg, planes, frames, width, record)


@pytest.mark.parametrize("F", FB_WIDTHS)
def test_fb_in_widths(built_lib, F):
    _fb_case(f"width {F}", F, 2, 22 if F >= 1025 else 38, seed=F)


@pytest.mark.parametrize("la", [0, 2])
@pytest.mark.parametrize("Tp", TPRIME)
def test_fb_in_clip_lengths(built_lib, Tp, la):
    _fb_case(f"T'={Tp} la={la}", 33, 2, Tp - la, la=la, seed=Tp + la, width="T'")


@pytest.mark.parametrize("ks,Tp", KERSIZES)
def test_fb_in_kernel_sizes(built_lib, ks, Tp):
    _fb_case(f"kersize {ks} T'={Tp}", 37, 2, Tp - 2, kersize=ks, seed=sum(ks), width="kersize")


@pytest.mark.parametrize("attn", ["TSSE", "SE", "CBAM", "ECA"])
@pytest.mark.parametrize("spectra", ["plain", "zero_mean", "constant"])
def test_fb_in_attention(built_lib, attn, spectra):
    _fb_case(f"{attn} {spectra}", 37, 2, 40, attn=attn, spectra=spectra, seed=len(attn), width=attn)


@pytest.mark.parametrize("sub,F", ECA_SUB)
def test_fb_in_eca_subband_num(built_lib, sub, F):
    s = F // 2 if sub == "half" else sub
    _fb_case(f"ECA subband_num {s} F={F}", F, 2, 30, attn="ECA", sub=s, seed=s + F, width="ECA sub")


@pytest.mark.parametrize("kind", ["plus", "fsn"])
@pytest.mark.parametrize("norm", FR.NORMS)
def test_fb_in_norm_types(built_lib, kind, norm):
    F, B, T = 33, 2, 60
    if kind == "plus":
        _fb_case(f"plus {norm}", F, B, T, norm=norm, spectra="zero_mean", seed=3, width=norm)
    else:
        m, params, cfg = _fsn(F, norm=norm, seed=4)
        planes = _spectra(B, F, T, 5)[:1]
        _run(m, planes, None)
        _fb_in_check(f"fsn {norm}", m, params, cfg, planes, width=norm)


@pytest.mark.parametrize("B", ROWS_B)
def test_fb_in_row_residues(built_lib, B):
    _fb_case(f"rows 3*B*F={3 * B * 33}", 33, B, 20, seed=B, width="rows")


@pytest.mark.parametrize("attn,frames", [("TSSE", RAGGED_TSSE), ("SE", RAGGED_SE), ("CBAM", RAGGED_SE)])
@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_layer_norm"])
def test_fb_in_ragged(built_lib, attn, frames, norm):
    T = 40
    _fb_case(f"ragged {attn} {norm}", 33, len(frames) + 1, T, frames=frames + [T], attn=attn, norm=norm, spectra="zero_mean",
             seed=7 + len(attn), width="ragged")


def test_fb_in_loud_clip(built_lib):
    """x30 speech with zero-mean real / imaginary parts: the normalised streams reach ~1e8"""
    cfg = O.default_plus_config()
    X = 30.0 * O.stft(O.synth_clips(2, seed0=4321))
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    real -= real.mean(axis=(1, 2, 3), keepdims=True)
    imag -= imag.mean(axis=(1, 2, 3), keepdims=True)
    m, params, cfg = _plus(257, hidden=64, seed=0)
    _run(m, (mag, real, imag), None)
    _fb_in_check("loud zero-mean clip", m, params, cfg, (mag, real, imag), width="loud")


@pytest.mark.parametrize("norm", ["cumulative_laplace_norm", "offline_gaussian_norm", "cumulative_layer_norm"])
@pytest.mark.parametrize("Tp", LONG_T)
def test_fb_in_long_clips(built_lib, Tp, norm):
    _fb_case(f"long T'={Tp} {norm}", 33, 1, Tp - 2, norm=norm, attn="SE", seed=Tp % 97, width="long")


def test_fb_in_hour_cumulative_laplace(built_lib):
    """One 60-minute clip through fullsubnet.Model (default geometry) with cumulative_laplace_norm: fb_in against fp64 in row chunks."""
    m, params, cfg = _fsn(257, norm="cumulative_laplace_norm", default=True, seed=11)
    T = HOUR_FRAMES
    rng = np.random.default_rng(12)
    mag = (np.abs(rng.standard_normal((1, 1, 257, T))) * 0.05 + 1e-3).astype(np.float32)
    t0 = time.perf_counter()
    _run(m, (mag,), None)
    torch.cuda.synchronize()
    sec = time.perf_counter() - t0
    Tp = T + cfg["look_ahead"]
    got = m.get_stage("fb_in", (1, 1, 257, Tp), DEV)[0, 0]
    x = np.zeros((257, Tp), np.float32)
    x[:, :T] = mag[0, 0]
    cm = np.cumsum(x.astype(np.float64).sum(axis=0)) / (257.0 * np.arange(1, Tp + 1))     # fp64 truth of the running mean
    sa32 = (1.0 / (np.cumsum(FR.seq_sum(x, 0).astype(np.float64)) / (257.0 * np.arange(1, Tp + 1)) + FR.EPS_F32)).astype(np.float32)
    err = eerr = ss = 0.0
    for r0 in range(0, 257, 32):
        want = x[r0:r0 + 32].astype(np.float64) / (cm + FR.EPS_F32)
        emu = (x[r0:r0 + 32] * sa32).astype(np.float64)
        g = got[r0:r0 + 32].cpu().double().numpy()
        err, eerr = max(err, float(np.abs(g - want).max())), max(eerr, float(np.abs(emu - want).max()))
        ss += float((want ** 2).sum())
    rms = (ss / (257 * Tp)) ** 0.5
    bound = 3 * eerr + 1e-6 * rms
    r = dict(err=err / rms, emu=eerr / rms, bound=bound / rms, ratio=err / max(eerr, 1e-300), rel=float("nan"))
    _line("60-minute clip", r, f" fsn cumulative_laplace_norm T'={Tp} forward {sec:.1f} s:")
    _record("fb_in", "60 min", "60-minute clip", r)
    assert err <= bound, r


# ---- sub-band input: TCN path (sb_in) ---------------------------------------------------------------------------------------------
def _sb_sources(m, cfg, kind, B, F, Tp, planes, frames=None):
    nbr = 3 if kind == "plus" else 1
    fb_in = m.get_stage("fb_in", (nbr, B, F, Tp), DEV).cpu().numpy()
    fb_out = m.get_stage("fb_out", (nbr, B, F, Tp), DEV).cpu().numpy()
    if kind == "plus":
        return fb_in[0], list(fb_out)
    win = np.zeros((B, F, Tp), np.float32)                               # the padded magnitude (fullsubnet.py:81,94)
    for b, n in enumerate([Tp - cfg["look_ahead"]] * B if frames is None else frames):
        win[b, :, :n] = planes[0][b, 0, :, :n]
    return win, [fb_out[0]]


def _zero_tails(win, fbs, frames, la):
    """the sources as the packer reads them: nothing past a clip's extent (the full-band outputs are finite there but unread)"""
    if frames is None:
        return win, fbs
    win, fbs = win.copy(), [o.copy() for o in fbs]
    for b, n in enumerate(frames):
        for x in [win] + fbs:
            x[b, :, n + la:] = 0
    return win, fbs


def _sb_truth(m, cfg, kind, planes, frames):
    B, _, F, T = planes[0].shape
    Tp = T + cfg["look_ahead"]
    win, fbs = _zero_tails(*_sb_sources(m, cfg, kind, B, F, Tp, planes, frames), frames, cfg["look_ahead"])
    want, mu_t = FR.sb_in_truth(cfg, win, fbs, frames)
    emu, mu_e = FR.sb_in_emulate(cfg, win, fbs, frames)
    mu = m.get_stage("sb_mu", (B,), DEV).cpu().double().numpy()
    assert (np.abs(mu - mu_t) <= 3 * np.abs(mu_e - mu_t) + 1e-6 * np.abs(mu_t)).all(), ("sb_mu", mu, mu_t, mu_e)
    return want, emu


def _valid_sb(B, F, I, Tp, ext):
    return np.broadcast_to(np.arange(Tp)[None, None, None, :] < np.asarray(ext)[:, None, None, None], (B, F, I, Tp))


def _sb_tcn_case(label, F, Ns, Tp, norm, B=2, frames=None, seed=0, width=None):
    m, params, cfg = _plus(F, Ns=Ns, seq="TCN", norm=norm, attn="SE", seed=seed)
    planes = _spectra(B, F, Tp - 2, seed + 1)
    _run(m, planes, frames)
    assert m.last_lstm_impl() == "tcn"
    I = FR.isb(cfg, 3)
    got = m.get_stage("sb_in", (B, F, I, Tp), DEV).cpu().double().numpy()
    want, emu = _sb_truth(m, cfg, "plus", planes, frames)
    valid = _valid_sb(B, F, I, Tp, FR.clip_extents(B, Tp, 2, frames))
    assert (got[~valid] == 0).all(), f"{label}: sb_in past a clip's extent is not zero"
    r = R.compare(torch.from_numpy(got), torch.from_numpy(want), torch.from_numpy(emu.astype(np.float64)), 1.0,
                  torch.from_numpy(np.ascontiguousarray(valid)))
    _line(label, r, f" F={F} Isb={I} B={B} T'={Tp} {norm}:")
    _record("sb_in (TCN)", I if width is None else width, label, r)
    assert r["finite"] and r["ok"], (label, r)


@pytest.mark.parametrize("norm", FR.NORMS)
@pytest.mark.parametrize("Ns", SB_TCN_NS)
def test_sb_in_tcn_norms(built_lib, Ns, norm):
    _sb_tcn_case(f"sb_in Ns={Ns} {norm}", 33, Ns, 42, norm, seed=Ns)


@pytest.mark.parametrize("F,Ns,Tp", SB_TCN_SHAPES)
def test_sb_in_tcn_shapes(built_lib, F, Ns, Tp):
    _sb_tcn_case(f"sb_in F={F} Ns={Ns} T'={Tp}", F, Ns, Tp, "offline_laplace_norm", seed=F + Tp)


@pytest.mark.parametrize("norm", ["offline_gaussian_norm", "cumulative_layer_norm"])
def test_sb_in_tcn_ragged(built_lib, norm):
    T = 40
    frames = RAGGED_SE + [T]
    _sb_tcn_case(f"sb_in ragged {norm}", 33, 3, T + 2, norm, B=len(frames), frames=frames, seed=9, width="ragged")


# ---- sub-band input: LSTM / GRU paths (sb_img) --------------------------------------------------------------------------------------
def _img_layout(m, I):
    if I <= 64:
        return "sw128"
    return "wide_layerwise" if m.last_lstm_impl() == "tcgen05" else "wide_tm"


def _img_case(label, kind, F, B, Tp, norm, impl, Ns=None, Nf=0, frames=None, seed=0, width=None, planes=None, lift_fb=False):
    la = 2
    if kind == "plus":
        m, params, cfg = _plus(F, Ns=Ns, Nf=Nf, norm=norm, impl=impl, attn="SE", seed=seed)
    else:
        def silence(p):                                                  # fb_out = ReLU(-100) = 0: the magnitude alone sets the mean
            p["fb_model.fc_output_layer.bias"] = np.full_like(p["fb_model.fc_output_layer.bias"], -100.0)
        m, params, cfg = _fsn(F, Ns=Ns, Nf=Nf, norm=norm, impl=impl, seed=seed, edit=silence if lift_fb else None)
    if planes is None:
        planes = _spectra(B, F, Tp - la, seed + 1)
        planes = planes if kind == "plus" else planes[:1]
    _run(m, planes, frames)
    impl_ran = m.last_lstm_impl()
    assert impl_ran == ("tcgen05" if impl == "auto" else "mma"), impl_ran
    nfb = 3 if kind == "plus" else 1
    I = FR.isb(cfg, nfb)
    rows = B * F
    nbytes = FR.img_bytes(rows, Tp, I > 64)
    raw = m.get_stage("sb_img", (nbytes // 4,), DEV).cpu().numpy().view(np.uint8)
    layout = _img_layout(m, I)
    vals, rest = FR.decode_sb_img(raw, rows, Tp, I, layout)
    assert (rest == 0).all(), f"{label}: the images are not zero outside the sub-band input ({np.count_nonzero(rest)} elements)"
    got = vals.astype(np.float64).reshape(B, F, I, Tp)
    want, emu = _sb_truth(m, cfg, kind, planes, frames)
    valid = _valid_sb(B, F, I, Tp, FR.clip_extents(B, Tp, la, frames))
    assert (got[~valid] == 0).all(), f"{label}: images past a clip's extent are not zero"
    over = valid & (np.abs(emu) > 65504)
    assert (got[over] == np.sign(emu[over]) * 65504).all(), f"{label}: out-of-range values are not clamped to +-65504"
    sel = valid & ~over
    g, w, e = got[sel], want[sel], emu[sel].astype(np.float64)
    rms = float(np.sqrt((w ** 2).mean())) or 1.0
    eerr = float(np.abs(e - w).max())
    bound = 3 * eerr + 1e-6 * rms + FR.fp16_spacing(w)
    err = np.abs(g - w)
    r = dict(err=float(err.max()) / rms, emu=eerr / rms, bound=float((3 * eerr + 1e-6 * rms + FR.fp16_spacing(w).max())) / rms,
             ratio=float(err.max()) / max(eerr, 1e-300), rel=float(np.linalg.norm(g - w) / max(np.linalg.norm(w), 1e-300)))
    _line(label, r, f" {kind} {layout} {impl_ran} F={F} Isb={I} B*F={rows} T'={Tp} {norm} clamped {int(over.sum())}:")
    _record(f"sb_img {layout}", I if width is None else width, label, r)
    assert (err <= bound).all(), (label, r, int((err > bound).sum()))
    return int(over.sum())


@pytest.mark.parametrize("impl", ["auto", "mma"])
@pytest.mark.parametrize("norm", FR.NORMS)
def test_sb_img_norms(built_lib, norm, impl):
    _img_case(f"sb_img {norm} {impl}", "plus", 33, 2, 42, norm, impl, Ns=3, seed=20)


@pytest.mark.parametrize("impl", ["auto", "mma"])
@pytest.mark.parametrize("F,B", SB_IMG_ROWS)
def test_sb_img_rows(built_lib, F, B, impl):
    _img_case(f"sb_img B*F={B * F} {impl}", "plus", F, B, 35, "offline_laplace_norm", impl, Ns=3, seed=F + B, width="rows")


@pytest.mark.parametrize("impl", ["auto", "mma"])
@pytest.mark.parametrize("norm", FR.NORMS)
@pytest.mark.parametrize("F,Ns,Nf", SB_IMG_WIDE)
def test_sb_img_wide(built_lib, F, Ns, Nf, norm, impl):
    _img_case(f"sb_img wide F={F} Ns={Ns} {norm} {impl}", "fsn", F, 2, 36, norm, impl, Ns=Ns, Nf=Nf, seed=Ns + len(norm))


@pytest.mark.parametrize("impl", ["auto", "mma"])
@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm"])
def test_sb_img_ragged(built_lib, norm, impl):
    T = 40
    frames = RAGGED_SE + [T]
    _img_case(f"sb_img ragged {norm} {impl}", "plus", 33, len(frames), T + 2, norm, impl, Ns=3, frames=frames, seed=30,
              width="ragged")
    _img_case(f"sb_img wide ragged {norm} {impl}", "fsn", 66, len(frames), T + 2, norm, impl, Ns=32, frames=frames, seed=31,
              width="ragged")


def test_sb_img_clamp(built_lib):
    """One loud bin in an otherwise quiet magnitude, the full-band output held at zero: x / (mean + 1e-5) reaches ~1.2e5 there, past
    the fp16 range, and must be stored as exactly 65504."""
    F, B, T = 257, 1, 498
    mag = np.full((B, 1, F, T), 1e-6, np.float32)
    mag[0, 0, 100, 200] = 10.0
    n = _img_case("sb_img clamp", "fsn", F, B, T + 2, "offline_laplace_norm", "auto", Ns=15, seed=40, planes=(mag,), lift_fb=True,
                  width="clamp")
    assert n > 0, "no value passed the fp16 range: the clamp was not exercised"


def test_sb_img_refused(built_lib, monkeypatch):
    """sb_img: FSN_EINVAL on the TCN path, FSN_ESTATE after a windowed forward"""
    from fsnplus_b200 import _lib
    m, _, _ = _plus(33, seq="TCN", attn="SE", seed=50)
    _run(m, _spectra(1, 33, 30, 51), None)
    with pytest.raises(_lib.FsnError, match="error -?\\d+: sb_img is the LSTM"):
        m.get_stage("sb_img", (FR.img_bytes(33, 32, False) // 4,), DEV)
    monkeypatch.setenv("FSN_SB_WINDOW", "32")
    m, _, _ = _plus(33, seed=52)
    monkeypatch.delenv("FSN_SB_WINDOW")
    _run(m, _spectra(1, 33, 100, 53), None)
    assert m.last_plan()[1] == 32, m.last_plan()
    with pytest.raises(_lib.FsnError, match="sb_img is not kept"):
        m.get_stage("sb_img", (FR.img_bytes(33, 102, False) // 4,), DEV)


def test_zz_worst_per_stage(built_lib):
    """The tables DESIGN.md §2 quotes: worst max err / RMS per stage, and per stage and width."""
    if not WORST:
        pytest.skip("no case of this file ran before")
    print("\nworst max err / RMS (ratio to the emulation's error, case):")
    for key in sorted(WORST, key=str):
        e, ratio, label = WORST[key]
        print(f"  {' / '.join(map(str, key)):40} {e:.2e}  x{ratio:.2f}  {label}")
