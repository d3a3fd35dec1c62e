"""The full-band models and the sub-band TCN against fp64, element by element.

Each truth is computed from the kernel's own stage input, so only the stage under test contributes error:
  * full-band TCN of FullSubNet_Plus: fb_in -> fb_out.  fb_in (get_stage) is the fp32 output of tsse_apply_kernel (k_front.cu), which
    writes the time-major copy the first TCN GEMM reads (out_tm) from the same value v as the [branch, B, F, P] copy get_stage returns;
    block 0's store scale comes from the same gate kernel.  Truth and emulation: tests/tcn_ref.py, per branch ("fb_model",
    "fb_model_real", "fb_model_imag"), compared on every clip's valid frames; the frames past a ragged clip's end must be finite.
  * sub-band TCN (sequence_model = "TCN"): sb_in -> mask, sampled rows (sb_rnn_ref.sample_rows);
  * full-band LSTM / GRU of fullsubnet.Model: fb_in -> fb_out (sb_rnn_ref with prefix "fb_model", head "fb"), on the weight-stationary
    kernel or lstm_mma_kernel; which one ran is read back (fsn_model_last_fb_ws) and checked against ws_eligible, a restatement of
    lstm_ws_supported (k_lstm_ws.cu).
Rule (sb_rnn_ref.compare): max |kernel - fp64| <= factor * (3 max |emulation - fp64| + 1e-6 RMS); factor tcn_ref.TCN_FACTOR for the TCNs,
1 / sb_rnn_ref.FAST_FACTOR for accurate / fast LSTM math.  One printed line per case: max err / RMS, the emulation's, the bound, their
ratio and the rel-L2; the last test prints the worst case per stage and per width (DESIGN.md §2).  test_full_band_cpu.py checks that
the case lists reach the edges they claim.
"""

import numpy as np
import pytest
import torch

import sb_rnn_ref as R
import sbtcn_oracle as S
import tcn_ref as TR
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FB_PREFIXES = ("fb_model", "fb_model_real", "fb_model_imag")

# ---- full-band TCN (FullSubNet_Plus): (F, B, T') -------------------------------------------------------------------------------
FB_WIDTHS = [4, 31, 32, 33, 64, 65, 96, 128, 129, 257, 513, 1025, 2048]           # Cp 32 / 64 (NT 64) .. 2048 (16 N tiles)
FB_ROWS = [(64, 1, 127), (64, 1, 128), (64, 1, 129), (65, 3, 43)]                   # B T' = 127 / 128 / 129; groups straddling tiles
FB_WAVES = (257, 64, 60)                                                            # 30 M tiles x 4 N tiles x 3 branches > 2 x 132
TPRIME = [1, 2, 3, 5, 9, 10, 18, 19, 255, 256, 257, 274, 275, 1000]
FB_TPRIME = [(Tp, 0 if Tp < 3 or i % 2 else 2, causal) for i, Tp in enumerate(TPRIME) for causal in (False, True)]
RAGGED = [1, 3, 9, 10, 19]                                                          # next to a full-length clip
ACTS = [None, "ReLU", "Tanh", "ReLU6"]
TSSE_MIN = 10                                                                       # the TSSE kernel sizes (3, 5, 10)

# ---- sub-band TCN: (Ns, Nf) -> Isb, and T' ---------------------------------------------------------------------------------------
SB_ISB = [(1, 0), (15, 0), (30, 0)]                                                 # Isb 6, 34, 64
SB_TPRIME = [(Tp, 0 if Tp < 3 or i % 2 else 2) for i, Tp in enumerate(TPRIME)]
SB_GROUPS = (257, 256, 3)                                                           # (F, B, T'): B F = 65792 > 65535 groups

# ---- fullsubnet.Model full band: (B, H, L, cell, fast, F) -----------------------------------------------------------------------
WS = [(1, 16, 1, "LSTM", True, 4), (2, 48, 2, "GRU", False, 33), (63, 64, 3, "LSTM", True, 257), (64, 256, 4, "GRU", True, 33),
      (2, 512, 2, "LSTM", False, 257), (64, 528, 2, "LSTM", True, 257), (1, 528, 1, "GRU", False, 513), (63, 256, 3, "GRU", False, 513),
      (2, 64, 4, "LSTM", False, 4), (1, 256, 1, "LSTM", True, 513)]
MMA = [(65, 256, 2, "LSTM", True, 257), (130, 64, 3, "GRU", False, 33)]             # rows > 64: lstm_mma_kernel
WS_LIMIT_LH = (2, 512)                                                              # the largest F that fits at (L, H) and the next
FSN_TPRIME = [(1, 0), (2, 0), (190, 2), (2000, 2)]                                  # (T', look_ahead)

WORST = {}


# ------------------------------------------------------------------------------------------------------------------------------------
def ws_smem(L, H, Ipad):
    """k_lstm_ws.cu ws_smem: the weight-stationary kernel's shared memory in bytes"""
    halves = sum(16 * ((Ipad if l == 0 else H) + H + 8) for l in range(L)) + 64 * (max(Ipad, H) + H + 8)
    return 2 * halves


def ws_eligible(L, H, F, rows, num_sms):
    """k_lstm_ws.cu lstm_ws_supported with Ipad = F rounded up to 16 (forward_impl)"""
    Ipad = (F + 15) // 16 * 16
    return 1 <= L <= 4 and rows <= 64 and H % 16 == 0 and H // 4 <= num_sms and ws_smem(L, H, Ipad) <= 227 * 1024


def ws_limit_widths(L, H):
    """(largest F whose ws_smem fits, the next F) at (L, H)"""
    F = max(f for f in range(1, 4097) if ws_smem(L, H, (f + 15) // 16 * 16) <= 227 * 1024)
    return F, F + 1


def tcn_tiles(F):
    """pack_tcn5 / pack_tcn_blocks: (Cp, NT, N tiles) of the full band's Cp-wide GEMMs"""
    Cp = (F + 31) // 32 * 32
    NT = 64 if Cp <= 64 else 128
    return Cp, NT, (Cp + NT - 1) // NT


def _num_sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _record(stage, width, label, r):
    for key in ((stage,), (stage, width)):
        if r["err"] >= WORST.get(key, (-1.0,))[0]:
            WORST[key] = (r["err"], r["ratio"], label)


def _line(label, r, extra=""):
    print(f"\n[{label}]{extra} max err/RMS {r['err']:.2e} emu {r['emu']:.2e} bound {r['bound']:.2e} ratio {r['ratio']:.2f} "
          f"rel-L2 {r['rel']:.2e}")


def _load(m, params):
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))          # the C handle reads the FSN_* knobs once, here
    return m


def _spectra(B, F, T, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    real = (rng.standard_normal((B, 1, F, T)) * 0.05 + 0.004) * scale
    imag = (rng.standard_normal((B, 1, F, T)) * 0.05 - 0.003) * scale
    return np.sqrt(real ** 2 + imag ** 2).astype(np.float32), real.astype(np.float32), imag.astype(np.float32)


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _valid(frames, la, n, Tp):
    """[n, 1, Tp] bool: the frames each clip's stage computes (frames[b] + look_ahead), all when frames is None"""
    tl = torch.full((n,), Tp) if frames is None else torch.as_tensor([f + la for f in frames])
    return torch.arange(Tp)[None, None, :] < tl[:, None, None], (None if frames is None else tl)


# ---- full-band TCN ------------------------------------------------------------------------------------------------------------------
def _plus_cfg(F, la=2, attn="TSSE", act="ReLU", causal=False, **over):
    c = O.default_plus_config()
    c.update(num_freqs=F, look_ahead=la, channel_attention_model=attn, fb_output_activate_function=act, sb_num_neighbors=1 if F < 16 else 3,
             sb_model_hidden_size=64, causal_tcn=causal)
    c.update(over)
    return c


def _fb_tcn_case(label, cfg, B, Tp, seed=0, frames=None, wscale=1.0, inputs=None, params=None, clips=None, record=True, width=None):
    """One FullSubNet_Plus forward; each branch's fb_out against the truth from its own fb_in.  clips: the clips compared (all)."""
    from fsnplus_b200.model import FullSubNet_Plus
    F, la = cfg["num_freqs"], cfg["look_ahead"]
    T = Tp - la
    if params is None:
        params = O.make_params_plus(cfg, seed=seed)
    TR.distinct_slopes(params, FB_PREFIXES)
    for k in params:
        if k.startswith("fb_model") and (".conv1x1." in k or ".sconv." in k):
            params[k] = params[k] * np.float32(wscale)
    m = _load(FullSubNet_Plus(**cfg), params)
    mag, real, imag = inputs if inputs is not None else _spectra(B, F, T, seed + 1)
    if frames is not None:                                           # NaN past each clip's end: never read
        mag, real, imag = (x.copy() for x in (mag, real, imag))
        for b, n in enumerate(frames):
            for x in (mag, real, imag):
                x[b, :, :, n:] = np.nan
    with torch.no_grad():
        m(_t(mag), _t(real), _t(imag), frames=frames)
    fb_in = m.get_stage("fb_in", (3, B, F, Tp), DEV)
    fb_out = m.get_stage("fb_out", (3, B, F, Tp), DEV)
    torch.cuda.synchronize()
    clips = list(range(B)) if clips is None else clips
    sel = torch.as_tensor(clips, device=DEV)
    valid, tl = _valid(None if frames is None else [frames[c] for c in clips], la, len(clips), Tp)
    mask = valid.expand(len(clips), F, Tp)
    assert torch.isfinite(fb_out).all(), f"{label}: non-finite full-band output (also past the clips' ends)"
    dev = DEV if len(clips) * Tp * max(F, 64) > 2e4 else "cpu"
    tld = None if tl is None else tl.to(dev)
    worst = None
    for br, pre in enumerate(FB_PREFIXES):
        x = fb_in[br][sel].to(dev)
        want = TR.truth(params, pre, x, tld, cfg["causal_tcn"], "fb", cfg["fb_output_activate_function"], device=dev)
        emu = TR.emulate(params, pre, x, tld, cfg["causal_tcn"], "fb", cfg["fb_output_activate_function"], device=dev)
        r = R.compare(fb_out[br][sel], want, emu, TR.TCN_FACTOR, mask)
        assert r["ok"], (label, pre, r)
        if worst is None or r["err"] > worst[1]["err"]:
            worst = (pre, r)
    pre, r = worst
    Cp, NT, nt = tcn_tiles(F)
    _line(label, r, f" F={F} Cp={Cp} NT={NT}x{nt} B={B} T'={Tp}{' causal' if cfg['causal_tcn'] else ''} worst branch {pre}:")
    if record:
        _record("full-band TCN", width if width is not None else F, label, r)
    return m, params


@pytest.mark.parametrize("F", FB_WIDTHS)
def test_fb_tcn_widths(built_lib, F):
    Tp = 24 if F >= 1025 else 40
    _fb_tcn_case(f"width {F}", _plus_cfg(F), 2, Tp, seed=F)


@pytest.mark.parametrize("F,B,Tp", FB_ROWS)
def test_fb_tcn_row_tiles(built_lib, F, B, Tp):
    _fb_tcn_case(f"rows B*T'={B * Tp}", _plus_cfg(F), B, Tp, seed=B * Tp)


def test_fb_tcn_more_than_two_waves(built_lib):
    """64 clips of 60 frames at F = 257; clips 0, 1, 31, 62, 63 and five random ones compared whole (gLN is per clip)."""
    F, B, Tp = FB_WAVES
    clips = sorted({0, 1, 31, 62, 63, *np.random.default_rng(0).choice(B, 5, replace=False).tolist()})
    _fb_tcn_case("waves", _plus_cfg(F), B, Tp, seed=5, clips=clips)


@pytest.mark.parametrize("Tp,la,causal", FB_TPRIME)
def test_fb_tcn_clip_lengths(built_lib, Tp, la, causal):
    cfg = _plus_cfg(64, la=la, attn="TSSE" if Tp >= TSSE_MIN else "SE", causal=causal)
    _fb_tcn_case(f"T'={Tp} la={la}{' causal' if causal else ''}", cfg, 2, Tp, seed=Tp + causal)


@pytest.mark.parametrize("causal", [False, True])
def test_fb_tcn_ragged(built_lib, causal):
    """Clips of 1, 3, 9, 10 and 19 frames next to a full-length one, NaN past each end (SE attention: TSSE needs 10 frames)."""
    T = 40
    cfg = _plus_cfg(65, attn="SE", causal=causal)
    _fb_tcn_case(f"ragged{' causal' if causal else ''}", cfg, len(RAGGED) + 1, T + 2, seed=21 + causal, frames=RAGGED + [T])


def test_fb_tcn_loud_zero_mean_clip(built_lib):
    """test_plus_extreme_real_imag_scale's clip: x30 with zero-mean real / imaginary parts, normalised streams ~1e8."""
    cfg = dict(O.default_plus_config(), causal_tcn=False)
    X = 30.0 * O.stft(O.synth_clips(2, seed0=4321))
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    real -= real.mean(axis=(1, 2, 3), keepdims=True)
    imag -= imag.mean(axis=(1, 2, 3), keepdims=True)
    T = mag.shape[-1]
    m, _ = _fb_tcn_case("loud zero-mean clip", cfg, 2, T + 2, seed=0, inputs=(mag, real, imag), width="loud")
    peak = float(m.get_stage("fb_in", (3, 2, 257, T + 2), DEV).abs().max())
    print(f"  fb_in peak {peak:.2e}")
    assert peak > 1e7


def test_fb_tcn_small_amplitude(built_lib):
    """SE gates near 6e-6 (fc2 bias -12): every stream max |x| < 1, so the store scale is 1 and the fp16 hidden activation reaches
    the subnormal range.  Left out of the worst-case table (a format question, DESIGN.md §5)."""
    cfg = _plus_cfg(64, attn="SE")
    params = O.make_params_plus(cfg, seed=31)
    for s in ("", "_real", "_imag"):
        params[f"channel_attention{s}.fc2.bias"] = np.full_like(params[f"channel_attention{s}.fc2.bias"], -12.0)
    m, _ = _fb_tcn_case("small amplitude", cfg, 2, 40, seed=31, params=params, record=False)
    amax = float(m.get_stage("fb_in", (3, 2, 64, 40), DEV).abs().max())
    print(f"  fb_in max |x| {amax:.2e}")
    assert amax < 1


def test_fb_tcn_weights_x3(built_lib):
    _fb_tcn_case("conv weights x3", _plus_cfg(129), 2, 60, seed=33, wscale=3.0, width="x3")


@pytest.mark.parametrize("act", ACTS)
def test_fb_tcn_activations(built_lib, act):
    _fb_tcn_case(f"act {act}", _plus_cfg(64, act=act), 2, 40, seed=41, record=act in (None, "Tanh"))


# ---- sub-band TCN ---------------------------------------------------------------------------------------------------------------------
def _sb_cfg(F=33, Ns=1, Nf=0, la=2, attn="TSSE", act=False):
    c = O.default_plus_config()
    c.update(num_freqs=F, sb_num_neighbors=Ns, fb_num_neighbors=Nf, look_ahead=la, channel_attention_model=attn, sequence_model="TCN",
             sb_output_activate_function=act, sb_model_hidden_size=32)
    return c


def _sb_model(cfg, seed):
    from fsnplus_b200.model import FullSubNet_Plus
    params = S.make_params(cfg, seed=seed)
    for blk in range(8):                                             # slopes that differ per block, as in distinct_slopes
        for j, name in enumerate(("prelu1", "prelu2")):
            params[f"sb_model.sequence_model.{blk}.{name}.weight"] = np.array([0.07 + 0.03 * blk + 0.1 * j], np.float32)
    return _load(FullSubNet_Plus(**cfg), params), params


def _sb_check(label, m, params, cfg, B, Tp, mask_out, frames=None, record=True, sb_in=None):
    """mask_out [B, O, F, T] against the truth from sb_in (this forward's unless given) on sampled rows"""
    F, la = cfg["num_freqs"], cfg["look_ahead"]
    I = S.isb(cfg)
    if sb_in is None:
        sb_in = m.get_stage("sb_in", (B, F, I, Tp), DEV)
    rows = R.sample_rows(B * F)
    ridx = torch.as_tensor(rows, device=DEV)
    dev = DEV if len(rows) * Tp > 2e3 else "cpu"
    x = sb_in.reshape(B * F, I, Tp)[ridx].to(dev)
    tl = None if frames is None else torch.as_tensor([frames[r // F] + la for r in rows], device=dev)
    act = cfg["sb_output_activate_function"]
    want = TR.truth(params, "sb_model", x, tl, False, "sb", act, la, device=dev)
    emu = TR.emulate(params, "sb_model", x, tl, False, "sb", act, la, device=dev)
    O_ = mask_out.shape[1]
    got = mask_out.permute(0, 2, 1, 3).reshape(B * F, O_, Tp - la)[ridx]
    mask = None
    if frames is not None:
        fr = torch.as_tensor([frames[r // F] for r in rows])
        mask = (torch.arange(Tp - la)[None, None, :] < fr[:, None, None]).expand(len(rows), O_, Tp - la)
    r = R.compare(got, want, emu, TR.TCN_FACTOR, mask)
    _line(label, r, f" Isb={I} rows {len(rows)}/{B * F} T'={Tp}:")
    if record:
        _record("sub-band TCN", I, label, r)
    assert r["finite"], label
    assert r["ok"], (label, r)
    return want, rows


def _sb_case(label, cfg, B, Tp, seed, frames=None, record=True):
    m, params = _sb_model(cfg, seed)
    F = cfg["num_freqs"]
    mag, real, imag = _spectra(B, F, Tp - cfg["look_ahead"], seed + 1)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag), frames=frames)
    assert m.last_lstm_impl() == "tcn"
    _sb_check(label, m, params, cfg, B, Tp, out, frames=frames, record=record)
    return m, params, (mag, real, imag), out


@pytest.mark.parametrize("Ns,Nf", SB_ISB)
def test_sb_tcn_input_widths(built_lib, Ns, Nf):
    cfg = _sb_cfg(F=64, Ns=Ns, Nf=Nf)
    _sb_case(f"sb Isb={S.isb(cfg)}", cfg, 2, 40, seed=50 + Ns)


@pytest.mark.parametrize("Tp,la", SB_TPRIME)
def test_sb_tcn_clip_lengths(built_lib, Tp, la):
    cfg = _sb_cfg(la=la, attn="TSSE" if Tp >= TSSE_MIN else "SE")
    _sb_case(f"sb T'={Tp} la={la}", cfg, 1, Tp, seed=60 + Tp)


def test_sb_tcn_ragged(built_lib):
    cfg = _sb_cfg(attn="SE")
    T = 40
    m, params = _sb_model(cfg, 70)
    frames = RAGGED + [T]
    B = len(frames)
    mag, real, imag = _spectra(B, 33, T, 71)
    for b, n in enumerate(frames):
        for x in (mag, real, imag):
            x[b, :, :, n:] = np.nan
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag), frames=frames)
    for b, n in enumerate(frames):
        assert (out[b, :, :, n:] == 0).all(), f"clip {b}: mask past frames[b] is not zero"
    _sb_check("sb ragged", m, params, cfg, B, T + 2, out, frames=frames)


def test_sb_tcn_more_than_65535_groups(built_lib):
    F, B, Tp = SB_GROUPS
    _sb_case(f"sb B*F={B * F}", _sb_cfg(F=F, Ns=1, la=0, attn="SE"), B, Tp, seed=80)


def test_sb_tcn_bin_chunks(built_lib, monkeypatch):
    """FSN_SB_CHUNK = 7 and 16 over 33 bins (the last chunk narrower): each chunked mask against the truth from the unchunked sb_in,
    and bit-identical to the unchunked run."""
    cfg = _sb_cfg()
    m, params, ins, whole = _sb_case("sb chunks unchunked", cfg, 2, 42, seed=90)
    sb_in = m.get_stage("sb_in", (2, 33, S.isb(cfg), 42), DEV)
    for chunk in ("7", "16"):
        monkeypatch.setenv("FSN_SB_CHUNK", chunk)
        mc, _ = _sb_model(cfg, 90)
        monkeypatch.delenv("FSN_SB_CHUNK")
        with torch.no_grad():
            got = mc(*(_t(x) for x in ins))
        assert mc.last_plan_bins()[2] == int(chunk), mc.last_plan_bins()
        _sb_check(f"sb chunks {chunk}", mc, params, cfg, 2, 42, got, sb_in=sb_in)
        assert torch.equal(got, whole), f"FSN_SB_CHUNK={chunk}: not bit-identical to the unchunked run"


@pytest.mark.parametrize("act", ACTS)
def test_sb_tcn_activations(built_lib, act):
    _sb_case(f"sb act {act}", _sb_cfg(act=act), 2, 40, seed=100, record=act in (None, "Tanh"))


def test_sb_tcn_enhance_entry_point(built_lib):
    """enhance_spectrum: decompress_cIRM(the kernel's own mask) x noisy to fp32 tolerance; the mask itself against fp64."""
    cfg = _sb_cfg()
    m, params, (mag, real, imag), mask = _sb_case("sb enhance mask", cfg, 2, 42, seed=110)
    with torch.no_grad():
        enh = m.enhance_spectrum(_t(mag), _t(real), _t(imag)).cpu().to(torch.complex128)
    d = torch.from_numpy(O.decompress_cIRM(mask.cpu().double().numpy()))
    noisy = torch.complex(torch.from_numpy(real[:, 0]).double(), torch.from_numpy(imag[:, 0]).double())
    own = torch.complex(d[:, 0], d[:, 1]) * noisy
    assert torch.allclose(enh, own, rtol=2e-5, atol=2e-5 * float(own.abs().max())), "enhanced spectrum != decompress_cIRM(mask) x noisy"


# ---- fullsubnet.Model full band -------------------------------------------------------------------------------------------------------
def _fsn_case(label, B, H, L, kind, fast, F, Tp=40, la=2, frames=None, seed=0, record=True, expect_ws=None):
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=F, fb_model_hidden_size=H, sequence_model=kind, look_ahead=la, sb_num_neighbors=1 if F < 16 else 15,
               sb_model_hidden_size=64)
    params = O.make_params_fsn(cfg, seed=seed, num_layers=L)
    m = _load(Model(**cfg, num_layers=L, fast_math=fast), params)
    T = Tp - la
    mag = _spectra(B, F, T, seed + 1)[0]
    if frames is not None:
        mag = mag.copy()
        for b, n in enumerate(frames):
            mag[b, :, :, n:] = np.nan
    with torch.no_grad():
        m(_t(mag), frames=frames)
    ws = _lib.load_library().fsn_model_last_fb_ws(m._handle)
    want_ws = ws_eligible(L, H, F, B, _num_sms()) if expect_ws is None else expect_ws
    assert ws == int(want_ws), (label, ws, want_ws)
    fb_in = m.get_stage("fb_in", (1, B, F, Tp), DEV)[0]
    fb_out = m.get_stage("fb_out", (1, B, F, Tp), DEV)[0]
    torch.cuda.synchronize()
    clips = sorted({c for c in (0, 1, 31, 63, 64, B - 1) if c < B}) if B > 16 else list(range(B))
    sel = torch.as_tensor(clips, device=DEV)
    dev = DEV if len(clips) * Tp * H > 2e5 else "cpu"
    x = fb_in[sel].to(dev)
    act = cfg["fb_output_activate_function"]
    want = R.truth(params, kind, x, 0, act, device=dev, prefix="fb_model", head="fb")
    emu = R.emulate(params, kind, x, 0, act, device=dev, prefix="fb_model", head="fb")
    valid, _ = _valid(None if frames is None else [frames[c] for c in clips], la, len(clips), Tp)
    r = R.compare(fb_out[sel], want, emu, R.FAST_FACTOR if fast else 1.0, valid.expand(len(clips), F, Tp))
    path = "ws" if ws else "mma"
    _line(label, r, f" {kind} H={H} L={L} {'fast' if fast else 'acc '} F={F} B={B} T'={Tp} {path}:")
    if record:
        _record(f"full-band {path} {'fast' if fast else 'accurate'}", H, label, r)
    assert torch.isfinite(fb_out).all(), label
    assert r["ok"], (label, r)


@pytest.mark.parametrize("B,H,L,kind,fast,F", WS)
def test_fsn_weight_stationary(built_lib, B, H, L, kind, fast, F):
    assert ws_eligible(L, H, F, B, _num_sms())
    _fsn_case("ws", B, H, L, kind, fast, F, seed=H + L)


def test_fsn_weight_stationary_limits(built_lib):
    """The largest F whose ws_smem fits at (L, H) = WS_LIMIT_LH runs weight-stationary, the next falls back; H / 4 = num_sms is the
    largest grid (132 CTAs at H = 528 on an H100 SXM), one more unit of 4 falls back."""
    L, H = WS_LIMIT_LH
    fit, over = ws_limit_widths(L, H)
    _fsn_case(f"ws smem limit F={fit}", 2, H, L, "LSTM", True, fit, seed=3, expect_ws=True)
    _fsn_case(f"ws smem limit F={over}", 2, H, L, "LSTM", True, over, seed=3, expect_ws=False)
    n = _num_sms()
    _fsn_case(f"ws grid H={4 * n}", 2, 4 * n, 1, "GRU", True, 33, seed=4, expect_ws=True)
    _fsn_case(f"ws grid H={4 * n + 16}", 2, 4 * n + 16, 1, "GRU", True, 33, seed=4, expect_ws=False)


@pytest.mark.parametrize("B,H,L,kind,fast,F", MMA)
def test_fsn_generic_kernel(built_lib, B, H, L, kind, fast, F):
    assert not ws_eligible(L, H, F, B, _num_sms())
    _fsn_case("mma rows", B, H, L, kind, fast, F, seed=B)


def test_fsn_no_ws_knob(built_lib, monkeypatch):
    """FSN_NO_WS=1 (read when the handle is created) keeps an eligible shape on lstm_mma_kernel."""
    monkeypatch.setenv("FSN_NO_WS", "1")
    _fsn_case("FSN_NO_WS=1", 2, 256, 2, "LSTM", True, 257, seed=7, expect_ws=False)


@pytest.mark.parametrize("Tp,la", FSN_TPRIME)
def test_fsn_clip_lengths(built_lib, Tp, la):
    _fsn_case(f"fsn T'={Tp}", 2, 256, 2, "LSTM", True, 257, Tp=Tp, la=la, seed=Tp)


def test_fsn_ragged(built_lib):
    T = 40
    frames = RAGGED + [T]
    _fsn_case("fsn ragged", len(frames), 256, 2, "GRU", True, 257, Tp=T + 2, frames=frames, seed=9)


def test_zz_worst_per_path(built_lib):
    """The tables DESIGN.md §2 quotes: worst max err / RMS per stage, and per stage and width (F, Isb or H)."""
    if not WORST:
        pytest.skip("no case of this file ran before")
    print("\nworst max err / RMS (ratio to the emulation's error, case):")
    for key in sorted(WORST, key=str):
        e, ratio, label = WORST[key]
        print(f"  {' / '.join(map(str, key)):40} {e:.2e}  x{ratio:.2f}  {label}")
