"""The sub-band LSTM / GRU stage alone (fsn_model_sb_forward) against fp64, element by element.

The stage runs through the forward's own layer and window loop (lstm_tc5r_kernel, the gemm_f16 input projection of the deeper
layers, lstm_mma_kernel for lstm_impl="mma") on an fp16-representable input, so the fp64 references (tests/sb_rnn_ref.py) see exactly
the kernel's input.  Per case: max |kernel - fp64| / RMS over the compared elements must stay within
factor * (3 max |fp16 emulation - fp64| + 1e-6 RMS), factor 1 for accurate gate math and sb_rnn_ref.FAST_FACTOR for fast math.
Each case prints one line: max err / RMS, the emulation's, the bound, their ratio and the rel-L2; the last test prints the worst per
path and hidden size.

Fast-math factor (sb_rnn_ref.FAST_FACTOR = 1.5), measured once on one H100 80GB HBM3 SXM at its 700 W power limit: over every
fast-math case of this file the kernel's max err was at most 1.15x the fp16 emulation's (the mma GRU at H = 512, and the chaotic x8-weight
LSTM); layer-wise cases 0.31-0.91x, below the emulation because the fused output Linear reads h in fp32 where the emulation reads fp16.
Accurate math: at most 1.00x (|x| up to 1e4).

Coverage (the CPU test test_sb_recurrence_cpu.py checks these lists reach every ring plan and every mma row count):
  * every H in 64..512 with L = 1 (first and last layer in one launch) and L = 3 (first, middle, last), LSTM and GRU, fast math;
  * accurate math at H = 64, 256, 512 (L = 3, both cells); L = 4 at H = 512;
  * B*F = 4 (the smallest geometry, num_freqs >= 4: one nearly empty CTA and an empty cluster peer), 63, 64, 65, 128, 129 (a lone row
    in the third tile, padded tile pair), 257, and a grid of more than two waves on 132 SMs (sampled rows);
  * T' = 1, 2, 3, 5, 33, 190 with look_ahead 0 and 2; Isb = 6, 34, 64;
  * windows of 32 and 64 frames against fp64 (and bit-equal to the unwindowed run) at H = 512 L = 3 LSTM, H = 384 GRU, H = 64 L = 4;
  * ragged frames (a 1-frame clip next to full-length ones, NaN past each clip's end), the fused enhance epilogue with masks
    beyond the +-9.9 clamp, every output activation;
  * an all-zero input, |x| up to 1e4, x3 / x8 LSTM weights (saturated gates, the accurate path's +-43 clamp), T' = 2000;
  * lstm_impl = "mma" at H = 32, 48, 64, 96, 384, 512 with L up to 4 (R = 64, 32 and 16 rows per CTA); fullsubnet.Model once.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import sb_rnn_ref as R
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (H, L, cell) of the layer-wise kernel under fast math: every template instantiation and every layer role
INSTANCES = [(H, L, kind) for H in range(64, 513, 64) for L in (1, 3) for kind in ("LSTM", "GRU")]
ACCURATE = [(H, 3, kind) for H in (64, 256, 512) for kind in ("LSTM", "GRU")]
LAYERS4 = [(512, 4, "LSTM", True), (512, 4, "GRU", False)]
GEOMETRY = [(4, 1), (63, 1), (64, 1), (65, 1), (64, 2), (43, 3), (257, 1)]          # (num_freqs, B): B*F = 4 .. 257
TPRIME = [(1, 0), (2, 0), (3, 2), (5, 2), (33, 0), (190, 2)]                          # (T', look_ahead)
ISB = [(1, 0), (15, 0), (30, 0)]                                                      # (sb_num_neighbors, fb_num_neighbors): Isb 6, 34, 64
WINDOWS = [(512, 3, "LSTM"), (384, 2, "GRU"), (64, 4, "LSTM")]
MMA = [(32, 2, "LSTM", True), (48, 3, "GRU", False), (64, 4, "LSTM", True), (96, 2, "GRU", True), (384, 3, "LSTM", False),
       (512, 1, "GRU", True), (512, 2, "LSTM", True), (512, 4, "LSTM", False)]

WORST = {}


def _cfg(F=64, H=384, kind="LSTM", la=2, Ns=15, Nf=0, act=False, attn="TSSE"):
    c = O.default_plus_config()
    c.update(num_freqs=F, sb_model_hidden_size=H, sequence_model=kind, look_ahead=la, sb_num_neighbors=Ns, fb_num_neighbors=Nf,
             sb_output_activate_function=act, channel_attention_model=attn)
    return c


def _model(cfg, L, fast, impl="auto", seed=0, scale=1.0, fc_bias=None, fsn=False, fc_scale=1.0):
    from fsnplus_b200.model import FullSubNet_Plus, Model
    if fsn:
        params = O.make_params_fsn(cfg, seed=seed, lstm_scale=scale, num_layers=L)
        m = Model(**cfg, num_layers=L, lstm_impl=impl, fast_math=fast)
    else:
        params = O.make_params_plus(cfg, seed=seed, lstm_scale=scale, num_layers=L)
        m = FullSubNet_Plus(**cfg, num_layers=L, lstm_impl=impl, fast_math=fast)
    if fc_bias is not None:
        params["sb_model.fc_output_layer.bias"] = np.asarray(fc_bias, np.float32)
    params["sb_model.fc_output_layer.weight"] = params["sb_model.fc_output_layer.weight"] * np.float32(fc_scale)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    return m, params


def _isb(cfg, fsn=False):
    return 2 * cfg["sb_num_neighbors"] + 1 + (1 if fsn else 3) * (2 * cfg["fb_num_neighbors"] + 1)


def _input(B, F, I, Tp, seed=0, scale=1.0):
    """[B, F, I, Tp] fp32 holding fp16 values (the packer's rounding is then the identity)"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, F, I, Tp, device=DEV, generator=g) * scale
    return x.clamp(-1e4, 1e4).half().float()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p()


def _sb(m, x, T, Tw=0, frames=None, noisy=None):
    """fsn_model_sb_forward: the mask [B, 2, F, T], or with noisy = (real, imag) the enhanced spectrum [B, F, T] complex64."""
    from fsnplus_b200 import _lib
    B, F = x.shape[0], x.shape[1]
    fr = (C.c_int32 * B)(*frames) if frames is not None else None
    out = enh = None
    if noisy is None:
        out = torch.full((B, 2, F, T), float("nan"), device=DEV)
    else:
        enh = torch.full((B, F, T), complex(float("nan"), 0.0), dtype=torch.complex64, device=DEV)
    with torch.cuda.device(DEV):
        stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
        _lib.check(_lib.load_library().fsn_model_sb_forward(m._handle, _ptr(x), B, T, Tw, fr, _ptr(out), _ptr(noisy[0] if noisy else None),
                                                            _ptr(noisy[1] if noisy else None), _ptr(enh), stream))
    torch.cuda.synchronize()
    return out if noisy is None else enh


def _plan(lib, impl, H, L):
    if impl == "mma":
        return f"mma R={lib.fsn_lstm_mma_rows(L, H, 64, 2)}"
    roles = [(l == 0, l == L - 1) for l in range(L)]
    return "stages " + "/".join(str(lib.fsn_tc5r_ring_stages(H, int(f), int(la))) for f, la in roles)


def _check(label, m, params, cfg, L, fast, x, got, impl="auto", frames=None, fsn=False, record=True):
    """Compare the kernel's mask got [B, 2, F, T] on sampled rows (and, ragged, valid frames) with fp64; returns (truth, rows)."""
    from fsnplus_b200 import _lib
    B, F, I, Tp = x.shape
    la, H, kind, act = cfg["look_ahead"], cfg["sb_model_hidden_size"], cfg["sequence_model"], cfg["sb_output_activate_function"]
    T = Tp - la
    rows = R.sample_rows(B * F)
    dev = DEV if len(rows) * Tp * H > 2e6 else "cpu"
    xs = x.reshape(B * F, I, Tp)[torch.as_tensor(rows, device=DEV)].to(dev)
    want = R.truth(params, kind, xs, la, act, device=dev)
    emu = R.emulate(params, kind, xs, la, act, device=dev)
    g = got.permute(0, 2, 1, 3).reshape(B * F, 2, T)[torch.as_tensor(rows, device=DEV)]
    mask = None
    if frames is not None:
        fr = torch.as_tensor([frames[r // F] for r in rows])
        mask = (torch.arange(T)[None, None, :] < fr[:, None, None]).expand(len(rows), 2, T)
    factor = R.FAST_FACTOR if fast else 1.0
    r = R.compare(g, want, emu, factor, mask)
    lib = _lib.load_library()
    path = ("mma" if impl == "mma" else "layer-wise") + (" fast" if fast else " accurate")
    print(f"\n[{label}] {kind} H={H} L={L} {'fast' if fast else 'acc '} {_plan(lib, impl, H, L)} rows {len(rows)}/{B * F} T'={Tp}: "
          f"max err/RMS {r['err']:.2e} emu {r['emu']:.2e} bound {r['bound']:.2e} ratio {r['ratio']:.2f} rel-L2 {r['rel']:.2e}")
    if record:
        for key in (path, (path, H)):
            if r["err"] >= WORST.get(key, (-1.0,))[0]:
                WORST[key] = (r["err"], r["ratio"], label)
    assert r["finite"], label
    assert r["ok"], (label, r)
    return want, rows


def _case(label, cfg, L, fast, B, Tp, impl="auto", seed=0, scale=1.0, x_scale=1.0, zero=False, fsn=False, Tw=0, fc_bias=None, record=True):
    m, params = _model(cfg, L, fast, impl=impl, seed=seed, scale=scale, fsn=fsn, fc_bias=fc_bias)
    x = _input(B, cfg["num_freqs"], _isb(cfg, fsn), Tp, seed=seed + 1, scale=x_scale)
    if zero:
        x.zero_()
    got = _sb(m, x, Tp - cfg["look_ahead"], Tw=Tw)
    _check(label, m, params, cfg, L, fast, x, got, impl=impl, fsn=fsn, record=record)
    return m, params, x, got


@pytest.mark.parametrize("H,L,kind", INSTANCES)
def test_every_instantiation_fast(built_lib, H, L, kind):
    _case("instance", _cfg(F=64, H=H, kind=kind), L, True, B=4, Tp=40, seed=H + L)


@pytest.mark.parametrize("H,L,kind", ACCURATE + [(H, L, k) for H, L, k, f in LAYERS4 if not f])
def test_accurate_math(built_lib, H, L, kind):
    _case("accurate", _cfg(F=64, H=H, kind=kind), L, False, B=4, Tp=40, seed=H + 7)


@pytest.mark.parametrize("H,L,kind", [(H, L, k) for H, L, k, f in LAYERS4 if f])
def test_four_layers_fast(built_lib, H, L, kind):
    _case("4 layers", _cfg(F=64, H=H, kind=kind), L, True, B=4, Tp=40, seed=11)


@pytest.mark.parametrize("F,B", GEOMETRY)
def test_row_geometry(built_lib, F, B):
    _case(f"B*F={B * F}", _cfg(F=F, H=384, Ns=1 if F < 16 else 15), 2, True, B=B, Tp=40, seed=F + B)


def test_more_than_two_waves(built_lib):
    """70 x 257 rows = 141 tiles -> 284 CTAs, more than two waves of one CTA per SM on 132 SMs; sampled rows."""
    _case("waves", _cfg(F=257, H=384), 2, True, B=70, Tp=33, seed=3)


@pytest.mark.parametrize("Tp,la", TPRIME)
def test_short_and_long_sequences(built_lib, Tp, la):
    _case(f"T'={Tp} la={la}", _cfg(F=64, H=384, la=la), 2, True, B=2, Tp=Tp, seed=Tp)


@pytest.mark.parametrize("Ns,Nf", ISB)
def test_input_widths(built_lib, Ns, Nf):
    cfg = _cfg(F=64, H=256, Ns=Ns, Nf=Nf)
    _case(f"Isb={_isb(cfg)}", cfg, 2, True, B=2, Tp=40, seed=Ns)


@pytest.mark.parametrize("H,L,kind", WINDOWS)
def test_windows_against_fp64(built_lib, H, L, kind):
    """T' = 150 is a multiple of neither window: each windowed run is compared with fp64, then with the unwindowed run (bit-equal)."""
    cfg = _cfg(F=64, H=H, kind=kind)
    m, params, x, whole = _case("windows Tw=0", cfg, L, True, B=2, Tp=150, seed=H)
    for Tw in (32, 64):
        got = _sb(m, x, 150 - cfg["look_ahead"], Tw=Tw)
        _check(f"windows Tw={Tw}", m, params, cfg, L, True, x, got)
        assert torch.equal(got, whole), f"window {Tw}: not bit-identical to the unwindowed run"


@pytest.mark.parametrize("impl", ["auto", "mma"])
def test_ragged_frames_and_nan_past_the_end(built_lib, impl):
    """SE attention: the TSSE convolutions would need frames + look_ahead >= 10 (the forward's rule, which the hook keeps)."""
    cfg = _cfg(F=64, H=128 if impl == "auto" else 96, attn="SE")
    m, params = _model(cfg, 2, True, impl=impl, seed=5)
    B, Tp, la = 4, 70, cfg["look_ahead"]
    T = Tp - la
    frames = [1, T, 37, T - 5]
    x = _input(B, 64, _isb(cfg), Tp, seed=6)
    clean = _sb(m, x, T, frames=frames)
    for b, n in enumerate(frames):                                      # NaN poison past each clip's end (frames[b] + look_ahead)
        x[b, :, :, n + la:] = float("nan")
    got = _sb(m, x, T, frames=frames)
    assert torch.equal(got, clean), "inputs past a clip's end changed the output"
    for b, n in enumerate(frames):
        assert (got[b, :, :, n:] == 0).all() and not torch.signbit(got[b, :, :, n:]).any(), f"clip {b}: output past frames[b] is not +0"
    x = torch.nan_to_num(x, nan=0.0)                                    # the truth of clip b only reads its first frames[b] + la frames
    _check(f"ragged {impl}", m, params, cfg, 2, True, x, got, impl=impl, frames=frames)


@pytest.mark.parametrize("impl", ["auto", "mma"])
def test_enhance_epilogue_beyond_the_clamp(built_lib, impl):
    """fc_output_layer weight x40 and bias (+9.5, -9.5): masks spread across +-9.9.  The enhanced spectrum must equal
    decompress_cIRM(mask) x noisy to fp32 tolerance: against the kernel's own mask everywhere, and against the fp64 mask wherever
    that lies beyond the clamp."""
    cfg = _cfg(F=64, H=128 if impl == "auto" else 96)
    m, params = _model(cfg, 2, True, impl=impl, seed=8, fc_bias=(9.5, -9.5), fc_scale=40.0)
    B, Tp = 2, 60
    T = Tp - cfg["look_ahead"]
    x = _input(B, 64, _isb(cfg), Tp, seed=9)
    mask = _sb(m, x, T)
    want, rows = _check(f"enhance mask {impl}", m, params, cfg, 2, True, x, mask, impl=impl)
    g = torch.Generator(device=DEV).manual_seed(10)
    real, imag = (torch.randn(B, 64, T, device=DEV, generator=g) for _ in range(2))
    enh = _sb(m, x, T, noisy=(real, imag)).cpu()
    noisy = torch.complex(real, imag).cpu().to(torch.complex128)

    def enhance(mk):                                                    # mk [B, 2, F, T] -> decompress_cIRM(mk) x noisy
        d = torch.from_numpy(O.decompress_cIRM(mk.cpu().double().numpy()))
        return torch.complex(d[:, 0], d[:, 1]) * noisy

    e64 = enh.to(torch.complex128)
    own = enhance(mask)
    assert torch.allclose(e64, own, rtol=2e-5, atol=2e-5 * float(own.abs().max())), "enhanced spectrum != decompress_cIRM(mask) x noisy"
    B_, F = B, 64
    wmask = torch.full((B_ * F, 2, T), float("nan"), dtype=torch.float64)
    wmask[torch.as_tensor(rows)] = want.cpu()
    wmask = wmask.reshape(B_, F, 2, T).permute(0, 2, 1, 3)
    sel = (wmask.abs() >= 9.9 + 1e-2).all(dim=1)                        # both mask components clamped in fp64 (and so in the kernel)
    assert (wmask[:, 0] >= 9.9 + 1e-2).any() and (wmask[:, 1] <= -9.9 - 1e-2).any(), "the clamp was not exercised"
    assert sel.sum() > 0
    ref = enhance(torch.nan_to_num(wmask))
    assert torch.allclose(e64[sel], ref[sel], rtol=2e-5, atol=2e-5 * float(ref.abs().max()))
    print(f"[enhance {impl}] {int(sel.sum())} elements with both mask components beyond the clamp")


@pytest.mark.parametrize("act", [None, "ReLU", "Tanh", "ReLU6"])
def test_output_activations(built_lib, act):
    """fc_output_layer.bias = 0 (ReLU6: 6 on the first output): both sides of every activation's kinks are reached.  ReLU zeroes most
    outputs, which makes the RMS small: the clamping activations stay out of the worst-case table."""
    _case(f"act {act}", _cfg(F=64, H=128, act=act), 2, True, B=2, Tp=40, seed=12, fc_bias=(6.0 if act == "ReLU6" else 0.0, 0.0),
          record=act in (None, "Tanh"))


def test_all_zero_input(built_lib):
    _case("zero input", _cfg(F=64, H=384), 2, True, B=2, Tp=40, seed=13, zero=True)


@pytest.mark.parametrize("fast", [True, False])
def test_large_inputs(built_lib, fast):
    """x ~ N(0, 2500^2) clipped to +-1e4: the first layer's gates saturate.  The fp16 rounding of W_ih alone then moves a gate
    argument by O(1), so the error is the emulation's (7e-2 of the RMS); left out of the worst-case table."""
    _case("|x| <= 1e4", _cfg(F=64, H=256), 2, fast, B=2, Tp=40, seed=14, x_scale=2500.0, record=False)


@pytest.mark.parametrize("scale,fast", [(3.0, True), (8.0, True), (8.0, False)])
def test_saturated_gates(built_lib, scale, fast):
    """x8 weights make the recurrence chaotic: the fp16 rounding of the weights alone moves outputs by O(RMS) after 60 steps, so that
    case checks finiteness and the +-43 clamp against the same bound rather than accuracy; left out of the worst-case table."""
    _case(f"LSTM weights x{scale:g}", _cfg(F=64, H=384), 2, fast, B=2, Tp=60, seed=15, scale=scale, record=scale < 8)


def test_long_recurrence(built_lib):
    """T' = 2000 at H = 384: error growth along the recurrence."""
    _case("T'=2000", _cfg(F=64, H=384), 2, True, B=2, Tp=2000, seed=16)


@pytest.mark.parametrize("H,L,kind,fast", MMA)
def test_generic_kernel(built_lib, H, L, kind, fast):
    _case("mma", _cfg(F=64, H=H, kind=kind), L, fast, B=2, Tp=40, impl="mma", seed=H + L)


def test_fullsubnet_model(built_lib):
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=64)
    _case("fullsubnet.Model", cfg, 2, True, B=2, Tp=40, seed=17, fsn=True)


def test_hook_argument_checks(built_lib):
    """FSN_EINVAL for a sub-band TCN model, a bad window, a window on the mma path and bad frame counts; FSN_ESTATE before finalize."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus
    lib = _lib.load_library()
    cfg = _cfg(F=64, H=128)
    m, _ = _model(cfg, 2, True)
    x = _input(1, 64, _isb(cfg), 10)
    out = torch.empty(1, 2, 64, 8, device=DEV)
    s = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)

    def call(h, Tw=0, frames=None, B=1, xx=x, o=out):
        fr = (C.c_int32 * len(frames))(*frames) if frames is not None else None
        return lib.fsn_model_sb_forward(h, _ptr(xx), B, 8, Tw, fr, _ptr(o), None, None, None, s), lib.fsn_last_error()

    assert call(m._handle)[0] == 0
    for kw, needle in (({"Tw": 48}, b"multiple of 32"), ({"Tw": -32}, b"multiple of 32"), ({"frames": [0]}, b"outside 1..T"),
                       ({"frames": [9]}, b"outside 1..T"), ({"B": 0}, b"bad batch"), ({"xx": None}, b"null"), ({"o": None}, b"null")):
        rc, msg = call(m._handle, **kw)
        assert rc == -1 and needle in msg, (kw, rc, msg)
    mm, _ = _model(cfg, 2, True, impl="mma")
    rc, msg = call(mm._handle, Tw=32)
    assert rc == -1 and b"layer-wise" in msg
    assert call(mm._handle)[0] == 0
    h = C.c_void_p()
    _lib.check(lib.fsn_model_create(C.byref(m._cfg), C.byref(h)))
    try:
        rc, msg = call(h)
        assert rc == -3 and b"finalize" in msg
    finally:
        lib.fsn_model_destroy(h)
    t = FullSubNet_Plus(**dict(_cfg(F=64), sequence_model="TCN", weight_init=True)).to(DEV).eval()
    with torch.cuda.device(DEV):
        t._ensure_handle(torch.device(DEV))
    rc, msg = call(t._handle)
    assert rc == -1 and b"TCN" in msg
    torch.cuda.synchronize()


def test_zz_worst_per_path(built_lib):
    """The table DESIGN.md §2 quotes: worst max err / RMS per path, and per path and hidden size."""
    if not WORST:
        pytest.skip("no case of this file ran before")
    print("\nworst max err / RMS (ratio to the fp16 emulation's error, case):")
    for key in sorted(WORST, key=str):
        e, ratio, label = WORST[key]
        print(f"  {key!s:32} {e:.2e}  x{ratio:.2f}  {label}")
