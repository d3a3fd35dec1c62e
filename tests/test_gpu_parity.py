"""GPU parity tests: the CUDA path, called through the C ABI (via the Python mirror of the reference API),
against the numpy oracle on the same seeded inputs and against the committed golden vectors generated from the
unmodified reference.

Tolerances (relative L2 over the whole tensor, truth = float64 reference/oracle):
  * final cIRM mask ................ 1e-3  (the bar BASELINE.json's north_star states)
  * full-band stages (TF32 convs) .. 2e-3 on fb_out, 1e-5 on fb_in (fp32 CUDA-core math)
"""
import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASK_TOL = 1e-3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def build_plus(cfg, params, **kw):
    from fsnplus_b200.model import FullSubNet_Plus
    m = FullSubNet_Plus(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    return m.to(DEV).eval()


def build_fsn(cfg, params, **kw):
    from fsnplus_b200.model import Model
    m = Model(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    return m.to(DEV).eval()


def small_cfg(H):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=H)
    return c


def small_inputs(B, F, T, seed):
    rng = np.random.default_rng(seed)
    real = rng.standard_normal((B, 1, F, T)) * 0.05 + 0.004
    imag = rng.standard_normal((B, 1, F, T)) * 0.05 - 0.003
    mag = np.sqrt(real ** 2 + imag ** 2)
    return mag.astype(np.float32), real.astype(np.float32), imag.astype(np.float32)


@pytest.mark.parametrize("impl,H", [("mma", 32), ("mma", 64), ("tcgen05", 64), ("tcgen05", 128)])
def test_plus_small_vs_oracle(built_lib, impl, H):
    cfg = small_cfg(H)
    params = O.make_params_plus(cfg, seed=3)
    mag, real, imag = small_inputs(3, 33, 20, 7)
    st = {}
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag, stages=st)
    m = build_plus(cfg, params, lstm_impl=impl)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    assert out.shape == (3, 2, 33, 20) and out.dtype == torch.float32
    assert m.last_lstm_impl() == impl
    fb_in = m.get_stage("fb_in", (3, 3, 33, 22), DEV).cpu().numpy()
    fb_out = m.get_stage("fb_out", (3, 3, 33, 22), DEV).cpu().numpy()
    assert O.rel_l2(fb_in, st["fb_in"]) < 1e-5
    assert O.rel_l2(fb_out, st["fb_out"]) < 2e-3
    assert O.rel_l2(out.cpu().numpy(), ref) < MASK_TOL


def test_plus_small_golden_from_reference(built_lib, golden):
    """Committed reference output (H=32 config of make_golden.py)."""
    g = golden("plus_small")
    cfg = small_cfg(32)
    m = build_plus(cfg, O.make_params_plus(cfg, seed=3))
    with torch.no_grad():
        out = m(_t(g["mag"]), _t(g["real"]), _t(g["imag"]))
    assert O.rel_l2(out.cpu().numpy(), g["out"]) < MASK_TOL


@pytest.mark.parametrize("attn", ["SE", "ECA", "CBAM"])
def test_plus_small_other_attentions_golden(built_lib, golden, attn):
    """channel_attention_model = SE / ECA / CBAM (fullsubnet_plus.py:52-70) against committed reference outputs."""
    g, gi = golden(f"plus_small_{attn}"), golden("plus_small")
    cfg = dict(small_cfg(32), channel_attention_model=attn)
    m = build_plus(cfg, O.make_params_plus(cfg, seed=5))
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    fb_in = m.get_stage("fb_in", (3, 3, 33, 22), DEV).cpu().numpy()
    e_in, err = O.rel_l2(fb_in, g["fb_in"]), O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[{attn}] fb_in {e_in:.2e} cIRM {err:.3e}")
    assert e_in < 1e-5
    assert err < MASK_TOL


@pytest.mark.parametrize("attn", ["SE", "ECA", "CBAM"])
def test_plus_default_size_other_attentions_vs_oracle(built_lib, golden, attn):
    """Default geometry (F=257, H=384, tensor-core LSTM path), one clip, oracle as truth; for CBAM the mag branch has all-positive
    rows and the real/imag branches a negative normaliser, which exercises the min/max selection of the squeeze."""
    gi = golden("plus_default")
    cfg = dict(O.default_plus_config(), channel_attention_model=attn)
    params = O.make_params_plus(cfg, seed=9)
    ref = O.fullsubnet_plus_forward(params, cfg, gi["mag"], gi["real"], gi["imag"])
    m = build_plus(cfg, params)
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[{attn} default size] cIRM {err:.3e}")
    assert err < MASK_TOL


@pytest.mark.parametrize("sub", [2, 3])
def test_plus_small_subband_num_golden(built_lib, golden, sub):
    """subband_num > 1 with ECA (the combination the reference forward supports, fullsubnet_plus.py:146-153)."""
    g, gi = golden(f"plus_small_ECA_sub{sub}"), golden("plus_small")
    cfg = dict(small_cfg(32), channel_attention_model="ECA", subband_num=sub)
    m = build_plus(cfg, O.make_params_plus(cfg, seed=5))
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    fb_in = m.get_stage("fb_in", (3, 3, 33, 22), DEV).cpu().numpy()
    e_in, err = O.rel_l2(fb_in, g["fb_in"]), O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[ECA subband_num={sub}] fb_in {e_in:.2e} cIRM {err:.3e}")
    assert e_in < 1e-5 and err < MASK_TOL


def test_gru_small_goldens_from_reference(built_lib, golden):
    """sequence_model = "GRU" (sequence_model.py:39-46), committed reference outputs: FullSubNet+ (H = 32 -> mma kernel) and
    fullsubnet.Model (full-band GRU on the weight-stationary kernel, sub-band GRU on the mma kernel)."""
    gi = golden("plus_small")
    cfg = dict(small_cfg(32), sequence_model="GRU")
    m = build_plus(cfg, O.make_params_plus(cfg, seed=8, lstm_scale=2.0))
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    err = O.rel_l2(out.cpu().numpy(), golden("plus_small_GRU")["out"])
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48, sequence_model="GRU")
    m = build_fsn(cfg, O.make_params_fsn(cfg, seed=8, lstm_scale=2.0))
    with torch.no_grad():
        out = m(_t(gi["mag"]))
    g = golden("fsn_small_GRU")
    e_fb = O.rel_l2(m.get_stage("fb_out", (3, 33, 22), DEV).cpu().numpy(), g["fb_out"])
    err2 = O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[GRU small] FullSubNet+ cIRM {err:.3e}; fullsubnet.Model fb_out {e_fb:.2e} cIRM {err2:.3e}")
    assert err < MASK_TOL and err2 < MASK_TOL and e_fb < 2e-3


@pytest.mark.parametrize("impl,H", [("mma", 64), ("tcgen05", 64), ("tcgen05", 128)])
@pytest.mark.parametrize("fast", [True, False])
def test_gru_plus_small_vs_oracle(built_lib, impl, H, fast):
    cfg = dict(small_cfg(H), sequence_model="GRU")
    params = O.make_params_plus(cfg, seed=13, lstm_scale=2.0)
    mag, real, imag = small_inputs(5, 33, 27, 3)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag)
    m = build_plus(cfg, params, lstm_impl=impl, fast_math=fast)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    assert m.last_lstm_impl() == impl
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[GRU {impl} H={H} fast={fast}] cIRM {err:.3e}")
    assert err < MASK_TOL


def test_gru_default_size_vs_oracle(built_lib, golden):
    """Default geometry with a GRU sub-band model (tensor-core LSTM path, H = 384) and the GRU fullsubnet.Model (H = 512 full
    band on the weight-stationary kernel); one 3 s clip, oracle fp64 as truth; a parameter update must re-expand the gates."""
    gi = golden("plus_default")
    cfg = dict(O.default_plus_config(), sequence_model="GRU")
    params = O.make_params_plus(cfg, seed=17, lstm_scale=2.0)
    ref = O.fullsubnet_plus_forward(params, cfg, gi["mag"], gi["real"], gi["imag"])
    m = build_plus(cfg, params)
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
        assert m.last_lstm_impl() == "tcgen05"
        err = O.rel_l2(out.cpu().numpy(), ref)
        m.sb_model.sequence_model.bias_hh_l0.mul_(1.0)              # bumps the version -> parameters are pushed again
        out2 = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    assert torch.equal(out, out2)
    fcfg = dict(O.default_fsn_config(), sequence_model="GRU")
    fparams = O.make_params_fsn(fcfg, seed=18, lstm_scale=2.0)
    fref = O.fullsubnet_forward(fparams, fcfg, gi["mag"])
    fm = build_fsn(fcfg, fparams)
    with torch.no_grad():
        fout = fm(_t(gi["mag"]))
    ferr = O.rel_l2(fout.cpu().numpy(), fref)
    print(f"\n[GRU default size] FullSubNet+ cIRM {err:.3e}; fullsubnet.Model cIRM {ferr:.3e}")
    assert err < MASK_TOL and ferr < MASK_TOL


@pytest.mark.parametrize("impl", ["tcgen05", "mma"])
@pytest.mark.parametrize("stress", [False, True])
def test_plus_default_config_golden(built_lib, golden, impl, stress):
    """BASELINE config #1: default config/inference.toml, one 3 s clip, reference fp64 output as truth."""
    gi = golden("plus_default")
    g = golden("plus_default_stress") if stress else gi
    cfg = O.default_plus_config()
    m = build_plus(cfg, O.make_params_plus(cfg, seed=0, lstm_scale=3.0 if stress else 1.0), lstm_impl=impl)
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    assert out.shape == (1, 2, 257, 188)
    err = O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[{impl} stress={stress}] cIRM rel-L2 vs reference fp64 = {err:.3e}")
    if not stress:
        fb_in = m.get_stage("fb_in", (3, 1, 257, 190), DEV).cpu().numpy()
        fb_out = m.get_stage("fb_out", (3, 1, 257, 190), DEV).cpu().numpy()
        e_in, e_out = O.rel_l2(fb_in, gi["fb_in"]), O.rel_l2(fb_out, gi["fb_out"])
        print(f"   stages: fb_in {e_in:.2e}  fb_out {e_out:.2e}")
        assert e_in < 1e-5 and e_out < 2e-3
    assert err < MASK_TOL


def test_plus_default_enhanced_waveform(built_lib, golden):
    """End of the inferencer method (inferencer.py:152-158): decompress, complex multiply, iSTFT."""
    g = golden("plus_default")
    cfg = O.default_plus_config()
    m = build_plus(cfg, O.make_params_plus(cfg, seed=0))
    with torch.no_grad():
        out = m(_t(g["mag"]), _t(g["real"]), _t(g["imag"])).cpu().numpy().astype(np.float64)
    X = g["real"][:, 0].astype(np.float64) + 1j * g["imag"][:, 0].astype(np.float64)
    enh = O.istft(O.enhance(X, out), length=48000)
    assert O.rel_l2(enh, g["enhanced"]) < 2e-3


def test_fsn_default_golden(built_lib, golden):
    gi, g = golden("plus_default"), golden("fsn_default")
    cfg = O.default_fsn_config()
    m = build_fsn(cfg, O.make_params_fsn(cfg, seed=1))
    with torch.no_grad():
        out = m(_t(gi["mag"]))
    fb_out = m.get_stage("fb_out", (1, 1, 257, 190), DEV).cpu().numpy()
    e_fb, err = O.rel_l2(fb_out[0], g["fb_out"]), O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[fullsubnet.Model] fb_out {e_fb:.2e}  cIRM {err:.3e}")
    assert e_fb < 2e-3 and err < MASK_TOL


def test_fsn_small_golden(built_lib, golden):
    g = golden("fsn_small_offline_laplace_norm")
    c = O.default_fsn_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48)
    m = build_fsn(c, O.make_params_fsn(c, seed=4))
    with torch.no_grad():
        out = m(_t(g["mag"]))
    assert O.rel_l2(out.cpu().numpy(), g["out"]) < MASK_TOL


def test_three_layer_subband(built_lib):
    """num_layers=3 (BASELINE config #5's additive knob) runs on the generic kernel."""
    cfg = small_cfg(48)
    params = O.make_params_plus(cfg, seed=9, num_layers=3)
    mag, real, imag = small_inputs(2, 33, 18, 1)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag, num_layers=3)
    m = build_plus(cfg, params, num_layers=3)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    assert m.last_lstm_impl() == "mma"
    assert O.rel_l2(out.cpu().numpy(), ref) < MASK_TOL


def test_edge_shapes(built_lib):
    """Ragged / minimal inputs the reference accepts: T just above the largest TSSE kernel, a row count that is
    not a multiple of the 128-row tile, look_ahead = 0."""
    for (B, T, la) in ((1, 9, 2), (5, 13, 0), (4, 31, 1)):
        cfg = small_cfg(64)
        cfg["look_ahead"] = la
        params = O.make_params_plus(cfg, seed=2)
        mag, real, imag = small_inputs(B, 33, T, 3)
        ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag)
        for impl in ("tcgen05", "mma"):
            m = build_plus(cfg, params, lstm_impl=impl)
            with torch.no_grad():
                out = m(_t(mag), _t(real), _t(imag))
            assert out.shape == (B, 2, 33, T)
            assert O.rel_l2(out.cpu().numpy(), ref) < MASK_TOL, (B, T, la, impl)


def test_batch_invariance_full_size(built_lib, golden):
    """Size-independent property at BASELINE's full batch (64 clips): every sample is processed independently, so
    sample i of a batched call must equal the same sample run alone
    and a permuted batch must give the permuted output."""
    g = golden("plus_default")
    cfg = O.default_plus_config()
    m = build_plus(cfg, O.make_params_plus(cfg, seed=0))
    B = 64
    rng = np.random.default_rng(0)
    scale = rng.uniform(0.3, 3.0, size=(B, 1, 1, 1)).astype(np.float32)
    shift = rng.integers(0, 188, size=B)
    mk = lambda x: np.stack([np.roll(x[0], int(s), axis=-1) for s in shift]) * scale
    mag, real, imag = mk(g["mag"]), mk(g["real"]), mk(g["imag"])
    with torch.no_grad():
        full = m(_t(mag), _t(real), _t(imag))
        assert torch.isfinite(full).all()
        for i in (0, 17, 63):
            one = m(_t(mag[i:i + 1]), _t(real[i:i + 1]), _t(imag[i:i + 1]))
            # identical arithmetic per sequence; only the fp64 atomics of the gLN statistics may reorder
            assert O.rel_l2(one[0].cpu().numpy(), full[i].cpu().numpy()) < 1e-5, i
        perm = torch.from_numpy(rng.permutation(B)).to(DEV)
        fullp = m(_t(mag)[perm], _t(real)[perm], _t(imag)[perm])
        assert O.rel_l2(fullp.cpu().numpy(), full[perm].cpu().numpy()) < 1e-5


def test_host_buffer_entry_point(built_lib):
    cfg = small_cfg(64)
    params = O.make_params_plus(cfg, seed=3)
    mag, real, imag = small_inputs(3, 33, 20, 7)
    m = build_plus(cfg, params)
    with torch.no_grad():
        dev = m(_t(mag), _t(real), _t(imag)).cpu()
    pin = lambda x: torch.from_numpy(x).pin_memory()
    host = m.forward_host(pin(mag), pin(real), pin(imag), device=DEV)
    assert torch.equal(host, dev)
    # pipelined (double-buffered, async) variant: several batches in flight, results valid after sync_host()
    outs = [m.forward_host(pin(mag * s), pin(real * s), pin(imag * s), device=DEV, pipelined=True) for s in (1.0, 2.0, 1.0, 0.5)]
    m.sync_host()
    assert torch.equal(outs[0], dev) and torch.equal(outs[2], dev)
    with torch.no_grad():
        ref2 = m(_t(mag * 2), _t(real * 2), _t(imag * 2)).cpu()
    assert torch.equal(outs[1], ref2)


@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm", "offline_gaussian_norm", "cumulative_layer_norm"])
def test_fsn_small_all_norm_types_golden(built_lib, golden, norm):
    """Every norm_type the reference's norm_wrapper accepts (base_model.py:318-330), against reference outputs."""
    g = golden(f"fsn_small_{norm}")
    c = O.default_fsn_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48, norm_type=norm)
    m = build_fsn(c, O.make_params_fsn(c, seed=4))
    with torch.no_grad():
        out = m(_t(g["mag"]))
    fb_out = m.get_stage("fb_out", (1, 3, 33, 22), DEV).cpu().numpy()
    e_fb, err = O.rel_l2(fb_out[0], g["fb_out"]), O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[fullsubnet.Model {norm}] fb_out {e_fb:.2e} cIRM {err:.3e}")
    assert err < MASK_TOL


@pytest.mark.parametrize("norm", ["offline_gaussian_norm", "cumulative_layer_norm"])
@pytest.mark.parametrize("impl", ["tcgen05", "mma"])
def test_plus_small_centred_norms_vs_oracle(built_lib, norm, impl):
    """FullSubNet+ with the centred norms (the Laplace norms divide the real/imag branches by a near-zero running
    mean and are ill-conditioned in the reference itself, SURVEY.md 7.2 -- covered on fullsubnet.Model above)."""
    cfg = small_cfg(64)
    cfg["norm_type"] = norm
    params = O.make_params_plus(cfg, seed=6)
    mag, real, imag = small_inputs(2, 33, 21, 5)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag)
    m = build_plus(cfg, params, lstm_impl=impl)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[FullSubNet+ {norm} {impl}] cIRM {err:.3e}")
    assert err < MASK_TOL


def test_config4_causal_fullsubnet_long_clip(built_lib):
    """BASELINE config #4 (streaming/causal): fullsubnet.Model + cumulative_laplace_norm, look_ahead=2.
    (a) parity with the oracle on a 6 s clip; (b) causality on a 30 s clip (T=1876): changing the input from frame t0 on
    must leave every output frame before t0 - look_ahead untouched -- the property a frame-by-frame deployment relies on."""
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=21)
    m = build_fsn(cfg, params)
    mag6 = np.abs(O.stft(O.synth_clips(1, num_samples=96000, seed0=77)))[:, None].astype(np.float32)       # [1,1,257,376]
    ref = O.fullsubnet_forward(params, cfg, mag6)
    with torch.no_grad():
        out = m(_t(mag6))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[config4 6 s] cIRM rel-L2 {err:.3e}")
    assert err < MASK_TOL
    mag30 = np.abs(O.stft(O.synth_clips(1, num_samples=480000, seed0=78)))[:, None].astype(np.float32)     # T = 1876
    assert mag30.shape[-1] == 1876
    t0 = 1200
    alt = mag30.copy()
    alt[..., t0:] *= 1.7
    with torch.no_grad():
        a, b = m(_t(mag30)), m(_t(alt))
    assert torch.isfinite(a).all()
    assert torch.equal(a[..., : t0 - 2], b[..., : t0 - 2])
    assert not torch.equal(a[..., t0:], b[..., t0:])


def test_config5_large_model(built_lib):
    """BASELINE config #5 geometry: num_freqs=513 (n_fft=1024, hop 512 -> T=94 for 3 s), sub-band hidden 512, 3-layer
    LSTMs (additive num_layers knob; oracle = SequenceModel(num_layers=3) semantics, pinned by tests/golden/lstm3_small).
    Default = layer-wise wgmma path (k_lstm_tc5r.cu); lstm_impl="mma" = generic mma.sync kernel."""
    cfg = O.default_plus_config()
    cfg.update(num_freqs=513, sb_model_hidden_size=512, fb_model_hidden_size=512)
    params = O.make_params_plus(cfg, seed=31, num_layers=3)
    X = O.stft(O.synth_clips(1, seed0=91), n_fft=1024, hop=512, win=1024)
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    assert mag.shape == (1, 1, 513, 94)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag, num_layers=3)
    m = build_plus(cfg, params, num_layers=3)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[config5 large, {m.last_lstm_impl()}] cIRM rel-L2 {err:.3e}")
    assert m.last_lstm_impl() == "tcgen05"
    assert out.shape == (1, 2, 513, 94) and err < MASK_TOL
    m = build_plus(cfg, params, num_layers=3, lstm_impl="mma")     # the generic kernel stays reachable
    with torch.no_grad():
        out_mma = m(_t(mag), _t(real), _t(imag))
    assert m.last_lstm_impl() == "mma"
    assert O.rel_l2(out_mma.cpu().numpy(), ref) < MASK_TOL


def test_fused_postprocessing_matches_torch(built_lib):
    """fsn_apply_cirm == decompress_cIRM + complex multiply of the reference inferencer (inferencer.py:152-157)."""
    from fsnplus_b200 import inference as inf
    g = torch.Generator().manual_seed(3)
    crm = (torch.randn(3, 2, 33, 20, generator=g) * 6).to(DEV)            # exercises the +-9.9 clamp
    X = torch.complex(torch.randn(3, 33, 20, generator=g), torch.randn(3, 33, 20, generator=g)).to(DEV)
    got = inf.apply_cirm(crm, X)
    m = inf.decompress_cIRM(crm)
    want = torch.complex(m[:, 0] * X.real - m[:, 1] * X.imag, m[:, 1] * X.real + m[:, 0] * X.imag)
    assert torch.allclose(torch.view_as_real(got), torch.view_as_real(want), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("norm,rnn", [("cumulative_laplace_norm", "LSTM"), ("cumulative_layer_norm", "LSTM"), ("cumulative_laplace_norm", "GRU")])
def test_streaming_step_api_matches_offline(built_lib, norm, rnn):
    """BASELINE config #4, frame-by-frame: the stateful step API (carried LSTM state + running norm sums) must reproduce
    the offline forward of the same causal model, frame for frame, and the oracle within the mask tolerance."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=65, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=96, norm_type=norm, sequence_model=rnn)
    params = O.make_params_fsn(cfg, seed=13)
    B, T = 2, 23
    mag = small_inputs(B, 65, T, 9)[0]
    ref = O.fullsubnet_forward(params, cfg, mag)
    m = build_fsn(cfg, params, lstm_impl="mma")
    with torch.no_grad():
        offline = m(_t(mag))
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    frames = []
    x = _t(mag)
    for t in range(T):
        y = st.step(x[:, 0, :, t])
        assert (y is None) == (t < cfg["look_ahead"])
        if y is not None:
            frames.append(y)
    frames += st.flush()
    st.close()
    got = torch.stack(frames, dim=-1)                      # [B, 2, F, T]
    assert got.shape == offline.shape
    e_off, e_ref = O.rel_l2(got.cpu().numpy(), offline.cpu().numpy()), O.rel_l2(got.cpu().numpy(), ref)
    print(f"\n[streaming {norm} {rnn}] vs offline {e_off:.2e}  vs oracle {e_ref:.2e}")
    assert e_off < 1e-4 and e_ref < MASK_TOL      # offline scan sums squares in fp32 per column, the step API in fp64


def test_large_batch_multiple_waves_and_long_sequence(built_lib):
    """More CTAs than SMs (B*F = 167*33 rows... small F keeps the oracle cheap; 5511 rows = 44 tiles) is covered by
    the full-size test; here: (a) odd tile count + a batch whose last pair is half empty, (b) a long sequence (T = 400) on
    FullSubNet+, both against the oracle."""
    cfg = small_cfg(64)
    params = O.make_params_plus(cfg, seed=8)
    for (B, T) in ((35, 12), (2, 400)):                     # 35*33 = 1155 rows = 10 tiles (pad to 5 pairs) ; long T
        mag, real, imag = small_inputs(B, 33, T, 11)
        ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag)
        m = build_plus(cfg, params)
        with torch.no_grad():
            out = m(_t(mag), _t(real), _t(imag))
        err = O.rel_l2(out.cpu().numpy(), ref)
        print(f"\n[B={B} T={T}] cIRM rel-L2 {err:.3e}")
        assert err < MASK_TOL


def test_default_config_batch_130(built_lib, golden):
    """B = 130 clips at the default geometry: 33 410 rows = 262 tiles = 524 CTAs of 64 rows (four waves on 132 SMs)."""
    g = golden("plus_default")
    cfg = O.default_plus_config()
    m = build_plus(cfg, O.make_params_plus(cfg, seed=0))
    B = 130
    rep = lambda x: np.repeat(x, B, axis=0)
    with torch.no_grad():
        out = m(_t(rep(g["mag"])), _t(rep(g["real"])), _t(rep(g["imag"])))
    assert out.shape == (B, 2, 257, 188)
    for i in (0, 64, 129):
        assert O.rel_l2(out[i:i + 1].cpu().numpy(), g["out"]) < MASK_TOL
    assert O.rel_l2(out[129].cpu().numpy(), out[0].cpu().numpy()) < 1e-5


def test_accurate_gate_math_variant(built_lib, golden):
    """The default gate math is 5 tanh.approx per cell (MUFU.TANH); fast_math=False selects 5 ex2 + 3 rcp.  Both must meet
    the bar and agree with each other far below it (measured: identical to 3 digits, profiles/r01_fast_math_accuracy.txt)."""
    gi, gs = golden("plus_default"), golden("plus_default_stress")
    cfg = O.default_plus_config()
    for g, scale in ((gi, 1.0), (gs, 3.0)):
        p = O.make_params_plus(cfg, seed=0, lstm_scale=scale)
        outs = []
        for fm in (True, False):
            m = build_plus(cfg, p, fast_math=fm)
            with torch.no_grad():
                outs.append(m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"])).cpu().numpy())
            err = O.rel_l2(outs[-1], g["out"])
            print(f"\n[fast_math={fm}, lstm_scale={scale}] cIRM rel-L2 {err:.3e}")
            assert err < MASK_TOL
        assert O.rel_l2(outs[0], outs[1]) < 3e-4


def test_command_line_tool_matches_reference_pipeline(built_lib, golden, tmp_path):
    """fsnplus_b200.tools.inference with the reference's flags / TOML / checkpoint format: the file written for clip 0 must be
    the reference's enhanced waveform (golden, reference torch.istft) after the int16 scaling of base_inferencer.py:151-152,
    also when the clip is enhanced inside a batch of equal-length files; an odd-length file runs as its own batch."""
    from scipy.io import wavfile
    from fsnplus_b200.tools import inference as T
    import os
    REF_TOML = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inference_reference.toml")).read()
    g = golden("plus_default")
    clips = O.synth_clips(3).astype(np.float32)
    noisy = tmp_path / "noisy"
    noisy.mkdir()
    for i, c in enumerate(clips):
        wavfile.write(noisy / f"clip{i}.wav", 16000, c)
    wavfile.write(noisy / "odd.wav", 16000, clips[1][:20000])
    cfg = O.default_plus_config()
    torch.save({"model": {k: torch.from_numpy(v) for k, v in O.make_params_plus(cfg, seed=0).items()}, "epoch": 7}, tmp_path / "ckpt.tar")
    (tmp_path / "inference.toml").write_text(REF_TOML)
    T.main(["-C", str(tmp_path / "inference.toml"), "-M", str(tmp_path / "ckpt.tar"), "-I", str(noisy), "-O", str(tmp_path / "out"),
            "--batch_size", "8"])
    out_dir = tmp_path / "out" / "enhanced_0007"
    assert sorted(p.name for p in out_dir.iterdir()) == ["clip0.wav", "clip1.wav", "clip2.wav", "odd.wav"]
    rate, pcm = wavfile.read(out_dir / "clip0.wav")
    want = T.to_int16(g["enhanced"][0])
    assert rate == 16000 and pcm.dtype == np.int16 and pcm.shape == want.shape
    err = O.rel_l2(pcm.astype(np.float64), want.astype(np.float64))
    print(f"\n[CLI] int16 enhanced waveform vs reference pipeline rel-L2 {err:.3e}, max |diff| {np.abs(pcm.astype(int) - want.astype(int)).max()} LSB")
    assert err < 2e-3
    assert wavfile.read(out_dir / "odd.wav")[1].shape == (20000,)


@pytest.mark.parametrize("L,H,rnn", [(1, 64, "LSTM"), (3, 64, "LSTM"), (3, 128, "GRU"), (4, 64, "LSTM"), (3, 192, "LSTM"), (1, 448, "LSTM")])
def test_layerwise_tcgen05_vs_oracle(built_lib, L, H, rnn):
    """Layer-wise wgmma path (k_lstm_tc5r.cu: one recurrent launch per layer, preceded by an input-projection GEMM for the deeper
    layers; default for hidden % 64 == 0, <= 512).  First / middle / last layer roles, LSTM and GRU cells, more than one cluster
    (B*F = 5*33 = 165 rows -> 2 tiles) and a half-empty last tile."""
    cfg = dict(small_cfg(H), sequence_model=rnn)
    params = O.make_params_plus(cfg, seed=40 + L, num_layers=L, lstm_scale=2.0)
    mag, real, imag = small_inputs(5, 33, 26, 12)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag, num_layers=L)
    m = build_plus(cfg, params, num_layers=L)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
        out2 = m(_t(mag), _t(real), _t(imag))
    assert m.last_lstm_impl() == "tcgen05"
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[layer-wise L={L} H={H} {rnn}] cIRM {err:.3e}")
    assert torch.equal(out, out2)
    assert err < MASK_TOL


@pytest.mark.parametrize("case", ["plus_lstm", "plus_sbtcn", "fsn_ws", "fsn_no_ws"])
def test_weights_changed_after_forward(built_lib, monkeypatch, case):
    """Parameters changed in place after a forward are pushed again at the next call, and that forward reads them everywhere: the
    attention, the full-band TCN and the layer-wise sub-band LSTM's head (H = 64), the sub-band TCN, and fullsubnet.Model's full band on
    the weight-stationary and the generic kernel with its generic sub-band LSTM.  It must match a model built with the new weights."""
    from fsnplus_b200 import _lib
    if case == "fsn_no_ws":
        monkeypatch.setenv("FSN_NO_WS", "1")
    mag, real, imag = small_inputs(2, 33, 20, 7)
    if case.startswith("plus"):
        from sbtcn_oracle import make_params
        cfg = dict(small_cfg(64), sequence_model="TCN" if case == "plus_sbtcn" else "LSTM")
        params = make_params(cfg, seed=3) if case == "plus_sbtcn" else O.make_params_plus(cfg, seed=3)
        build, x = build_plus, (mag, real, imag)
    else:
        cfg = O.default_fsn_config()
        cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48)
        params, build, x = O.make_params_fsn(cfg, seed=4), build_fsn, (mag,)
    m = build(cfg, params)
    with torch.no_grad():
        before = m(*map(_t, x)).cpu().numpy()
        for p in m.parameters():
            p.mul_(1.25)
        after = m(*map(_t, x)).cpu().numpy()
    if case.startswith("fsn"):
        assert _lib.load_library().fsn_model_last_fb_ws(m._handle) == (case == "fsn_ws")
    fresh = build(cfg, {k: v * np.float32(1.25) for k, v in params.items()})
    with torch.no_grad():
        want = fresh(*map(_t, x)).cpu().numpy()
    changed, err = O.rel_l2(after, before), O.rel_l2(after, want)
    print(f"\n[{case}] changed {changed:.3e}, vs fresh model {err:.3e}")
    assert changed > 1e-3
    assert err < 1e-6
