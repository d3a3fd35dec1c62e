"""FullSubNet+ with a TCN sub-band model (sequence_model = "TCN", reference fullsubnet_plus.py:45,102-110) on the GPU.

The sub-band TCN runs on the full-band TCN's kernels (k_gemm_tc5.cu): tf32 first 1x1 convolution on the fp32 residual stream, fp16
hidden activations with a per-sequence power-of-two store scale, the gLN folded into the second 1x1 convolution, and a last epilogue
(EPI5_GLN_HEAD) that applies ReLU + Linear + activation and writes the mask.  Bar: cIRM rel-L2 <= 1e-3 against the fp64 reference.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASK_TOL = 1e-3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _small(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, sequence_model="TCN")
    c.update(over)
    return c


def _plus(cfg, params, **kw):
    from fsnplus_b200.model import FullSubNet_Plus
    m = FullSubNet_Plus(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))         # the C handle reads the FSN_* knobs once, here
    return m


def _inputs(B, F, T, seed):
    rng = np.random.default_rng(seed)
    real = rng.standard_normal((B, 1, F, T)) * 0.05 + 0.004
    imag = rng.standard_normal((B, 1, F, T)) * 0.05 - 0.003
    mag = np.sqrt(real ** 2 + imag ** 2)
    return mag.astype(np.float32), real.astype(np.float32), imag.astype(np.float32)


def _clips(n, num_samples=48000, seed0=1000):
    X = O.stft(O.synth_clips(n, num_samples=num_samples, seed0=seed0))
    return np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32)


def _sb_in_from_stages(m, cfg, B, Tp):
    """The sub-band input the packer must produce from this forward's own full-band stages (fullsubnet_plus.py:167-189), in fp64:
    the packer's arithmetic alone, without the full-band model's tf32 / fp16 error."""
    F, ns, nfb = cfg["num_freqs"], cfg["sb_num_neighbors"], cfg["fb_num_neighbors"]
    fb_in = m.get_stage("fb_in", (3, B, F, Tp), DEV).cpu().double().numpy()
    fb_out = m.get_stage("fb_out", (3, B, F, Tp), DEV).cpu().double().numpy()
    unf = [O.unfold(fb_out[k][:, None], nfb).reshape(B, F, 2 * nfb + 1, Tp) for k in range(3)]
    win = O.unfold(fb_in[0][:, None], ns).reshape(B, F, 2 * ns + 1, Tp)
    return O.NORMS[cfg["norm_type"]](np.concatenate([win] + unf, axis=2))


def test_small_golden_and_sb_in_stage(built_lib, golden):
    """The reference golden; the sb_in stage against the golden (it inherits the full-band model's error) and, at fp32 rounding,
    against the same normalisation applied in fp64 to this forward's own full-band stages."""
    g, gi = golden("plus_small_sbTCN"), golden("plus_small")
    cfg = _small()
    m = _plus(cfg, S.make_params(cfg, seed=int(g["seed"])))
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    assert m.last_lstm_impl() == "tcn"
    sb_in = m.get_stage("sb_in", g["sb_in"].shape, DEV).cpu().numpy()
    e_pack = O.rel_l2(sb_in, _sb_in_from_stages(m, cfg, 3, 22))
    e_sb, err = O.rel_l2(sb_in, g["sb_in"]), O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[sub-band TCN small golden] sb_in vs golden {e_sb:.2e}, vs own stages {e_pack:.2e}; cIRM {err:.3e}")
    assert e_pack < 1e-6 and e_sb < 2e-3 and err < MASK_TOL


@pytest.mark.parametrize("scale", [1.0, 3.0])
def test_default_golden(built_lib, golden, scale):
    """Default geometry (F = 257, Isb = 34), one 3 s clip: the reference golden for the default weights, the oracle for x3 weights."""
    gd = golden("plus_default")
    cfg = dict(O.default_plus_config(), sequence_model="TCN")
    params = S.make_params(cfg, seed=0, scale=scale)
    ref = golden("plus_default_sbTCN")["out"] if scale == 1.0 else S.forward(params, cfg, gd["mag"], gd["real"], gd["imag"])
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(gd["mag"]), _t(gd["real"]), _t(gd["imag"]))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[sub-band TCN default geometry x{scale}] cIRM {err:.3e}")
    assert err < MASK_TOL


VARIANTS = {
    "cumulative_laplace_norm": dict(norm_type="cumulative_laplace_norm"),
    "offline_gaussian_norm": dict(norm_type="offline_gaussian_norm"),
    "cumulative_layer_norm": dict(norm_type="cumulative_layer_norm"),
    "fb_num_neighbors_1": dict(fb_num_neighbors=1),
    "SE": dict(channel_attention_model="SE"),
    "ECA": dict(channel_attention_model="ECA"),
    "CBAM": dict(channel_attention_model="CBAM"),
    "ECA_subband_num_2": dict(channel_attention_model="ECA", subband_num=2),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_variants_against_oracle(built_lib, name):
    """Every norm type (offline_laplace_norm is the golden), fb_num_neighbors > 0, every attention, subband_num > 1: the sub-band
    input packer (at fp32 rounding, against the normalisation of this forward's own full-band stages) and the TCN against the fp64
    oracle."""
    cfg = _small(**VARIANTS[name])
    params = S.make_params(cfg, seed=90)
    mag, real, imag = _inputs(3, 33, 23, 29)
    ref = S.forward(params, cfg, mag, real, imag)
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    sb_in = m.get_stage("sb_in", (3, 33, 10 + 6 * cfg["fb_num_neighbors"], 25), DEV).cpu().numpy()
    e_pack, err = O.rel_l2(sb_in, _sb_in_from_stages(m, cfg, 3, 25)), O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[sub-band TCN {name}] sb_in vs own stages {e_pack:.2e} cIRM {err:.3e}")
    assert e_pack < 1e-5 and err < MASK_TOL


@pytest.mark.parametrize("act", ["Tanh", "ReLU", "ReLU6"])
def test_output_activation(built_lib, act):
    cfg = _small(sb_output_activate_function=act)
    params = S.make_params(cfg, seed=91)
    params["sb_model.fc_output_layer.weight"] = params["sb_model.fc_output_layer.weight"] * 4.0     # outputs on both sides of 0 and beyond 1
    params["sb_model.fc_output_layer.bias"] = np.array([-1.0, 0.3], np.float32)
    mag, real, imag = _inputs(3, 33, 19, 21)
    ref = S.forward(params, cfg, mag, real, imag)
    plain = S.forward(params, dict(cfg, sb_output_activate_function=False), mag, real, imag)
    assert O.rel_l2(plain, ref) > 0.02                                   # the activation matters on this fixture
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[sub-band TCN sb_act={act}] cIRM {err:.3e}")
    assert err < MASK_TOL


def test_x3_weights_small(built_lib):
    cfg = _small()
    params = S.make_params(cfg, seed=92, scale=3.0)
    mag, real, imag = _inputs(4, 33, 26, 5)
    ref = S.forward(params, cfg, mag, real, imag)
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[sub-band TCN x3 weights small] cIRM {err:.3e}")
    assert err < MASK_TOL


def test_batch_of_64_distinct_clips(built_lib):
    """64 different 3 s clips in one batch: every sample equals the same clip run alone and matches the per-clip fp32 CPU torch port
    (the reference's ATen op sequence)."""
    cfg = dict(O.default_plus_config(), sequence_model="TCN")
    params = S.make_params(cfg, seed=0)
    mag, real, imag = _clips(64)
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag)).cpu().numpy()
        alone = [m(_t(mag[i:i + 1]), _t(real[i:i + 1]), _t(imag[i:i + 1])).cpu().numpy() for i in range(64)]
    d_alone = max(O.rel_l2(out[i:i + 1], alone[i]) for i in range(64))
    port = S.TcnPort(params, cfg)
    errs = [O.rel_l2(out[i:i + 1], port.forward(*(torch.from_numpy(x[i:i + 1]) for x in (mag, real, imag))).numpy())
            for i in range(64)]
    print(f"\n[sub-band TCN 64 distinct clips] batch vs alone max {d_alone:.2e}; vs CPU port max {max(errs):.3e}")
    assert d_alone < 1e-5 and max(errs) < MASK_TOL


def test_30s_clip(built_lib):
    cfg = dict(O.default_plus_config(), sequence_model="TCN")
    params = S.make_params(cfg, seed=0)
    mag, real, imag = _clips(1, num_samples=480000, seed0=78)
    assert mag.shape == (1, 1, 257, 1876)
    ref = S.TcnPort(params, cfg).forward(*(torch.from_numpy(x) for x in (mag, real, imag))).numpy()
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag)).cpu().numpy()
    err, tail = O.rel_l2(out, ref), O.rel_l2(out[..., -63:], ref[..., -63:])
    print(f"\n[sub-band TCN 30 s clip] cIRM rel-L2 {err:.3e} (last second {tail:.3e})")
    assert np.isfinite(out).all() and err < MASK_TOL


def test_other_entry_points_agree_with_forward(built_lib, golden):
    """enhance_spectrum == the mask followed by fsn_apply_cirm (masks scaled so the +-9.9 clamp is exercised); submit / wait and
    forward_host(pipelined=True) == forward up to the order of the fp64 gLN atomics."""
    cfg = _small()
    params = S.make_params(cfg, seed=93)
    params["sb_model.fc_output_layer.weight"] = params["sb_model.fc_output_layer.weight"] * 40.0
    mag, real, imag = _inputs(5, 33, 21, 17)
    m = _plus(cfg, params)
    noisy = torch.view_as_real(torch.complex(_t(real)[:, 0], _t(imag)[:, 0])).contiguous()
    with torch.no_grad():
        crm = m(_t(mag), _t(real), _t(imag))
        assert (crm.abs() > 9.9).any() and (crm.abs() < 9.9).any()
        want = torch.empty_like(noisy)
        stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
        assert built_lib.fsn_apply_cirm(C.c_void_p(crm.data_ptr()), C.c_void_p(noisy.data_ptr()), C.c_void_p(want.data_ptr()),
                                        5, 33, 21, stream) == 0
        got = m.enhance_spectrum(_t(mag), _t(real), _t(imag))
        got_p = m.enhance_spectrum(_t(mag), _t(real), _t(imag), pipelined=True)
        m.wait()
    torch.cuda.synchronize()
    assert got.dtype == torch.complex64 and got.shape == (5, 33, 21)
    assert torch.allclose(torch.view_as_real(got), want, rtol=2e-5, atol=1e-6)
    assert O.rel_l2(torch.view_as_real(got_p).cpu().numpy(), torch.view_as_real(got).cpu().numpy()) < 1e-5

    g = golden("plus_default")
    dcfg = dict(O.default_plus_config(), sequence_model="TCN")
    md = _plus(dcfg, S.make_params(dcfg, seed=0))
    rng = np.random.default_rng(5)
    batches = []
    for k in range(4):
        scale = rng.uniform(0.3, 3.0, size=(3, 1, 1, 1)).astype(np.float32)
        shift = rng.integers(0, 188, size=3)
        batches.append(tuple(np.stack([np.roll(g[key][0], int(s), axis=-1) for s in shift]) * scale for key in ("mag", "real", "imag")))
    with torch.no_grad():
        want = [md(*(_t(x) for x in b)).cpu().numpy() for b in batches]
        outs = [md.submit(*(_t(x) for x in b)) for b in batches]
        md.wait()
    torch.cuda.synchronize()
    for k in range(4):
        assert O.rel_l2(outs[k].cpu().numpy(), want[k]) < 1e-5, k
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
    hb = [tuple(pin(x) for x in b) for b in batches]
    houts = [md.forward_host(*b, device=DEV, pipelined=True) for b in hb]
    md.sync_host()
    for k in range(4):
        assert O.rel_l2(houts[k].numpy(), want[k]) < 1e-5, k


def test_sub_batches_under_a_workspace_cap(built_lib, monkeypatch):
    """FSN_WS_CAP_GB (read at model creation): a batch whose workspace would exceed the cap runs as equal sub-batches with the same
    result; mask and fused-enhance outputs."""
    cfg = _small()
    params = S.make_params(cfg, seed=94)
    mag, real, imag = _inputs(11, 33, 20, 41)
    m = _plus(cfg, params)
    monkeypatch.setenv("FSN_WS_CAP_GB", "0.004")                       # a few MB: forces several sub-batches at this geometry
    ms = _plus(cfg, params)
    monkeypatch.delenv("FSN_WS_CAP_GB")
    with torch.no_grad():
        a, b = m(_t(mag), _t(real), _t(imag)), ms(_t(mag), _t(real), _t(imag))
        ea, eb = m.enhance_spectrum(_t(mag), _t(real), _t(imag)), ms.enhance_spectrum(_t(mag), _t(real), _t(imag))
    assert ms.last_launch_count() > m.last_launch_count()              # it really ran several sub-batches
    assert O.rel_l2(b.cpu().numpy(), a.cpu().numpy()) < 1e-5
    assert O.rel_l2(torch.view_as_real(eb).cpu().numpy(), torch.view_as_real(ea).cpu().numpy()) < 1e-5


def test_more_than_65535_sequences(built_lib):
    """B = 256 clips at F = 257: 65792 sequences, more than gridDim.z allows (the depth-wise convolution folds them into grid x).
    Short clips (T = 9, the shortest the TSSE attention's kernel of 10 frames accepts with look_ahead 2); the batch equals the same
    clips run in batches of 64."""
    cfg = dict(O.default_plus_config(), sequence_model="TCN")
    params = S.make_params(cfg, seed=0)
    mag, real, imag = _clips(256, num_samples=256 * 8, seed0=3000)
    assert mag.shape == (256, 1, 257, 9)
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag)).cpu().numpy()
        parts = np.concatenate([m(_t(mag[i:i + 64]), _t(real[i:i + 64]), _t(imag[i:i + 64])).cpu().numpy() for i in range(0, 256, 64)])
    d = O.rel_l2(out, parts)
    print(f"\n[sub-band TCN B = 256, F = 257] batch vs batches of 64 {d:.2e}")
    assert np.isfinite(out).all() and d < 1e-5
