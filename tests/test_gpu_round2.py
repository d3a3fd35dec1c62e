"""GPU parity tests added in round 2 (all run through the C ABI via the Python mirror of the reference API).

  * the three tests that were collected last and marked xfail-until-run in round 1: now plain;
  * sb_output_activate_function on every sub-band kernel (reference sequence_model.py:84-93,120-121);
  * BASELINE config #4 at its stated size: 30 s clip (T = 1876), fullsubnet.Model + cumulative_laplace_norm, normal and x3 weights,
    truth = the CPU torch port in float32 (the float64 port / numpy oracle need minutes per 30 s clip; fp32 vs fp64 on the 6 s prefix
    with x3 weights: 7e-7.  The port is pinned to the reference goldens for every norm_type, tests/test_oracle_golden.py);
  * the streaming step API at the DEFAULT geometry (F = 257, H = 512 / 384: weight-stationary full-band kernel + generic step kernel);
  * 64 DISTINCT clips in one batch against the per-clip CPU port;
  * the pipelined entry points (fsn_model_submit / _wait, forward_host pipelined): batches in flight, results identical to forward().
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


def _small(H):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=H)
    return c


def _plus(cfg, params, **kw):
    from fsnplus_b200.model import FullSubNet_Plus
    m = FullSubNet_Plus(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))         # the C handle (which reads the FSN_* knobs ONCE) is created here, not at the first forward
    return m


def _fsn(cfg, params, **kw):
    from fsnplus_b200.model import Model
    m = Model(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    return m


def _inputs(B, F, T, seed):
    rng = np.random.default_rng(seed)
    real = rng.standard_normal((B, 1, F, T)) * 0.05 + 0.004
    imag = rng.standard_normal((B, 1, F, T)) * 0.05 - 0.003
    mag = np.sqrt(real ** 2 + imag ** 2)
    return mag.astype(np.float32), real.astype(np.float32), imag.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# formerly tests/test_gpu_zz_pending.py
# ---------------------------------------------------------------------------------------------------------------------
def test_plus_fb_num_neighbors_golden(built_lib, golden):
    """fb_num_neighbors > 0: the full-band outputs are unfolded like the sub-band window (fullsubnet_plus.py:167-179)."""
    gi, g = golden("plus_small"), golden("plus_small_fbn1")
    cfg = dict(_small(32), fb_num_neighbors=1)
    m = _plus(cfg, O.make_params_plus(cfg, seed=6))
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    err = O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[FullSubNet+ fb_num_neighbors=1] cIRM {err:.3e}")
    assert err < MASK_TOL


def test_fsn_fb_num_neighbors_golden(built_lib, golden):
    gi, g = golden("plus_small"), golden("fsn_small_fbn2")
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48, fb_num_neighbors=2)
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=6))
    with torch.no_grad():
        out = m(_t(gi["mag"]))
    err = O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[fullsubnet.Model fb_num_neighbors=2] cIRM {err:.3e}")
    assert err < MASK_TOL


def test_layerwise_path_under_fullsubnet_model_with_cumulative_norm(built_lib):
    """Layer-wise wgmma path (k_lstm_tc5r.cu) fed by the cumulative packer's images."""
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64, fb_model_hidden_size=48, norm_type="cumulative_laplace_norm")
    params = O.make_params_fsn(cfg, seed=23, num_layers=3)
    rng = np.random.default_rng(4)
    mag = np.abs(rng.standard_normal((5, 1, 33, 24)) * 0.05 + 0.01).astype(np.float32)
    ref = O.fullsubnet_forward(params, cfg, mag, num_layers=3)
    m = _fsn(cfg, params, num_layers=3)
    with torch.no_grad():
        out = m(_t(mag))
    assert m.last_lstm_impl() == "tcgen05"
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[fullsubnet.Model, 3 x 64 sub-band, cumulative_laplace_norm, layer-wise] cIRM {err:.3e}")
    assert err < MASK_TOL


# ---------------------------------------------------------------------------------------------------------------------
# sb_output_activate_function on every sub-band kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["Tanh", "ReLU", "ReLU6"])
@pytest.mark.parametrize("path", ["fused", "layerwise", "mma"])
def test_sb_output_activation(built_lib, act, path):
    """The reference applies sb_output_activate_function to the Linear output (sequence_model.py:120-121); the shipped configs use
    false, so round 1's tensor-core epilogues silently skipped it.  Tensor-core path with two layers ("fused": H = 64) and three
    layers ("layerwise") and the generic mma.sync kernel (H = 32) against the oracle."""
    H, L, impl = {"fused": (64, 2, "tcgen05"), "layerwise": (64, 3, "tcgen05"), "mma": (32, 2, "mma")}[path]
    cfg = dict(_small(H), sb_output_activate_function=act)
    params = O.make_params_plus(cfg, seed=50, num_layers=L, lstm_scale=2.0)
    params["sb_model.fc_output_layer.weight"] = params["sb_model.fc_output_layer.weight"] * 16.0    # outputs on both sides of 0 and beyond 1
    params["sb_model.fc_output_layer.bias"] = np.array([-1.0, 0.3], np.float32)
    mag, real, imag = _inputs(3, 33, 19, 21)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag, num_layers=L)
    plain = O.fullsubnet_plus_forward(params, dict(cfg, sb_output_activate_function=False), mag, real, imag, num_layers=L)
    assert O.rel_l2(plain, ref) > 0.02                                   # the activation matters on this fixture
    m = _plus(cfg, params, num_layers=L, lstm_impl=impl)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag))
    assert m.last_lstm_impl() == impl
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"\n[sb_act={act} {path}] cIRM {err:.3e}")
    assert err < MASK_TOL


# ---------------------------------------------------------------------------------------------------------------------
# BASELINE config #4 at its stated size
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1.0, 3.0])
def test_config4_30s_clip_parity(built_lib, scale):
    """fullsubnet.Model + cumulative_laplace_norm, look_ahead 2, one 30 s clip (T = 1876), against the float32 CPU port; scale 3
    multiplies every LSTM weight by 3 (saturated gates, like a trained network) -- the long-clip worst case for fp16 h
    re-quantisation.  Also reports the error of the last second alone (drift would show there)."""
    from oracle.torch_port import TorchPort
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=21, lstm_scale=scale)
    mag = np.abs(O.stft(O.synth_clips(1, num_samples=480000, seed0=78)))[:, None].astype(np.float32)
    assert mag.shape == (1, 1, 257, 1876)
    ref = TorchPort(params, cfg, "fsn", dtype=torch.float32).forward(torch.from_numpy(mag)).numpy()
    m = _fsn(cfg, params)
    with torch.no_grad():
        out = m(_t(mag)).cpu().numpy()
    err, tail = O.rel_l2(out, ref), O.rel_l2(out[..., -63:], ref[..., -63:])
    print(f"\n[config4 30 s, lstm x{scale}] cIRM rel-L2 {err:.3e} (last second {tail:.3e})")
    assert np.isfinite(out).all()
    assert err < MASK_TOL and tail < 2 * MASK_TOL


def test_config4_30s_clip_plus_offline(built_lib):
    """FullSubNet+ cannot stream (TSSE pools over all time); SURVEY 8d asks for its offline number on the same 30 s clip."""
    from oracle.torch_port import TorchPort
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=0)
    X = O.stft(O.synth_clips(1, num_samples=480000, seed0=78))
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    ref = TorchPort(params, cfg, "plus", dtype=torch.float32).forward(*(torch.from_numpy(x) for x in (mag, real, imag))).numpy()
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag)).cpu().numpy()
    err = O.rel_l2(out, ref)
    print(f"\n[FullSubNet+ 30 s offline] cIRM rel-L2 {err:.3e}")
    assert err < MASK_TOL


@pytest.mark.parametrize("B", [1, 3])
def test_streaming_step_api_default_geometry(built_lib, B):
    """The path scripts/bench_stream.py and `bench.py --config 4` time: F = 257, full-band H = 512 (weight-stationary kernel),
    sub-band H = 384 (generic step kernel), cumulative_laplace_norm, frame by frame; against the oracle and the offline forward."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    T = 40
    mag = np.abs(O.stft(O.synth_clips(B, num_samples=256 * (T - 1), seed0=500)))[:, None].astype(np.float32)
    assert mag.shape == (B, 1, 257, T)
    ref = O.fullsubnet_forward(params, cfg, mag)
    m = _fsn(cfg, params)
    with torch.no_grad():
        offline = m(_t(mag))
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    x, frames = _t(mag), []
    for t in range(T):
        y = st.step(x[:, 0, :, t])
        assert (y is None) == (t < cfg["look_ahead"])
        if y is not None:
            frames.append(y)
    frames += st.flush()
    st.close()
    got = torch.stack(frames, dim=-1).cpu().numpy()
    e_off, e_ref, e_offline = O.rel_l2(got, offline.cpu().numpy()), O.rel_l2(got, ref), O.rel_l2(offline.cpu().numpy(), ref)
    print(f"\n[streaming default geometry B={B}] step vs offline {e_off:.2e}; step vs oracle {e_ref:.3e}; offline vs oracle {e_offline:.3e}")
    assert e_ref < MASK_TOL and e_offline < MASK_TOL and e_off < MASK_TOL


def test_batch_of_64_distinct_clips_vs_cpu_port(built_lib):
    """BASELINE config #2's batch with 64 DIFFERENT clips (seeds 1000..1063, SNR -5..20 dB, levels -35..-15 dBFS): every sample
    of the batched GPU forward against the per-clip fp32 CPU port (the reference's ATen op sequence, one clip per call)."""
    from oracle.torch_port import TorchPort
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=0)
    X = O.stft(O.synth_clips(64))
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag)).cpu().numpy()
    port = TorchPort(params, cfg, "plus")
    torch.set_num_threads(min(16, torch.get_num_threads()))
    errs = []
    for i in range(64):
        ref = port.forward(*(torch.from_numpy(x[i:i + 1]) for x in (mag, real, imag))).numpy()
        errs.append(O.rel_l2(out[i:i + 1], ref))
    print(f"\n[64 distinct clips] cIRM rel-L2 vs CPU port: max {max(errs):.3e}  median {np.median(errs):.3e}")
    assert max(errs) < MASK_TOL


def test_plus_extreme_real_imag_scale(built_lib):
    """offline_laplace_norm divides the real / imaginary branches by their MEAN (base_model.py:210-225), which is ~0 for any audio:
    the normalised branches reach 1e5 x the input (1e6 on the ordinary fixtures).  Here: a loud clip (x30) whose real and imaginary
    parts have exactly zero mean -> the scale is the 1 / 1e-5 of the epsilon and the TCN streams reach ~1e8, far beyond fp16.  The
    fp16 hidden activations of the TCN are stored with a per-sample power-of-two scale (fp16_store_scale) and must hold parity."""
    from oracle.torch_port import TorchPort
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=0)
    X = 30.0 * O.stft(O.synth_clips(2, seed0=4321))
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    real -= real.mean(axis=(1, 2, 3), keepdims=True)
    imag -= imag.mean(axis=(1, 2, 3), keepdims=True)
    peak = float(np.abs(real).max() / (abs(float(real[0].mean())) + 1e-5))
    ref = TorchPort(params, cfg, "plus", dtype=torch.float64).forward(*(torch.from_numpy(x).double() for x in (mag, real, imag))).numpy()
    ref32 = TorchPort(params, cfg, "plus", dtype=torch.float32).forward(*(torch.from_numpy(x) for x in (mag, real, imag))).numpy()
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(mag), _t(real), _t(imag)).cpu().numpy()
    err, err32 = O.rel_l2(out, ref), O.rel_l2(ref32, ref)
    print(f"\n[extreme real/imag scale: normalised peak {peak:.1e}] cIRM rel-L2 vs fp64 {err:.3e} (the reference's own fp32 arithmetic: {err32:.3e})")
    # at this scale the reference's fp32 arithmetic itself is ~1.5e-3 from the fp64 truth: the bar is the larger of 1e-3 and twice that
    assert peak > 1e7 and err < max(MASK_TOL, 2 * err32)


# ---------------------------------------------------------------------------------------------------------------------
# pipelined entry points
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("overlap", ["0", "1"])
def test_submit_wait_matches_forward(built_lib, golden, monkeypatch, overlap):
    """fsn_model_submit / fsn_model_wait: five batches in flight, default geometry, different batch contents; every result must be
    bit-identical to forward() up to the order of the fp64 atomics of the gLN statistics.  overlap = 1 (FSN_FRONT_OVERLAP, read at
    model creation): two workspace lanes, the front end of batch i+1 concurrent with the sub-band LSTM of batch i."""
    monkeypatch.setenv("FSN_FRONT_OVERLAP", overlap)
    g = golden("plus_default")
    cfg = O.default_plus_config()
    m = _plus(cfg, O.make_params_plus(cfg, seed=0))
    B = 6
    rng = np.random.default_rng(5)
    batches = []
    for k in range(5):
        scale = rng.uniform(0.3, 3.0, size=(B, 1, 1, 1)).astype(np.float32)
        shift = rng.integers(0, 188, size=B)
        mk = lambda x: _t(np.stack([np.roll(x[0], int(s), axis=-1) for s in shift]) * scale)
        batches.append((mk(g["mag"]), mk(g["real"]), mk(g["imag"])))
    with torch.no_grad():
        want = [m(*b) for b in batches]
        torch.cuda.synchronize()
        outs = [m.submit(*b) for b in batches]
        m.wait()
        torch.cuda.synchronize()
        for k in range(5):
            assert O.rel_l2(outs[k].cpu().numpy(), want[k].cpu().numpy()) < 1e-5, k
        # a plain forward right after pipelined work, and pipelined work right after a plain forward
        o1 = m.submit(*batches[0])
        o2 = m(*batches[1])
        o3 = m.submit(*batches[2])
        m.wait()
        torch.cuda.synchronize()
        for o, k in ((o1, 0), (o2, 1), (o3, 2)):
            assert O.rel_l2(o.cpu().numpy(), want[k].cpu().numpy()) < 1e-5, k


def test_submit_fullsubnet_model_single_lane(built_lib):
    """fullsubnet.Model through the pipelined API (one lane, no overlap: its full-band LSTM is a cooperative launch)."""
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64, fb_model_hidden_size=48)
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=4))
    xs = [_t(_inputs(3, 33, 22, s)[0]) for s in (1, 2, 3)]
    with torch.no_grad():
        want = [m(x) for x in xs]
        outs = [m.submit(x) for x in xs]
        m.wait()
    torch.cuda.synchronize()
    for a, b in zip(outs, want):
        assert torch.equal(a, b)


def test_forward_host_pipelined_default_geometry(built_lib, golden):
    """Host-buffer pipelined entry point at the default geometry, four batches, against forward()."""
    g = golden("plus_default")
    cfg = O.default_plus_config()
    m = _plus(cfg, O.make_params_plus(cfg, seed=0))
    pin = lambda x: torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
    hb = [tuple(pin(np.repeat(g[k], 4, axis=0) * s) for k in ("mag", "real", "imag")) for s in (1.0, 0.5, 2.0, 1.5)]
    with torch.no_grad():
        want = [m(*(x.to(DEV) for x in b)).cpu() for b in hb]
    outs = [m.forward_host(*b, device=DEV, pipelined=True) for b in hb]
    m.sync_host()
    for a, b in zip(outs, want):
        assert O.rel_l2(a.numpy(), b.numpy()) < 1e-5
    with pytest.raises(ValueError):
        m.forward_host(hb[0][0].double(), hb[0][1], hb[0][2], device=DEV)
    with pytest.raises(ValueError):
        m.forward_host(torch.from_numpy(np.ascontiguousarray(g["mag"])), hb[0][1][:1], hb[0][2][:1], device=DEV, pipelined=True)   # not pinned


# ---------------------------------------------------------------------------------------------------------------------
# causal FullSubNet+ variant (SURVEY.md 8f rank 2)
# ---------------------------------------------------------------------------------------------------------------------
def test_causal_tcn_variant(built_lib, golden):
    """TCNBlock(causal=True) in the full-band models: small config against the committed reference golden (incl. the fb_out
    stage), default geometry against the oracle, and the causality property of the full-band TCN chain's taps (with the
    non-causal gLN statistics held fixed this cannot be tested end to end, so the check is the golden)."""
    g, gi = golden("plus_small_causal"), golden("plus_small")
    cfg = dict(_small(32), causal_tcn=True)
    m = _plus(cfg, O.make_params_plus(cfg, seed=14))
    with torch.no_grad():
        out = m(_t(gi["mag"]), _t(gi["real"]), _t(gi["imag"]))
    fb_out = m.get_stage("fb_out", (3, 3, 33, 22), DEV).cpu().numpy()
    e_fb, err = O.rel_l2(fb_out, g["fb_out"]), O.rel_l2(out.cpu().numpy(), g["out"])
    print(f"\n[causal TCN small] fb_out {e_fb:.2e} cIRM {err:.3e}")
    assert e_fb < 2e-3 and err < MASK_TOL
    gd = golden("plus_default")
    cfg = dict(O.default_plus_config(), causal_tcn=True)
    params = O.make_params_plus(cfg, seed=0)
    ref = O.fullsubnet_plus_forward(params, cfg, gd["mag"], gd["real"], gd["imag"])
    m = _plus(cfg, params)
    with torch.no_grad():
        out = m(_t(gd["mag"]), _t(gd["real"]), _t(gd["imag"]))
    err = O.rel_l2(out.cpu().numpy(), ref)
    print(f"[causal TCN default geometry] cIRM {err:.3e} (differs from the non-causal golden by {O.rel_l2(ref, gd['out']):.2e})")
    assert err < MASK_TOL


# ---------------------------------------------------------------------------------------------------------------------
# fused post-processing (SURVEY.md 8f rank 1): decompress_cIRM x noisy spectrum in the LSTM epilogue
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["fused", "layerwise", "mma"])
def test_enhance_spectrum_matches_mask_then_postprocess(built_lib, path):
    """fsn_model_forward_enhance == fsn_model_forward followed by the reference's decompress_cIRM + complex multiply
    (inferencer.py:152-157, mask.py:60-63), on the three sub-band kernels; masks scaled so the +-9.9 clamp is exercised."""
    from fsnplus_b200 import inference as inf
    H, L, impl = {"fused": (64, 2, "tcgen05"), "layerwise": (64, 3, "tcgen05"), "mma": (32, 2, "mma")}[path]
    cfg = _small(H)
    params = O.make_params_plus(cfg, seed=61, num_layers=L, lstm_scale=2.0)
    params["sb_model.fc_output_layer.weight"] = params["sb_model.fc_output_layer.weight"] * 150.0
    mag, real, imag = _inputs(3, 33, 21, 17)
    m = _plus(cfg, params, num_layers=L, lstm_impl=impl)
    X = torch.complex(_t(real)[:, 0], _t(imag)[:, 0])
    with torch.no_grad():
        crm = m(_t(mag), _t(real), _t(imag))
        assert (crm.abs() > 9.9).any() and (crm.abs() < 9.9).any()
        d = inf.decompress_cIRM(crm)
        want = torch.complex(d[:, 0] * X.real - d[:, 1] * X.imag, d[:, 1] * X.real + d[:, 0] * X.imag)
        got = m.enhance_spectrum(_t(mag), _t(real), _t(imag))
        got_p = m.enhance_spectrum(_t(mag), _t(real), _t(imag), pipelined=True)
        m.wait()
    torch.cuda.synchronize()
    assert got.dtype == torch.complex64 and got.shape == (3, 33, 21)
    assert torch.allclose(torch.view_as_real(got), torch.view_as_real(want), rtol=2e-5, atol=1e-6)
    assert torch.equal(torch.view_as_real(got), torch.view_as_real(got_p))


def test_enhance_pipeline_matches_enhance_batch(built_lib, golden):
    """EnhancePipeline (pipelined submit, fused post-processing, side-stream iSTFT) == enhance_batch per batch == the reference
    pipeline's waveform on the golden clip."""
    from fsnplus_b200 import inference as inf
    g = golden("plus_default")
    cfg = O.default_plus_config()
    m = _plus(cfg, O.make_params_plus(cfg, seed=0))
    clips = torch.from_numpy(O.synth_clips(6).astype(np.float32)).to(DEV)
    batches = [clips[0:2], clips[2:4], clips[4:6], clips[0:2]]
    want = [inf.enhance_batch(m, b) for b in batches]
    for fused in (True, False):
        pipe = inf.EnhancePipeline(m, 48000, fused_post=fused)
        for b in batches:
            pipe.push(inf.stft(b))
        got = [r.clone() for r in pipe.flush()]                   # ring of 4 result slots: all four are still intact
        for k in range(4):
            assert O.rel_l2(got[k].cpu().numpy(), want[k].cpu().numpy()) < 1e-5, (fused, k)
    assert O.rel_l2(want[0][0].cpu().numpy(), g["enhanced"][0]) < 2e-3
    pin = lambda x: x.cpu().pin_memory()
    pipe = inf.EnhancePipeline(m, 48000, to_host=True, keep_results=False)
    outs = []
    for b in batches[:2]:
        X = inf.stft(b)
        pipe.push(host=(pin(X.abs().unsqueeze(1)), pin(X.real.unsqueeze(1).contiguous()), pin(X.imag.unsqueeze(1).contiguous())))
    pipe.flush()
    for k in (0, 1):
        assert O.rel_l2(pipe.host_out[k].numpy(), want[k].cpu().numpy()) < 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# small configurations and batch sizes on the tensor-core LSTM path (these once covered a small-batch column-split mode of an
# earlier kernel; the parameter S now only varies the weights' seed)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,S,rnn", [(64, 2, "LSTM"), (128, 2, "LSTM"), (128, 4, "LSTM"), (128, 4, "GRU"), (256, 4, "LSTM"), (192, 6, "LSTM"), (384, 6, "GRU")])
def test_column_split_small_configs(built_lib, H, S, rnn):
    """Against the oracle and against a second model instance: several row tiles (B*F = 9*33 = 297 rows -> 3 tiles -> 2 tile pairs,
    the second half empty), sb activation on, fused enhance output."""
    cfg = dict(_small(H), sequence_model=rnn, sb_output_activate_function="Tanh")
    params = O.make_params_plus(cfg, seed=70 + S, lstm_scale=2.0)
    mag, real, imag = _inputs(9, 33, 23, 31)
    ref = O.fullsubnet_plus_forward(params, cfg, mag, real, imag)
    m1 = _plus(cfg, params, lstm_impl="tcgen05")
    ms = _plus(cfg, params, lstm_impl="tcgen05")
    with torch.no_grad():
        o1 = m1(_t(mag), _t(real), _t(imag))
        os_ = ms(_t(mag), _t(real), _t(imag))
        os2 = ms(_t(mag), _t(real), _t(imag))
        e1 = m1.enhance_spectrum(_t(mag), _t(real), _t(imag))
        es = ms.enhance_spectrum(_t(mag), _t(real), _t(imag))
    err, dsplit = O.rel_l2(os_.cpu().numpy(), ref), O.rel_l2(os_.cpu().numpy(), o1.cpu().numpy())
    print(f"\n[small config H={H} S={S} {rnn}] cIRM vs oracle {err:.3e}; vs second instance {dsplit:.2e}")
    assert torch.equal(os_, os2)                                         # deterministic
    assert err < MASK_TOL and dsplit < 1e-5                              # same arithmetic
    assert O.rel_l2(torch.view_as_real(es).cpu().numpy(), torch.view_as_real(e1).cpu().numpy()) < 1e-5


@pytest.mark.parametrize("B", [1, 2, 8, 20])
def test_column_split_default_geometry_auto(built_lib, golden, B):
    """Default geometry at small and medium batch sizes (B = 20 -> 21 row-tile pairs): sample 0 is the golden clip, the others are
    shifted / scaled copies; every sample against a second model instance, sample 0 against the reference golden."""
    g = golden("plus_default")
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=0)
    m = _plus(cfg, params)
    m1 = _plus(cfg, params)
    rng = np.random.default_rng(B)
    sc = np.concatenate([[1.0], rng.uniform(0.5, 2.0, B - 1)]).astype(np.float32).reshape(B, 1, 1, 1)
    sh = np.concatenate([[0], rng.integers(0, 188, B - 1)])
    rep = lambda x: np.stack([np.roll(x[0], int(k), axis=-1) for k in sh]) * sc
    ins = [_t(rep(g[k])) for k in ("mag", "real", "imag")]
    with torch.no_grad():
        out, out1 = m(*ins), m1(*ins)
    e0, d = O.rel_l2(out[0:1].cpu().numpy(), g["out"]), O.rel_l2(out.cpu().numpy(), out1.cpu().numpy())
    print(f"\n[default geometry B={B}] sample 0 vs reference golden {e0:.3e}; batch vs second instance {d:.2e}")
    assert e0 < MASK_TOL and d < 1e-5


def test_internal_batch_split_under_a_workspace_cap(built_lib, monkeypatch):
    """FSN_WS_CAP_GB (read at model creation): a batch whose workspace would exceed the cap runs as equal sub-batches on the same stream;
    samples are independent, so the result equals the unsplit forward.  Layer-wise path (its time-batched input projection is the big
    buffer) with three and two layers; mask and fused-enhance outputs."""
    for L, H in ((3, 64), (2, 64)):
        cfg = _small(H)
        params = O.make_params_plus(cfg, seed=81, num_layers=L)
        mag, real, imag = _inputs(11, 33, 20, 41)
        m = _plus(cfg, params, num_layers=L)
        monkeypatch.setenv("FSN_WS_CAP_GB", "0.002")                   # ~2 MB: forces 3-4 sub-batches at this geometry
        ms = _plus(cfg, params, num_layers=L)
        monkeypatch.delenv("FSN_WS_CAP_GB")
        with torch.no_grad():
            a, b = m(_t(mag), _t(real), _t(imag)), ms(_t(mag), _t(real), _t(imag))
            ea, eb = m.enhance_spectrum(_t(mag), _t(real), _t(imag)), ms.enhance_spectrum(_t(mag), _t(real), _t(imag))
        assert ms.last_launch_count() > m.last_launch_count()          # it really ran several sub-batches
        assert O.rel_l2(b.cpu().numpy(), a.cpu().numpy()) < 1e-5
        assert O.rel_l2(torch.view_as_real(eb).cpu().numpy(), torch.view_as_real(ea).cpu().numpy()) < 1e-5


@pytest.mark.parametrize("B", [2, 20])
def test_chained_front_end_launches_match_plain_launches(built_lib, monkeypatch, B):
    """FSN_PDL (read at model creation): programmatic dependent launch of the front-end kernel chain (every kernel runs
    griddepcontrol.launch_dependents / griddepcontrol.wait).  Default geometry; B = 2 is inside the automatic small-batch regime, B = 20
    outside it, so both settings are forced.  The two paths run the same kernels in the same order: equal up to the order of the fp64
    atomics of the gLN statistics, over several back-to-back forwards (the chain of forward i+1 follows the LSTM of forward i)."""
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=0)
    X = O.stft(O.synth_clips(B, seed0=7000))
    mag, real, imag = (np.abs(X)[:, None].astype(np.float32), X.real[:, None].astype(np.float32), X.imag[:, None].astype(np.float32))
    monkeypatch.setenv("FSN_PDL", "0")
    m0 = _plus(cfg, params)
    monkeypatch.setenv("FSN_PDL", "1")
    m1 = _plus(cfg, params)
    monkeypatch.delenv("FSN_PDL")
    with torch.no_grad():
        outs0 = [m0(_t(mag), _t(real), _t(imag)).clone() for _ in range(3)]
        outs1 = [m1(_t(mag), _t(real), _t(imag)).clone() for _ in range(3)]
    for a, b in zip(outs0, outs1):
        assert O.rel_l2(b.cpu().numpy(), a.cpu().numpy()) < 1e-5
    assert O.rel_l2(outs1[2].cpu().numpy(), outs1[0].cpu().numpy()) < 1e-5
