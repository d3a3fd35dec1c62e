"""Long clips with the sub-band TCN on the GPU: the sub-band TCN in bin chunks (DESIGN.md §3.8).

Truth is the unchunked forward of the same model.  Every (clip, bin) sequence is its own gLN group and passes through its own eight
blocks whichever chunk it is in, and the packer reads the same whole-clip front-end outputs, so only the order of the fp64 gLN
atomics (and of the full-band TCN's) can differ between two forwards.  The bar is rel-L2 <= 1e-5, the one of the TCN sub-batch
tests; each case prints whether the outputs came out bit-identical.
"""
import time

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CHUNK_TOL = 1e-5
MASK_TOL = 1e-3
PER_CHUNK_LAUNCHES = 25                                          # one pack + eight blocks of three launches


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _load(cfg, params, monkeypatch, chunk=None, cap_gb=None, cls=None, **kw):
    """A model whose C handle was created with FSN_SB_CHUNK / FSN_WS_CAP_GB as given (the knobs are read once, at create)."""
    from fsnplus_b200.model import FullSubNet_Plus
    cls = cls or FullSubNet_Plus
    for k, v in (("FSN_SB_CHUNK", chunk), ("FSN_WS_CAP_GB", cap_gb)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    monkeypatch.delenv("FSN_SB_CHUNK", raising=False)
    monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
    return m


def _small(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, sequence_model="TCN")
    c.update(over)
    return c


def _tcn(**over):
    return dict(O.default_plus_config(), sequence_model="TCN", **over)


def _spectra(B, F, n_samples, seed=0):
    n_fft = 2 * (F - 1)
    X = O.stft(O.synth_clips(B, num_samples=n_samples, seed0=seed), n_fft, n_fft // 2, n_fft)
    return tuple(a[:, None].astype(np.float32) for a in (np.abs(X), X.real, X.imag))


def _forward(m, ins, enhance=False, frames=None):
    with torch.no_grad():
        x = [_t(a) for a in ins]
        return (m.enhance_spectrum(*x, frames=frames) if enhance else m(*x, frames=frames)).cpu()


def _compare(got, want, label):
    eq = torch.equal(got, want)
    d = torch.view_as_real(got) - torch.view_as_real(want) if got.is_complex() else got - want
    w = torch.view_as_real(want) if want.is_complex() else want
    rel = float(d.double().norm() / max(float(w.double().norm()), 1e-30))
    print(f"\n[{label}] chunked == unchunked: {eq} (rel-L2 {rel:.2e})")
    assert torch.isfinite(torch.view_as_real(got) if got.is_complex() else got).all()
    assert rel <= CHUNK_TOL, (label, rel)


VARIANTS = {
    "offline_laplace_norm": {},
    "cumulative_laplace_norm": dict(norm_type="cumulative_laplace_norm"),
    "offline_gaussian_norm": dict(norm_type="offline_gaussian_norm"),
    "cumulative_layer_norm": dict(norm_type="cumulative_layer_norm"),
    "fb_num_neighbors_1": dict(fb_num_neighbors=1),
    "ECA_subband_num_2": dict(channel_attention_model="ECA", subband_num=2),
    "Tanh": dict(sb_output_activate_function="Tanh"),
    "ReLU": dict(sb_output_activate_function="ReLU"),
}


@pytest.mark.parametrize("name", list(VARIANTS))
def test_forced_chunks_small(built_lib, monkeypatch, name):
    """Chunks of 1, 7, 16 and 100 bins (F = 33: 33 one-bin chunks, 7 + 7 + 7 + 7 + 5, 16 + 16 + 1, unchunked), mask and enhanced
    spectrum, against the unchunked forward; the launch count grows by one pack and eight blocks per extra chunk."""
    cfg = _small(**VARIANTS[name])
    params = S.make_params(cfg, seed=40)
    if name in ("Tanh", "ReLU"):
        params["sb_model.fc_output_layer.weight"] = params["sb_model.fc_output_layer.weight"] * 4.0
        params["sb_model.fc_output_layer.bias"] = np.array([-1.0, 0.3], np.float32)
    ins = _spectra(2, 33, 3000, seed=41)
    base = _load(cfg, params, monkeypatch)
    want = {e: _forward(base, ins, e) for e in (False, True)}
    n0 = base.last_launch_count()
    assert base.last_plan_bins() == (2, 0, 0)
    for fc in (1, 7, 16, 100):
        m = _load(cfg, params, monkeypatch, chunk=fc)
        for e in (False, True):
            got = _forward(m, ins, e)
            assert m.last_plan_bins() == (2, 0, fc if fc < 33 else 0)
            nch = -(-33 // fc)
            assert m.last_launch_count() == n0 + (nch - 1) * PER_CHUNK_LAUNCHES
            _compare(got, want[e], f"{name} chunk {fc} {'enh' if e else 'mask'}")


def test_default_geometry_last_chunk_one_bin(built_lib, monkeypatch):
    """One 20 s clip at F = 257 in chunks of 64 bins: 4 x 64 + 1, the last chunk one bin wide."""
    cfg = _tcn()
    params = S.make_params(cfg, seed=42)
    ins = _spectra(1, 257, 20 * 16000, seed=43)
    want = {e: _forward(_load(cfg, params, monkeypatch), ins, e) for e in (False, True)}
    m = _load(cfg, params, monkeypatch, chunk=64)
    for e in (False, True):
        got = _forward(m, ins, e)
        assert m.last_plan_bins() == (1, 0, 64)
        _compare(got, want[e], f"default 20 s chunk 64 {'enh' if e else 'mask'}")


def test_ragged_batch_chunks(built_lib, monkeypatch):
    cfg = _small()
    params = S.make_params(cfg, seed=44)
    mag, real, imag = _spectra(3, 33, 3000, seed=45)
    frames = [mag.shape[-1], 70, 33]
    for a in (mag, real, imag):
        for b, n in enumerate(frames):
            a[b, :, :, n:] = 0.0
    base = _load(cfg, params, monkeypatch)
    m = _load(cfg, params, monkeypatch, chunk=10)
    for e in (False, True):
        want = _forward(base, (mag, real, imag), e, frames)
        got = _forward(m, (mag, real, imag), e, frames)
        assert m.last_plan_bins()[2] == 10
        for b, n in enumerate(frames):
            tail = got[b, ..., n:]
            assert torch.equal(tail, torch.zeros_like(tail))
        _compare(got, want, f"ragged chunk 10 {'enh' if e else 'mask'}")


@pytest.mark.parametrize("B,seconds,cap_gb", [(1, 90, 2), (3, 60, 0.4)])
def test_cap_triggered_chunks(built_lib, monkeypatch, B, seconds, cap_gb):
    """FSN_WS_CAP_GB=2: a 90 s clip is chunked; at 0.4 three 60 s clips are also split into sub-batches.  Same results as the default
    cap's unchunked forward, and the workspace stays within the cap."""
    cfg = _tcn()
    params = S.make_params(cfg, seed=46)
    ins = _spectra(B, 257, seconds * 16000, seed=47)
    base = _load(cfg, params, monkeypatch)
    want = _forward(base, ins, True)
    assert base.last_plan_bins() == (B, 0, 0)
    del base
    torch.cuda.empty_cache()
    m = _load(cfg, params, monkeypatch, cap_gb=cap_gb)
    got = _forward(m, ins, True)
    bs, tw, fc = m.last_plan_bins()
    print(f"\n[cap {cap_gb} GB, {B} x {seconds} s] plan Bs={bs} Fc={fc}, workspace {m.workspace_bytes() / 1e9:.2f} GB")
    assert tw == 0 and fc > 0 and m.workspace_bytes() <= cap_gb * 1e9
    if B > 1:
        assert bs < B
    _compare(got, want, f"cap {cap_gb} GB {B} x {seconds} s")


def test_30s_chunked_parity_vs_torch_port(built_lib, monkeypatch):
    cfg = _tcn()
    params = S.make_params(cfg, seed=0)
    mag, real, imag = _spectra(1, 257, 30 * 16000, seed=48)
    ref = S.TcnPort(params, cfg).forward(*(torch.from_numpy(x) for x in (mag, real, imag))).numpy()
    m = _load(cfg, params, monkeypatch, chunk=40)
    out = _forward(m, (mag, real, imag)).numpy()
    assert m.last_plan_bins()[2] == 40
    err = O.rel_l2(out, ref)
    print(f"\n[sub-band TCN 30 s, chunks of 40 bins] cIRM rel-L2 vs fp32 torch port {err:.3e}")
    assert err < MASK_TOL


def test_one_hour_clip_default_cap(built_lib, monkeypatch):
    from fsnplus_b200 import inference as H
    cfg = _tcn()
    m = _load(cfg, S.make_params(cfg, seed=49), monkeypatch)
    n = 3600 * 16000
    noisy = (torch.randn(1, n, generator=torch.Generator().manual_seed(0)) * 0.05).to(DEV)
    with torch.no_grad():
        H.enhance_batch(m, noisy[:, :16000 * 5])                   # warm-up (allocations of a small geometry)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        y = H.enhance_batch(m, noisy)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    bs, tw, fc = m.last_plan_bins()
    print(f"\n[60 min clip, sub-band TCN] {dt:.1f} s wall, RTF {dt / 3600:.2e}, plan Bs={bs} Fc={fc}, "
          f"workspace {m.workspace_bytes() / 1e9:.2f} GB")
    assert y.shape == noisy.shape and torch.isfinite(y).all()
    assert fc > 0 and m.workspace_bytes() <= 24e9


def test_chunked_forward_gives_back_stale_workspace(built_lib, monkeypatch):
    """At FSN_WS_CAP_GB=2: a model that ran a wide unchunked batch and a longer chunked clip holds at most the cap after each forward,
    a shorter chunked clip included, and model.plan_bins() is the plan it used."""
    cfg = _tcn()
    m = _load(cfg, S.make_params(cfg, seed=50), monkeypatch, cap_gb=2)
    sizes = []
    for B, seconds in ((4, 6), (1, 150), (1, 90)):
        ins = _spectra(B, 257, seconds * 16000, seed=51)
        plan = m.plan_bins(B, ins[0].shape[-1])
        out = _forward(m, ins, True)
        assert torch.isfinite(torch.view_as_real(out)).all()
        assert plan[:3] == m.last_plan_bins() and m.workspace_bytes() <= plan[3]
        sizes.append((B, seconds, m.last_plan_bins(), m.workspace_bytes()))
    print("\n[stale workspace, cap 2 GB] " + ", ".join(f"{b} x {s} s plan {p}: {w / 1e9:.2f} GB" for b, s, p, w in sizes))
    assert sizes[0][2][2] == 0 and sizes[1][2][2] > 0 and sizes[2][2][2] > 0
    assert all(w <= 2e9 for *_, w in sizes)


def test_unchanged_paths(built_lib, monkeypatch):
    """The pipelined entry points run unchunked under FSN_SB_CHUNK; get_stage("sb_in") refuses after a chunked forward and works after
    an unchunked one; an LSTM model ignores the knob (fullsubnet.Model: no atomics anywhere, so its forwards must be bit-identical)."""
    cfg = _small()
    params = S.make_params(cfg, seed=52)
    ins = _spectra(2, 33, 3000, seed=53)
    want = _forward(_load(cfg, params, monkeypatch), ins)
    m = _load(cfg, params, monkeypatch, chunk=7)
    with torch.no_grad():
        x = [_t(a) for a in ins]
        out = m.submit(*x)
        m.wait()
        got = out.cpu()
        n_plain = m.last_launch_count()
    _compare(got, want, "submit under FSN_SB_CHUNK=7")
    host = m.forward_host(*(torch.from_numpy(np.ascontiguousarray(a)).pin_memory() for a in ins), pipelined=True)
    m.sync_host()
    _compare(host, want, "forward_host(pipelined=True) under FSN_SB_CHUNK=7")
    B, F, T = 2, 33, ins[0].shape[-1] + cfg["look_ahead"]
    shape = (B, F, 10, T)
    sb_in = m.get_stage("sb_in", shape, DEV)                        # the last forward ran unchunked
    assert torch.isfinite(sb_in).all()
    _compare(_forward(m, ins), want, "plain forward under FSN_SB_CHUNK=7")
    assert m.last_plan_bins()[2] == 7 and m.last_launch_count() == n_plain + (5 - 1) * PER_CHUNK_LAUNCHES
    from fsnplus_b200 import _lib
    with pytest.raises(_lib.FsnError, match="chunked"):
        m.get_stage("sb_in", shape, DEV)
    from fsnplus_b200.model import Model
    lcfg = O.default_fsn_config()
    lparams = O.make_params_fsn(lcfg, seed=54)
    mag = _t(_spectra(2, 257, 8000, seed=55)[0])
    with torch.no_grad():
        a = _load(lcfg, lparams, monkeypatch, cls=Model)(mag).cpu()
        lm = _load(lcfg, lparams, monkeypatch, chunk=7, cls=Model)
        b = lm(mag).cpu()
    print(f"\n[LSTM under FSN_SB_CHUNK=7] bit-identical: {torch.equal(a, b)}")
    assert torch.equal(a, b) and lm.last_plan_bins() == (2, 0, 0)
