"""Long clips on the GPU: the sub-band LSTM in time windows (DESIGN.md §3.7).

Truth is the unwindowed forward of the same model.  The carried h (fp16) and c (fp32) have the precision of the in-kernel state,
and neither the packed images nor the input-projection GEMM rows depend on where a window starts, so a windowed forward is
predicted to be bit-identical.  fullsubnet.Model must be (torch.equal).  For FullSubNet+ the full-band TCN's fp64 atomic gLN sums
may reorder between any two forwards, so the bar is rel-L2 <= 1e-5 and each case prints whether the outputs were equal.
"""
import time

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WIN_TOL = 1e-5
MASK_TOL = 1e-3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _load(cls, cfg, params, monkeypatch, window=None, cap_gb=None, **kw):
    """A model whose C handle was created with FSN_SB_WINDOW / FSN_WS_CAP_GB as given (the knobs are read once, at create)."""
    for k, v in (("FSN_SB_WINDOW", window), ("FSN_WS_CAP_GB", cap_gb)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    monkeypatch.delenv("FSN_SB_WINDOW", raising=False)
    monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
    return m


def _small(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    c.update(over)
    return c


def _spectra(B, F, n_samples, seed=0):
    n_fft = 2 * (F - 1)
    X = O.stft(O.synth_clips(B, num_samples=n_samples, seed0=seed), n_fft, n_fft // 2, n_fft)
    return tuple(a[:, None].astype(np.float32) for a in (np.abs(X), X.real, X.imag))


def _forward(m, ins, plus, enhance=False, frames=None):
    with torch.no_grad():
        x = [_t(a) for a in ins]
        if enhance:
            return m.enhance_spectrum(*x, frames=frames).cpu()
        return (m(*x, frames=frames) if plus else m(x[0], frames=frames)).cpu()


def _compare(got, want, label, exact):
    eq = torch.equal(got, want)
    d = torch.view_as_real(got) - torch.view_as_real(want) if got.is_complex() else got - want
    w = torch.view_as_real(want) if want.is_complex() else want
    rel = float(d.double().norm() / max(float(w.double().norm()), 1e-30))
    print(f"\n[{label}] windowed == unwindowed: {eq} (rel-L2 {rel:.2e})")
    assert torch.isfinite(torch.view_as_real(got) if got.is_complex() else got).all()
    assert eq if exact else rel <= WIN_TOL, (label, rel)


def _check_windows(cls, cfg, params, ins, monkeypatch, plus=True, windows=(32, 64, 96), frames=None, label="", **kw):
    base = _load(cls, cfg, params, monkeypatch, **kw)
    outs = {e: _forward(base, ins, plus, e, frames) for e in ((False, True) if plus else (False,))}
    assert base.last_plan()[1] == 0
    T = ins[0].shape[-1] + cfg["look_ahead"]
    assert any(T % w for w in windows), "at least one window must leave a partial last window"
    for w in windows:
        m = _load(cls, cfg, params, monkeypatch, window=w, **kw)
        for e, want in outs.items():
            got = _forward(m, ins, plus, e, frames)
            assert m.last_plan()[1] == w
            _compare(got, want, f"{label} window {w} {'enh' if e else 'mask'}", exact=not plus)


def test_default_geometry_windows(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=1)
    ins = _spectra(2, 257, 48000, seed=3)                       # B = 2, 3 s, T = 188
    _check_windows(FullSubNet_Plus, cfg, params, ins, monkeypatch, label="default")


@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm", "offline_gaussian_norm", "cumulative_layer_norm"])
def test_small_norm_types_windows(built_lib, monkeypatch, norm):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small(norm_type=norm)
    _check_windows(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=2), _spectra(2, 33, 3000, seed=5), monkeypatch, label=norm)


@pytest.mark.parametrize("variant", ["GRU", "layers1", "layers3", "hidden512", "lstm_x3"])
def test_small_variants_windows(built_lib, monkeypatch, variant):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg, kw, nl, scale = _small(), {}, 2, 1.0
    if variant == "GRU":
        cfg["sequence_model"] = "GRU"
    elif variant == "hidden512":
        cfg["sb_model_hidden_size"] = 512
    elif variant == "lstm_x3":
        scale = 3.0
    else:
        nl = 1 if variant == "layers1" else 3
        kw["num_layers"] = nl
    params = O.make_params_plus(cfg, seed=4, lstm_scale=scale, num_layers=nl)
    _check_windows(FullSubNet_Plus, cfg, params, _spectra(2, 33, 3000, seed=6), monkeypatch, label=variant, **kw)


@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm"])
def test_fullsubnet_model_windows_bit_identical(built_lib, monkeypatch, norm):
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    cfg["norm_type"] = norm
    ins = _spectra(2, 257, 40000, seed=7)
    _check_windows(Model, cfg, O.make_params_fsn(cfg, seed=8), ins, monkeypatch, plus=False, label=f"fullsubnet.Model {norm}")


def test_ragged_batch_windows(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small()
    mag, real, imag = _spectra(3, 33, 3000, seed=9)
    frames = [mag.shape[-1], 70, 33]
    for a in (mag, real, imag):
        for b, n in enumerate(frames):
            a[b, :, :, n:] = 0.0
    _check_windows(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=10), (mag, real, imag), monkeypatch, frames=frames, label="ragged")


@pytest.mark.parametrize("B,seconds,cap_gb", [(1, 90, 2), (3, 60, 0.4)])
def test_cap_triggered_windows(built_lib, monkeypatch, B, seconds, cap_gb):
    """FSN_WS_CAP_GB=2: a 90 s clip is windowed; at 0.4 three 60 s clips are also split into sub-batches.  Same results as the default
    cap's unwindowed forward, and the workspace stays within the cap."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=11)
    ins = _spectra(B, 257, seconds * 16000, seed=12)
    base = _load(FullSubNet_Plus, cfg, params, monkeypatch)
    want = _forward(base, ins, True, True)
    assert base.last_plan() == (B, 0)
    del base
    torch.cuda.empty_cache()
    m = _load(FullSubNet_Plus, cfg, params, monkeypatch, cap_gb=cap_gb)
    got = _forward(m, ins, True, True)
    bs, tw = m.last_plan()
    print(f"\n[cap {cap_gb} GB, {B} x {seconds} s] plan Bs={bs} Tw={tw}, workspace {m.workspace_bytes() / 1e9:.2f} GB")
    assert tw > 0 and tw % 32 == 0 and m.workspace_bytes() <= cap_gb * 1e9
    if B > 1:
        assert bs < B
    _compare(got, want, f"cap {cap_gb} GB {B} x {seconds} s", exact=False)


def test_60s_windowed_parity_vs_torch_port(built_lib, monkeypatch):
    from oracle.torch_port import TorchPort
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=0)
    mag, real, imag = _spectra(1, 257, 60 * 16000, seed=13)
    ref = TorchPort(params, cfg, "plus", dtype=torch.float32).forward(*(torch.from_numpy(x) for x in (mag, real, imag))).numpy()
    m = _load(FullSubNet_Plus, cfg, params, monkeypatch, window=2048)
    out = _forward(m, (mag, real, imag), True).numpy()
    assert m.last_plan()[1] == 2048
    err = O.rel_l2(out, ref)
    print(f"\n[FullSubNet+ 60 s, windows of 2048] cIRM rel-L2 vs fp32 torch port {err:.3e}")
    assert err < MASK_TOL


def test_one_hour_clip_default_cap(built_lib, monkeypatch):
    from fsnplus_b200 import inference as H
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    m = _load(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=14), monkeypatch)
    n = 3600 * 16000
    noisy = (torch.randn(1, n, generator=torch.Generator().manual_seed(0)) * 0.05).to(DEV)
    with torch.no_grad():
        H.enhance_batch(m, noisy[:, :16000 * 5])                   # warm-up (allocations of a small geometry)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        y = H.enhance_batch(m, noisy)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
    bs, tw = m.last_plan()
    print(f"\n[60 min clip] {dt:.1f} s wall, RTF {dt / 3600:.2e}, plan Bs={bs} Tw={tw}, workspace {m.workspace_bytes() / 1e9:.2f} GB")
    assert y.shape == noisy.shape and torch.isfinite(y).all()
    assert tw > 0 and m.workspace_bytes() <= 24e9


def test_unchanged_paths_report_no_window(built_lib, monkeypatch):
    """The sub-band TCN and lstm_impl="mma" have no windowed form: even with FSN_SB_WINDOW they run unwindowed."""
    import sbtcn_oracle as S
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small(sequence_model="TCN")
    m = _load(FullSubNet_Plus, cfg, S.make_params(cfg, seed=1), monkeypatch, window=32)
    _forward(m, _spectra(1, 33, 3000), True)
    assert m.last_plan() == (1, 0)
    cfg = _small()
    m = _load(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=1), monkeypatch, window=32, lstm_impl="mma")
    _forward(m, _spectra(1, 33, 3000), True)
    assert m.last_plan() == (1, 0) and m.last_lstm_impl() == "mma"


def test_windowed_forward_gives_back_stale_workspace(built_lib, monkeypatch):
    """At FSN_WS_CAP_GB=2: a model that ran a wide unwindowed batch and a longer windowed clip holds at most the cap after a
    shorter windowed clip too (every grow-only buffer an earlier forward left larger is given back)."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    m = _load(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=15), monkeypatch, cap_gb=2)
    sizes = []
    for B, seconds in ((4, 6), (1, 150), (1, 90)):
        out = _forward(m, _spectra(B, 257, seconds * 16000, seed=16), True, True)
        assert torch.isfinite(torch.view_as_real(out)).all()
        sizes.append((B, seconds, m.last_plan(), m.workspace_bytes()))
    print("\n[stale workspace, cap 2 GB] " + ", ".join(f"{b} x {s} s plan {p}: {w / 1e9:.2f} GB" for b, s, p, w in sizes))
    assert sizes[0][2][1] == 0 and sizes[1][2][1] > 0 and sizes[2][2][1] > 0
    assert all(w <= 2e9 for *_, w in sizes)


def test_release_workspace_and_model_plan(built_lib, monkeypatch):
    """release_workspace() frees every forward workspace and the next forward is unchanged; model.plan() is the plan the handle uses,
    with the knobs it read at creation (a later environment change, or FSN_LSTM_IMPL, does not make them disagree)."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=17)
    ins = _spectra(1, 257, 90 * 16000, seed=18)
    m = _load(FullSubNet_Plus, cfg, params, monkeypatch, cap_gb=2)
    T = ins[0].shape[-1]
    monkeypatch.setenv("FSN_WS_CAP_GB", "50")                       # read at creation only: must not change the model's plan
    plan = m.plan(1, T)
    a = _forward(m, ins, True, True)
    assert plan[:2] == m.last_plan() and plan[1] > 0 and m.workspace_bytes() <= plan[2] <= 2e9
    m.release_workspace()
    assert m.workspace_bytes() == 0
    b = _forward(m, ins, True, True)
    _compare(b, a, "after release_workspace", exact=False)
    monkeypatch.delenv("FSN_WS_CAP_GB")
    monkeypatch.setenv("FSN_LSTM_IMPL", "1")                        # mma: no windows, and the plan says so
    mm = _load(FullSubNet_Plus, cfg, params, monkeypatch, cap_gb=2)
    monkeypatch.delenv("FSN_LSTM_IMPL")
    assert mm.plan(1, T)[1] == 0
    _forward(mm, ins, True)
    assert mm.last_plan()[1] == 0 and mm.last_lstm_impl() == "mma"
