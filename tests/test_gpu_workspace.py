"""The forward workspace the model holds is exactly what the plan counts (fsn_model_plan_bins: ws_sizes in fsn_api.cu).

A fresh model that ran one ragged plain forward holds the plan's bytes, on every path that allocates its own buffers: the layer-wise
LSTM, its time windows (with the cumulative norm's running sums), the generic mma kernel, the sub-band TCN whole and in bin chunks, and
fullsubnet.Model's weight-stationary full-band LSTM.  The one buffer the plan leaves out is the generic kernel's scratch mask of the
enhanced-spectrum output.  A model that runs a wide batch and then windowed clips of decreasing length holds exactly each windowed
forward's plan: every buffer an earlier forward left larger is given back.
"""
import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _load(cls, cfg, params, monkeypatch, env=None, **kw):
    """A model whose C handle was created with the FSN_* knobs in env (they are read once, at create)."""
    knobs = ("FSN_SB_WINDOW", "FSN_SB_CHUNK", "FSN_WS_CAP_GB")
    for k in knobs:
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, str(v))
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    for k in knobs:
        monkeypatch.delenv(k, raising=False)
    return m


def _small(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    c.update(over)
    return c


def _spectra(B, F, n_samples, seed=0):
    n_fft = 2 * (F - 1)
    X = O.stft(O.synth_clips(B, num_samples=n_samples, seed0=seed), n_fft, n_fft // 2, n_fft)
    return [_t(a[:, None].astype(np.float32)) for a in (np.abs(X), X.real, X.imag)]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _run(m, ins, frames, enhance=False):
    """ins: (mag, real, imag) for FullSubNet+, (mag,) for fullsubnet.Model."""
    with torch.no_grad():
        out = m.enhance_spectrum(*ins, frames=frames) if enhance else m(*ins, frames=frames)
        torch.cuda.synchronize()
    assert torch.isfinite(torch.view_as_real(out) if out.is_complex() else out).all()
    return out


def _check_fresh(m, ins, label, enhance=False, extra=0):
    B, T = ins[0].shape[0], ins[0].shape[-1]
    frames = [T] * (B - 1) + [T - 5]                                # ragged: the clip lengths buffer exists too
    _run(m, ins, frames, enhance)
    plan = m.plan_bins(B, T)
    held = m.workspace_bytes()
    print(f"\n[{label}] plan {plan[:3]}: {plan[3]} bytes, held {held}")
    assert m.last_plan_bins() == plan[:3]
    assert held == plan[3] + extra, (label, held, plan)


@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm"])
@pytest.mark.parametrize("window", [0, 32])
def test_layerwise_lstm_holds_the_plan(built_lib, monkeypatch, norm, window):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small(norm_type=norm)
    m = _load(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=1), monkeypatch, {"FSN_SB_WINDOW": window} if window else None)
    _check_fresh(m, _spectra(2, 33, 3000, seed=2), f"layer-wise {norm} window {window}")
    assert m.last_lstm_impl() != "mma" and m.last_plan_bins()[1] == window


def test_mma_lstm_holds_the_plan_and_its_scratch_mask(built_lib, monkeypatch):
    """lstm_impl="mma": the mask output holds the plan; the enhanced-spectrum output adds the scratch mask [B, 2, F, T] fp32."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small()
    params = O.make_params_plus(cfg, seed=3)
    ins = _spectra(2, 33, 3000, seed=4)
    m = _load(FullSubNet_Plus, cfg, params, monkeypatch, lstm_impl="mma")
    _check_fresh(m, ins, "mma mask")
    assert m.last_lstm_impl() == "mma"
    m = _load(FullSubNet_Plus, cfg, params, monkeypatch, lstm_impl="mma")
    B, T = ins[0].shape[0], ins[0].shape[-1]
    _check_fresh(m, ins, "mma enhanced spectrum", enhance=True, extra=B * 2 * cfg["num_freqs"] * T * 4)


@pytest.mark.parametrize("chunk", [0, 7])
def test_subband_tcn_holds_the_plan(built_lib, monkeypatch, chunk):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small(sequence_model="TCN")
    m = _load(FullSubNet_Plus, cfg, S.make_params(cfg, seed=5), monkeypatch, {"FSN_SB_CHUNK": chunk} if chunk else None)
    _check_fresh(m, _spectra(2, 33, 3000, seed=6), f"sub-band TCN chunk {chunk}")
    assert m.last_plan_bins()[2] == chunk


def test_fullsubnet_model_holds_the_plan(built_lib, monkeypatch):
    """fullsubnet.Model at B <= 64 runs its full-band LSTM on the weight-stationary kernel, with its h exchange buffer and barrier."""
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    m = _load(Model, cfg, O.make_params_fsn(cfg, seed=7), monkeypatch)
    _check_fresh(m, _spectra(2, 257, 8000, seed=8)[:1], "fullsubnet.Model")


def test_windowed_sequence_holds_each_plan(built_lib, monkeypatch):
    """At FSN_WS_CAP_GB=2: a wide unwindowed batch, then a long and a shorter windowed clip (ragged).  After each windowed forward the
    model holds exactly that forward's plan."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    m = _load(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=9), monkeypatch, {"FSN_WS_CAP_GB": 2})
    for i, (B, seconds) in enumerate(((4, 6), (1, 150), (1, 90))):
        ins = _spectra(B, 257, seconds * 16000, seed=10 + i)
        T = ins[0].shape[-1]
        _run(m, ins, None if i == 0 else [T - 7], enhance=True)
        plan = m.plan_bins(B, T)
        held = m.workspace_bytes()
        print(f"\n[{B} x {seconds} s, cap 2 GB] plan {plan[:3]}: {plan[3] / 1e9:.3f} GB, held {held / 1e9:.3f} GB")
        assert m.last_plan_bins() == plan[:3]
        if i == 0:
            assert plan[1] == 0 and held <= 2e9
        else:
            assert plan[1] > 0 and held == plan[3]
