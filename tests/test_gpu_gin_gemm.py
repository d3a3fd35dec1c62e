"""The sub-band LSTM's input-projection GEMM on 128 x 256 tiles shared by a CTA pair (gemm_f16_pair_kernel, DESIGN.md §3.3)
against the 128 x 128 kernel it replaces.

Both run the same k order (64-wide k-blocks, four 16-wide wgmma steps, fp32 accumulation) and round once to fp16, so their
outputs must be bit-identical: the GEMM alone at the shapes the layer-wise path runs it with, and whole forwards with
FSN_GIN_GEMM=128 (the old kernel) against the default.  fullsubnet.Model is deterministic and must be torch.equal.  FullSubNet+'s
full-band TCN sums its gLN statistics with fp64 atomics whose order may change between any two forwards, so there a difference is
accepted only if the old kernel's own second forward differs from its first as well, and then by rel-L2 <= 1e-5.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

DEV = "cuda:0"


def _tile_n(lib, M, N, K, tile_n=0):
    return int(lib.fsn_gemm_f16_tile_n(M, N, K, tile_n))


# ---------------------------------------------------------------------------------------------------------------------
# dispatch (host only)
# ---------------------------------------------------------------------------------------------------------------------
def test_dispatch_table(built_lib):
    lib = built_lib
    assert _tile_n(lib, 130 * 190 * 128, 1536, 384) == 256           # config #2, layer 1
    assert _tile_n(lib, 130 * 96 * 128, 2048, 512) == 256            # config #5, layers 1 and 2
    assert _tile_n(lib, 2 * 128 * 32, 1536, 384) == 256              # one tile pair, a 32-frame window
    assert _tile_n(lib, 130 * 190 * 128, 1536, 384, 128) == 128      # FSN_GIN_GEMM=128
    assert _tile_n(lib, 130 * 190 * 128, 1536, 384, 256) == 256
    assert _tile_n(lib, 33 * 128, 1536, 384) == 128                  # odd number of 128-row tiles: no pairs
    assert _tile_n(lib, 32 * 128, 1152, 384) == 128                  # N not a multiple of 256
    assert _tile_n(lib, 100, 1536, 384) == -1                        # M not a multiple of 128


# ---------------------------------------------------------------------------------------------------------------------
# the GEMM alone
# ---------------------------------------------------------------------------------------------------------------------
def _gemm(lib, A, B, tile_n):
    M, K = A.shape
    N = B.shape[0]
    Cm = torch.empty(M, N, device=DEV, dtype=torch.half)
    rc = lib.fsn_gemm_f16(C.c_void_p(A.data_ptr()), C.c_void_p(B.data_ptr()), C.c_void_p(Cm.data_ptr()), M, N, K, tile_n,
                          C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream))
    assert rc == 0, lib.fsn_last_error().decode()
    torch.cuda.synchronize()
    return Cm


def _operands(M, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = (torch.randn(M, K, device=DEV, generator=g) * 0.5).half()
    B = (torch.randn(N, K, device=DEV, generator=g) * (1.0 / K ** 0.5)).half()
    return A, B


def _check_vs_fp32(A, B, Cm, seed):
    """Rows sampled from the start, the end and at random, against an fp32 matmul of the same fp16 operands: the kernel's only
    rounding is the final one to fp16."""
    M = A.shape[0]
    g = torch.Generator(device=DEV).manual_seed(seed)
    idx = torch.cat([torch.arange(0, min(256, M), device=DEV), torch.arange(max(M - 256, 0), M, device=DEV),
                     torch.randint(0, M, (1024,), device=DEV, generator=g)])
    ref = A[idx].float() @ B.float().T
    got = Cm[idx].float()
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    assert bool((err <= 1e-3 + 1e-3 * ref.abs()).all()), float(err.max())


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(130 * 190 * 128, 1536, 384),      # config #2's layer-1 projection
                                   (130 * 96 * 128, 2048, 512),       # config #5's
                                   (2 * 128 * 32, 1536, 384)],        # one tile pair of a 32-frame window
                         ids=["config2", "config5", "window32"])
def test_gemm_pair_tiles_bit_identical(built_lib, M, N, K):
    lib = built_lib
    assert _tile_n(lib, M, N, K) == 256
    A, B = _operands(M, N, K, seed=M % 1000 + N)
    new = _gemm(lib, A, B, 0)
    old = _gemm(lib, A, B, 128)
    same = torch.equal(new, old)
    if not same:
        d = (new.float() - old.float()).abs()
        pytest.fail(f"128 x 256 differs from 128 x 128 in {int((d > 0).sum())} of {new.numel()} elements (max {float(d.max()):.3e})")
    _check_vs_fp32(A, B, new, seed=3)


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K", [(33 * 128, 1536, 384), (32 * 128, 1152, 384), (2 * 128, 1536, 64)], ids=["odd_tiles", "n1152", "k64"])
def test_gemm_other_shapes(built_lib, M, N, K):
    """Shapes without tile pairs run the 128 x 128 kernel; the smallest pair shape (one pair, one k-block) runs the new one."""
    lib = built_lib
    A, B = _operands(M, N, K, seed=11)
    got = _gemm(lib, A, B, 0)
    _check_vs_fp32(A, B, got, seed=5)
    assert torch.equal(got, _gemm(lib, A, B, 128))


# ---------------------------------------------------------------------------------------------------------------------
# whole forwards, FSN_GIN_GEMM=128 against the default
# ---------------------------------------------------------------------------------------------------------------------
def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _load(cls, cfg, params, monkeypatch, gin=None, window=None, **kw):
    """A model whose C handle was created with FSN_GIN_GEMM / FSN_SB_WINDOW as given (both are read once, at create)."""
    for k, v in (("FSN_GIN_GEMM", gin), ("FSN_SB_WINDOW", window)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    monkeypatch.delenv("FSN_GIN_GEMM", raising=False)
    monkeypatch.delenv("FSN_SB_WINDOW", raising=False)
    return m


def _spectra(B, F, n_samples, seed):
    n_fft = 2 * (F - 1)
    X = O.stft(O.synth_clips(B, num_samples=n_samples, seed0=seed), n_fft, n_fft // 2, n_fft)
    return tuple(a[:, None].astype(np.float32) for a in (np.abs(X), X.real, X.imag))


def _run(m, ins, plus, enhance, frames):
    with torch.no_grad():
        x = [_t(a) for a in ins]
        if enhance:
            return m.enhance_spectrum(*x, frames=frames).cpu()
        return (m(*x, frames=frames) if plus else m(x[0], frames=frames)).cpu()


def _rel(a, b):
    a = torch.view_as_real(a) if a.is_complex() else a
    b = torch.view_as_real(b) if b.is_complex() else b
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-30))


def _check_knob(cls, cfg, params, ins, monkeypatch, plus=True, frames=None, window=None, label="", **kw):
    old = _load(cls, cfg, params, monkeypatch, gin=128, window=window, **kw)
    new = _load(cls, cfg, params, monkeypatch, gin=None, window=window, **kw)
    for enhance in ((False, True) if plus else (False,)):
        want = _run(old, ins, plus, enhance, frames)
        got = _run(new, ins, plus, enhance, frames)
        eq = torch.equal(got, want)
        tag = f"{label} {'enh' if enhance else 'mask'}"
        print(f"\n[{tag}] 128 x 256 == 128 x 128: {eq} (rel-L2 {_rel(got, want):.2e})")
        assert torch.isfinite(torch.view_as_real(got) if got.is_complex() else got).all()
        if eq:
            continue
        assert plus, f"{tag}: fullsubnet.Model is deterministic, the outputs must be equal"
        again = _run(old, ins, plus, enhance, frames)
        assert not torch.equal(again, want), f"{tag}: the old kernel repeats its own result exactly, the new one differs"
        assert _rel(got, want) <= 1e-5, tag
    if window:
        assert new.last_plan()[1] == window and old.last_plan()[1] == window


@pytest.mark.gpu
def test_default_config_b64(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    _check_knob(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=1), _spectra(64, 257, 48000, seed=3), monkeypatch, label="default B=64")


@pytest.mark.gpu
def test_config5_geometry(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    cfg.update(num_freqs=513, sb_model_hidden_size=512, fb_model_hidden_size=512)
    params = O.make_params_plus(cfg, seed=2, num_layers=3)
    _check_knob(FullSubNet_Plus, cfg, params, _spectra(8, 513, 48000, seed=4), monkeypatch, label="config5", num_layers=3)


@pytest.mark.gpu
def test_gru(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    cfg["sequence_model"] = "GRU"
    _check_knob(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=5), _spectra(4, 257, 48000, seed=6), monkeypatch, label="GRU")


@pytest.mark.gpu
def test_windowed_long_clip(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    _check_knob(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=7), _spectra(1, 257, 16000 * 12, seed=8), monkeypatch,
                window=96, label="window 96")


@pytest.mark.gpu
def test_ragged_batch(built_lib, monkeypatch):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    ins = _spectra(6, 257, 48000, seed=9)
    T = ins[0].shape[-1]
    frames = [T, T - 40, 33, T - 1, 90, 64]
    for a in ins:
        for b, n in enumerate(frames):
            a[b, :, :, n:] = 0.0
    _check_knob(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=10), ins, monkeypatch, frames=frames, label="ragged")


@pytest.mark.gpu
def test_fullsubnet_model_exact(built_lib, monkeypatch):
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    _check_knob(Model, cfg, O.make_params_fsn(cfg, seed=12), _spectra(8, 257, 48000, seed=13), monkeypatch, plus=False, label="Model")
