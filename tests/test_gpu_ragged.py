"""Ragged batches on the GPU (fsn_model_forward_ragged / fsn_model_forward_enhance_ragged, ``frames=`` of the Python forward).

Truth is the existing forward of each clip alone: clip b of a ragged batch must match it on its first frames[b] frames and be exactly
zero after, whatever the batch holds there.  Rows are independent in every kernel, so only the order of the fp64 atomic sums of the
gLN statistics differs: the bar is rel-L2 <= 1e-5 (a prediction from the code).  Against the fp64 oracle the project bar, cIRM
rel-L2 <= 1e-3, applies.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CLIP_TOL = 1e-5
MASK_TOL = 1e-3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _load(cls, cfg, params, **kw):
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))         # the C handle reads the FSN_* knobs once, here
    return m


def _plus(cfg, params=None, seed=3, **kw):
    from fsnplus_b200.model import FullSubNet_Plus
    if params is None:
        params = S.make_params(cfg, seed=seed) if cfg.get("sequence_model") == "TCN" else O.make_params_plus(cfg, seed=seed)
    return _load(FullSubNet_Plus, cfg, params, **kw)


def _fsn(cfg, seed=3, **kw):
    from fsnplus_b200.model import Model
    return _load(Model, cfg, O.make_params_fsn(cfg, seed=seed), **kw)


def _small(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    c.update(over)
    return c


def _batch(lengths, F, seed=0, poison=False):
    """Spectra of distinct clips (centred STFT of synthetic audio), scattered into a zero [B, 1, F, T_max] batch.  Returns the
    batch, the frame counts and the per-clip planes.  poison: NaN at every t >= frames[b] instead of zeros."""
    n_fft = 2 * (F - 1)
    hop = n_fft // 2
    clips, frames = [], []
    for i, n in enumerate(lengths):
        X = O.stft(O.synth_clips(1, num_samples=n, seed0=seed + 37 * i), n_fft, hop, n_fft)
        clips.append(X[0])
        frames.append(X.shape[-1])
    T = max(frames)
    fill = np.nan if poison else 0.0
    mag, real, imag = (np.full((len(lengths), 1, F, T), fill, np.float32) for _ in range(3))
    for b, X in enumerate(clips):
        n = frames[b]
        mag[b, 0, :, :n], real[b, 0, :, :n], imag[b, 0, :, :n] = np.abs(X), X.real, X.imag
    return (mag, real, imag), frames


def _run(m, ins, frames=None, enhance=False, plus=True):
    with torch.no_grad():
        x = [_t(a) if a is not None else None for a in ins]
        if enhance:
            return m.enhance_spectrum(*x, frames=frames)
        return m(*x, frames=frames) if plus else m(x[0], frames=frames)


def _check_per_clip(m, ins, frames, plus=True, label=""):
    """Mask and enhanced spectrum of the ragged batch against each clip's own forward; exact zeros past each clip."""
    worst = 0.0
    for enhance in ((False, True) if ins[1] is not None else (False,)):
        out = _run(m, ins, frames, enhance, plus).cpu()
        assert not torch.isnan(out).any()
        for b, n in enumerate(frames):
            one = [a[b:b + 1, :, :, :n] if a is not None else None for a in ins]
            want = _run(m, one, None, enhance, plus).cpu()
            got = out[b:b + 1, ..., :n]
            err = O.rel_l2(torch.view_as_real(got).numpy() if enhance else got.numpy(),
                           torch.view_as_real(want).numpy() if enhance else want.numpy())
            worst = max(worst, err)
            assert err <= CLIP_TOL, (label, enhance, b, n, err)
            assert (out[b, ..., n:] == 0).all(), (label, enhance, b)
    print(f"\n[ragged vs per clip] {label}: worst rel-L2 {worst:.2e}")
    return worst


def test_equal_lengths_take_the_unmasked_path(built_lib):
    """frames = [T] * B and frames = None are bit-identical to the plain entry points, with the same launch count."""
    cfg = O.default_plus_config()
    m = _plus(cfg)
    ins, _ = _batch([16000] * 3, 257, seed=11)
    T = ins[0].shape[-1]
    for enhance in (False, True):
        plain = _run(m, ins, None, enhance)
        n_plain = m.last_launch_count()
        for fr in ([T] * 3, torch.tensor([T] * 3)):
            got = _run(m, ins, fr, enhance)
            assert torch.equal(got, plain) and m.last_launch_count() == n_plain
        lib = built_lib
        fn = lib.fsn_model_forward_enhance_ragged if enhance else lib.fsn_model_forward_ragged
        out = torch.empty_like(plain)
        x = [_t(a) for a in ins]
        stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
        assert fn(m._handle, *(C.c_void_p(a.data_ptr()) for a in x), 3, T, None, C.c_void_p(out.data_ptr()), stream) == 0
        assert torch.equal(out, plain) and m.last_launch_count() == n_plain


def test_default_geometry_ragged_vs_per_clip(built_lib):
    m = _plus(O.default_plus_config())
    ins, frames = _batch([16000, 4000, 9100, 2600, 12345, 16384], 257, seed=3)
    _check_per_clip(m, ins, frames, label="FullSubNet+ default")


SMALL = {
    "laplace": _small(),
    "cumulative_laplace": _small(norm_type="cumulative_laplace_norm"),
    "gaussian": _small(norm_type="offline_gaussian_norm"),
    "cumulative_layer": _small(norm_type="cumulative_layer_norm"),
    "SE": _small(channel_attention_model="SE"),
    "CBAM": _small(channel_attention_model="CBAM"),
    "ECA": _small(channel_attention_model="ECA"),
    "ECA_sub2": _small(channel_attention_model="ECA", subband_num=2),
    "GRU": _small(sequence_model="GRU"),
    "causal_tcn": dict(_small(), causal_tcn=True),
    "sbTCN": _small(sequence_model="TCN", sb_model_hidden_size=32),
}


@pytest.mark.parametrize("name", list(SMALL) + ["mma"])
def test_small_configs_ragged_vs_per_clip(built_lib, name):
    cfg = SMALL.get(name, _small())
    m = _plus(cfg, lstm_impl="mma") if name == "mma" else _plus(cfg)
    ins, frames = _batch([2000, 700, 1500, 2222, 1024], 33, seed=5)
    _check_per_clip(m, ins, frames, label=name)
    if name == "mma":
        assert m.last_lstm_impl() == "mma"


@pytest.mark.parametrize("no_ws", [False, True])
def test_fullsubnet_model_ragged_vs_per_clip(built_lib, monkeypatch, no_ws):
    """fullsubnet.Model: the weight-stationary full-band LSTM, and the mma one (FSN_NO_WS=1); the enhance entry point too."""
    if no_ws:
        monkeypatch.setenv("FSN_NO_WS", "1")
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48)
    m = _fsn(cfg)
    ins, frames = _batch([2000, 700, 1500, 2222], 33, seed=9)
    _check_per_clip(m, (ins[0], None, None), frames, plus=False, label=f"Model no_ws={no_ws}")
    out = _run(m, ins, frames, enhance=True).cpu()                 # the enhance entry point reads the planes for Model too
    for b, n in enumerate(frames):
        want = _run(m, [a[b:b + 1, :, :, :n] for a in ins], None, enhance=True).cpu()
        assert O.rel_l2(torch.view_as_real(out[b:b + 1, :, :n]).numpy(), torch.view_as_real(want).numpy()) <= CLIP_TOL
        assert (out[b, :, n:] == 0).all()


@pytest.mark.parametrize("name", ["default", "gaussian", "sbTCN", "mma", "fsn"])
def test_poison_past_the_end_changes_nothing(built_lib, name):
    """NaN in mag, real and imag at every t >= frames[b]: bit-identical outputs, no NaN, exact zeros past each clip."""
    if name == "fsn":
        cfg = O.default_fsn_config()
        cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48)
        m, F = _fsn(cfg), 33
    elif name == "default":
        m, F = _plus(O.default_plus_config()), 257
    else:
        m, F = (_plus(_small(), lstm_impl="mma") if name == "mma" else _plus(SMALL[name])), 33
    lengths = [6000, 2600, 4100] if F == 257 else [2000, 700, 1500]
    clean, frames = _batch(lengths, F, seed=21)
    dirty, _ = _batch(lengths, F, seed=21, poison=True)
    for enhance in (False, True):
        plus = name != "fsn"
        a = _run(m, clean if plus or enhance else (clean[0], None, None), frames, enhance, plus)
        b = _run(m, dirty if plus or enhance else (dirty[0], None, None), frames, enhance, plus)
        assert not torch.isnan(b).any() and torch.equal(a, b), (name, enhance)
        for i, n in enumerate(frames):
            assert (b[i, ..., n:] == 0).all()


def test_ragged_against_fp64_oracle(built_lib):
    """A ragged small-config batch and a default-config batch of 64 clips of 1-10 s, against the fp64 reference per clip (a subset
    of the 64 for time)."""
    cfg = _small()
    params = O.make_params_plus(cfg, seed=8)
    m = _plus(cfg, params)
    ins, frames = _batch([2000, 700, 1500, 2222, 1024], 33, seed=13)
    out = _run(m, ins, frames).cpu().numpy()
    for b, n in enumerate(frames):
        ref = O.fullsubnet_plus_forward(params, cfg, *(a[b:b + 1, :, :, :n] for a in ins))
        assert O.rel_l2(out[b:b + 1, ..., :n], ref) < MASK_TOL
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=9)
    m = _plus(cfg, params)
    rng = np.random.default_rng(64)
    lengths = [int(x) for x in rng.integers(16000, 160001, 64)]
    ins, frames = _batch(lengths, 257, seed=17)
    out = _run(m, ins, frames).cpu().numpy()
    errs = []
    for b in np.argsort(frames)[:3]:                               # the three shortest clips
        n = frames[b]
        ref = O.fullsubnet_plus_forward(params, cfg, *(a[b:b + 1, :, :, :n] for a in ins))
        errs.append(O.rel_l2(out[b:b + 1, ..., :n], ref))
        assert (out[b, ..., n:] == 0).all()
    print(f"\n[ragged vs fp64] default config, 64 clips, rel-L2 of the 3 shortest: {', '.join(f'{e:.2e}' for e in errs)}")
    assert max(errs) < MASK_TOL


def test_shortest_clip_next_to_full_length(built_lib):
    """The shortest clip the TSSE allows (frames + look_ahead = max(kersize)) and, without TSSE, one frame, next to frames = T."""
    ins, _ = _batch([2000, 2000], 33, seed=30)
    T = ins[0].shape[-1]
    _check_per_clip(_plus(_small()), ins, [10 - 2, T], label="TSSE shortest")
    _check_per_clip(_plus(SMALL["SE"]), ins, [1, T], label="SE one frame")


def test_workspace_cap_split_equals_unsplit(built_lib, monkeypatch):
    """A cap so small that every sample runs as its own sub-batch: the frame counts are sliced with the batch."""
    cfg = _small()
    params = O.make_params_plus(cfg, seed=4)
    ins, frames = _batch([2000, 700, 1500, 2222, 1024], 33, seed=31)
    whole = _run(_plus(cfg, params), ins, frames).cpu().numpy()
    monkeypatch.setenv("FSN_WS_CAP_GB", "1e-6")
    split = _run(_plus(cfg, params), ins, frames).cpu().numpy()
    err = O.rel_l2(split, whole)
    print(f"\n[ragged, split into sub-batches] rel-L2 vs unsplit {err:.2e}")
    assert err <= CLIP_TOL
    for b, n in enumerate(frames):
        assert (split[b, ..., n:] == 0).all()


def test_host_frames_array_reused_between_calls(built_lib):
    """Successive ragged calls that rewrite the SAME host array right after each call returns (no synchronisation in between):
    each result follows its own counts."""
    cfg = _small()
    m = _plus(cfg)
    ins, _ = _batch([2000, 2000, 2000], 33, seed=40)
    T = ins[0].shape[-1]
    x = [_t(a) for a in ins]
    sets = [[T, 8, 12], [9, T, 11], [T - 1, 20, T], [8, 8, 8]]
    h = (C.c_int32 * 3)()
    outs = [torch.empty((3, 2, 33, T), device=DEV) for _ in sets]
    stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    for fr, out in zip(sets, outs):
        for i, n in enumerate(fr):
            h[i] = n
        assert built_lib.fsn_model_forward_ragged(m._handle, *(C.c_void_p(a.data_ptr()) for a in x), 3, T, h,
                                                  C.c_void_p(out.data_ptr()), stream) == 0
    torch.cuda.synchronize()
    for fr, out in zip(sets, outs):
        assert torch.equal(out, _run(m, ins, fr))


def test_invalid_frame_counts(built_lib):
    from fsnplus_b200 import _lib
    m = _plus(_small())
    ins, _ = _batch([2000, 2000], 33, seed=50)
    T = ins[0].shape[-1]
    for fr, word in (([T, 0], "frames[1] = 0"), ([T + 1, T], "frames[0]"), ([T, 7], "TSSE kernel size")):
        with pytest.raises(_lib.FsnError, match=word.replace("[", r"\[").replace("]", r"\]")):
            _run(m, ins, fr)
    _run(_plus(SMALL["SE"]), ins, [T, 1])                          # one frame is fine without TSSE
