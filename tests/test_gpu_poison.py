"""No output depends on what its scratch held before the call (DESIGN.md §2, "Scratch that nothing wrote").

A handle created with FSN_POISON=1 fills every scratch buffer that is not promised zero with 0xFF bytes (NaN in fp16 / fp32 / fp64,
-1 in int32) at the start of every call that uses it.  Each case runs the same calls on a poisoned handle and on a fresh unpoisoned
twin with the same weights and inputs, and every output must be bit-for-bit the twin's: a kernel that reads an element nothing wrote
in the call reads NaN, and NaN reaches its output.  Every tensor the package allocates for an output is pre-filled with NaN (torch.empty
is wrapped), and no output may hold NaN, so an element the contract writes -- the zeros past a clip's end, after a slot's nout, in a
held slot's row included -- but a kernel skips shows too.

Buffers promised zero (WS_ZERO, grow-only) cannot be poisoned; the geometry histories cover them: a poisoned handle runs a series of
calls at other geometries first, and its last call must equal a fresh twin that ran only that call.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from fsnplus_b200 import _lib, metrics
from fsnplus_b200.model import FullSubNet_Plus, Model
from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP, ChunkStream, StreamingFullSubNet
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KNOBS = ("FSN_POISON", "FSN_SB_WINDOW", "FSN_WS_CAP_GB", "FSN_SB_CHUNK", "FSN_NO_WS", "FSN_FRONT_OVERLAP", "FSN_LSTM_IMPL")
INF = float("inf")


@pytest.fixture
def nan_out(monkeypatch):
    """Every tensor made by torch.empty while the test runs is filled first: NaN (floating, complex), 0xFF (uint8), -1 (integers)."""
    empty = torch.empty

    def filled(*a, **k):
        t = empty(*a, **k)
        if t.is_floating_point() or t.is_complex():
            t.fill_(float("nan"))
        elif t.dtype != torch.bool:
            t.fill_(255 if t.dtype == torch.uint8 else -1)
        return t

    monkeypatch.setattr(torch, "empty", filled)


def _make(cls, cfg, params, monkeypatch, poison, **env):
    """A model whose handle was created with FSN_POISON = poison and the knobs env (all read once, at create)."""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    if poison:
        monkeypatch.setenv("FSN_POISON", "1")
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))
    m = cls(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    return m


def _bits(t):
    t = t.detach()
    if t.is_complex():
        t = torch.view_as_real(t)
    t = t.contiguous()
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16, 1: torch.uint8}[t.element_size()])


def _same(got, want, label):
    """Bit-for-bit equal, with where they first differ otherwise, and free of NaN: every output the contract writes is finite, so a
    NaN is poison that reached it or an element a kernel left as the caller's NaN pre-fill -- in both handles alike when a store is
    skipped."""
    if isinstance(got, (tuple, list)):
        assert len(got) == len(want), label
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"{label}[{i}]")
        return
    assert tuple(got.shape) == tuple(want.shape), (label, tuple(got.shape), tuple(want.shape))
    a, b = _bits(got), _bits(want)
    for t, who in ((got, "poisoned handle"), (want, "twin")):
        r = torch.view_as_real(t) if t.is_complex() else t
        if r.is_floating_point() and torch.isnan(r).any():
            raise AssertionError(f"{label}: the {who}'s output holds {int(torch.isnan(r).sum())} NaN, first at "
                                 f"{tuple(torch.isnan(r).nonzero()[0].tolist())}")
    if torch.equal(a, b):
        return
    bad = (a != b).nonzero()
    raise AssertionError(f"{label}: {bad.shape[0]} elements differ from the unpoisoned twin, first at {tuple(bad[0].tolist())}")


# ---------------------------------------------------------------------------------------------------------------------------------
# configurations and inputs
F = 33                                                           # n_fft 64, hop 32
HOP = F - 1


def _plus(**over):
    c = O.default_plus_config()
    c.update(num_freqs=F, sb_num_neighbors=3, sb_model_hidden_size=64)
    c.update(over)
    return c


def _fsn(**over):
    c = O.default_fsn_config()
    c.update(num_freqs=F, sb_num_neighbors=3, sb_model_hidden_size=64, fb_model_hidden_size=48)
    c.update(over)
    return c


# name: (model class, config, knobs); wide Isb 66 = 9 + 3 * 19, 128 = 5 + 3 * 41 (FullSubNet+)
OFFLINE = {
    "lstm": (FullSubNet_Plus, _plus(), {}),
    "gru": (FullSubNet_Plus, _plus(sequence_model="GRU"), {}),
    "mma": (FullSubNet_Plus, _plus(lstm_impl="mma"), {}),
    "tcn": (FullSubNet_Plus, _plus(sequence_model="TCN", sb_model_hidden_size=32), {}),
    "wide66": (FullSubNet_Plus, _plus(sb_num_neighbors=4, fb_num_neighbors=9), {}),
    "wide66_mma": (FullSubNet_Plus, _plus(sb_num_neighbors=4, fb_num_neighbors=9, lstm_impl="mma"), {}),
    "wide128": (FullSubNet_Plus, _plus(sb_num_neighbors=2, fb_num_neighbors=20), {}),
    "wide128_mma": (FullSubNet_Plus, _plus(sb_num_neighbors=2, fb_num_neighbors=20, lstm_impl="mma"), {}),
    "cum_laplace": (FullSubNet_Plus, _plus(norm_type="cumulative_laplace_norm"), {}),
    "gaussian": (FullSubNet_Plus, _plus(norm_type="offline_gaussian_norm"), {}),
    "cum_layer": (FullSubNet_Plus, _plus(norm_type="cumulative_layer_norm"), {}),
    "fsn_ws": (Model, _fsn(), {}),
    "fsn_no_ws": (Model, _fsn(), {"FSN_NO_WS": 1}),
    "fsn_gru_cum": (Model, _fsn(sequence_model="GRU", norm_type="cumulative_layer_norm"), {}),
}


def _params(cls, cfg, seed=3):
    if cfg["sequence_model"] == "TCN":
        return S.make_params(cfg, seed=seed)
    return (O.make_params_plus if cls is FullSubNet_Plus else O.make_params_fsn)(cfg, seed=seed)


def _pair(cls, cfg, monkeypatch, **env):
    p = _params(cls, cfg)
    return _make(cls, cfg, p, monkeypatch, True, **env), _make(cls, cfg, p, monkeypatch, False, **env)


def _spec(B, T, seed):
    """Noisy spectra [B, 1, F, T] (mag, real, imag) on the device."""
    X = O.stft(O.synth_clips(B, num_samples=(T - 1) * HOP, seed0=seed), 2 * HOP, HOP, 2 * HOP)[..., :T]
    return tuple(torch.from_numpy(np.ascontiguousarray(a[:, None].astype(np.float32))).to(DEV) for a in (np.abs(X), X.real, X.imag))


def _wave(B, L, seed):
    return torch.from_numpy(O.synth_clips(B, num_samples=L, seed0=seed).astype(np.float32)).to(DEV)


def _isb(m):
    c = m._cfg
    return 2 * c.sb_num_neighbors + 1 + (3 if c.model_kind == _lib.KIND_PLUS else 1) * (2 * c.fb_num_neighbors + 1)


def _hook(m, x, B, T, Tw, frames=None):
    """fsn_model_sb_forward: the sub-band stage alone over the raw input x [B F, Isb, T + look_ahead] -> mask [B, 2, F, T]."""
    out = torch.empty((B, 2, F, T), dtype=torch.float32, device=DEV)
    fr = (C.c_int32 * B)(*frames) if frames is not None else None
    with torch.cuda.device(DEV):
        s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(_lib.load_library().fsn_model_sb_forward(m._handle, C.c_void_p(x.data_ptr()), B, T, Tw, fr, C.c_void_p(out.data_ptr()),
                                                            None, None, None, s))
    return out


def _call(m, name, B, T, seed):
    """One offline entry point on model m: its output"""
    plus = m._cfg.model_kind == _lib.KIND_PLUS
    mag, real, imag = _spec(B, T, seed)
    frames = [T] + [max(10, T - 7 * i) for i in range(1, B)]
    with torch.no_grad():
        if name == "forward":
            return m._run(mag, real if plus else None, imag if plus else None)
        if name == "forward_enhance":
            return m.enhance_spectrum(mag, real, imag)
        if name == "ragged":
            return m._run(mag, real if plus else None, imag if plus else None, frames=frames)
        if name == "ragged_enhance":
            return m.enhance_spectrum(mag, real, imag, frames=frames)
        if name == "enhance_lim":
            return m.enhance_spectrum(mag, real, imag, frames=frames, atten_lim_db=[6.0] + [INF] * (B - 2) + [20.0])
        L = (T - 1) * HOP
        lens = [L] + [max(HOP + 1, L - 37 * i - 5) for i in range(1, B)]
        if name == "audio":
            y = m.enhance_audio(_wave(B, L, seed), lens)
            if m.last_plan()[0] < B:
                return y
            # one sub-batch: the analysis planes and the enhanced spectrum it kept, zero past each clip's frames
            return y, m.get_stage("stft", (3, B, F, T), DEV), m.get_stage("enh", (B, F, T, 2), DEV)
        if name == "audio_lim":
            return m.enhance_audio(_wave(B, L, seed), lens, atten_lim_db=[12.0] + [INF] * (B - 1))
        if name == "hook":
            x = torch.randn((B * F, _isb(m), T + m._cfg.look_ahead), generator=torch.Generator().manual_seed(seed)).abs().to(DEV)
            return _hook(m, x, B, T, 32 if _layerwise(m) else 0, frames)
    raise ValueError(name)


ENTRY = ["forward", "forward_enhance", "ragged", "ragged_enhance", "enhance_lim", "audio", "audio_lim", "hook"]


def _layerwise(m):
    """The sub-band LSTM / GRU runs on the layer-wise kernels (time windows allowed): lstm_impl auto, hidden 64 (no FSN_LSTM_IMPL here)"""
    return not m._cfg.sb_tcn and m._cfg.lstm_impl == _lib.LSTM_IMPL["auto"]


def _twin_calls(P, Q, calls, label):
    """calls: (entry, B, T, seed) run on the poisoned P and the twin Q; every output and launch count equal"""
    for name, B, T, seed in calls:
        if name == "hook" and P._cfg.sb_tcn:
            continue
        got = _call(P, name, B, T, seed)
        nP = P.last_launch_count()
        want = _call(Q, name, B, T, seed)
        torch.cuda.synchronize()
        _same(got, want, f"{label} {name} B={B} T={T}")
        assert nP == Q.last_launch_count(), (label, name, nP, Q.last_launch_count())


@pytest.mark.parametrize("variant", list(OFFLINE))
def test_offline_entry_points(variant, monkeypatch, nan_out):
    """Every offline entry point on every route: forward, enhance, ragged, limited, audio, the sub-band hook (windows on the layer-wise
    route)"""
    cls, cfg, env = OFFLINE[variant]
    P, Q = _pair(cls, cfg, monkeypatch, **env)
    _twin_calls(P, Q, [(e, 3, 45, 11 + i) for i, e in enumerate(ENTRY)], variant)
    if variant.startswith("fsn"):
        _call(Q, "forward", 2, 20, 1)
        assert _lib.load_library().fsn_model_last_fb_ws(Q._handle) == (variant != "fsn_no_ws")
    expect = "tcn" if variant == "tcn" else "tcgen05" if _layerwise(Q) else "mma"
    assert Q.last_lstm_impl() == expect, (variant, Q.last_lstm_impl())


def test_offline_default_geometry(monkeypatch, nan_out):
    """The default FullSubNet+ (F = 257, hidden 384): forward, ragged enhance, audio"""
    cfg = O.default_plus_config()
    p = O.make_params_plus(cfg, seed=2)
    P, Q = (_make(FullSubNet_Plus, cfg, p, monkeypatch, z) for z in (True, False))
    X = O.stft(O.synth_clips(2, num_samples=16000, seed0=7), 512, 256, 512)
    mag, real, imag = (torch.from_numpy(np.ascontiguousarray(a[:, None].astype(np.float32))).to(DEV) for a in (np.abs(X), X.real, X.imag))
    T = mag.shape[-1]
    wave = _wave(2, 16000, 8)
    with torch.no_grad():
        for m in (P, Q):
            m._outs = [m(mag, real, imag), m.enhance_spectrum(mag, real, imag, frames=[T, T - 20]),
                       m.enhance_audio(wave, [16000, 9999], atten_lim_db=[10.0, INF])]
    _same(P._outs, Q._outs, "default geometry")


def test_pipelined_lanes(monkeypatch, nan_out):
    """submit and forward_host(pipelined) with both workspace lanes in flight (FSN_FRONT_OVERLAP=1)"""
    P, Q = _pair(FullSubNet_Plus, _plus(), monkeypatch, FSN_FRONT_OVERLAP=1)
    ins = [_spec(3, 40, 20 + i) for i in range(3)]
    host = [tuple(t.cpu().pin_memory() for t in x) for x in (_spec(2, 37, 30), _spec(4, 29, 31))]
    outs = {}
    with torch.no_grad():
        for m in (P, Q):
            o = [m.submit(*x) for x in ins]
            m.wait()
            e = [m.enhance_spectrum(*x, pipelined=True) for x in ins[:2]]
            m.wait()
            h = [m.forward_host(*x, pipelined=True) for x in host]
            m.sync_host()
            torch.cuda.synchronize()
            outs[id(m)] = o + e + [t.clone() for t in h]
    _same(outs[id(P)], outs[id(Q)], "pipelined")


# ---------------------------------------------------------------------------------------------------------------------------------
# planner paths
def test_planner_sub_batches_and_windows(monkeypatch, nan_out):
    """Sub-batches under a small cap, FSN_SB_WINDOW windows with a cumulative norm (the packer's sums across windows)"""
    cfg = _plus(norm_type="cumulative_laplace_norm")
    cap = _lib.plan_forward(FullSubNet_Plus(**cfg)._cfg, 2, 70, cap_bytes=1e12)[2] / 1e9      # windows, or sub-batches with them
    for env in ({"FSN_WS_CAP_GB": cap}, {"FSN_SB_WINDOW": 32}, {"FSN_SB_WINDOW": 64, "FSN_WS_CAP_GB": cap / 2}):
        P, Q = _pair(FullSubNet_Plus, cfg, monkeypatch, **env)
        _twin_calls(P, Q, [("forward", 6, 70, 40), ("ragged_enhance", 5, 70, 41), ("audio", 4, 70, 42)], str(env))
        bs, tw = P.last_plan()
        assert (bs < 4 or tw > 0) and (tw > 0 or "FSN_SB_WINDOW" not in env), (env, bs, tw)


def test_planner_bin_chunks(monkeypatch, nan_out):
    """The sub-band TCN in FSN_SB_CHUNK bin chunks, alone and with sub-batches"""
    cfg = _plus(sequence_model="TCN", sb_model_hidden_size=32)
    b1 = _lib.plan_forward_bins(FullSubNet_Plus(**cfg)._cfg, 1, 50, cap_bytes=1e12, force_bins=16)[3]
    for env in ({"FSN_SB_CHUNK": 7}, {"FSN_SB_CHUNK": 16, "FSN_WS_CAP_GB": 2.5 * b1 / 1e9}):
        P, Q = _pair(FullSubNet_Plus, cfg, monkeypatch, **env)
        _twin_calls(P, Q, [("forward", 5, 50, 50), ("ragged_enhance", 4, 50, 51), ("audio_lim", 3, 50, 52)], str(env))
        assert P.last_plan_bins()[2] > 0


# ---------------------------------------------------------------------------------------------------------------------------------
# geometry histories: the zero-promised grow-only buffers (fbin, fbout, magpad, fbx, hseq, xn, tsse_scale, sb_rowsum, cstate)
HISTORIES = {
    "B_shrinks": [("forward", 130, 24, 60), ("forward", 65, 24, 61), ("forward", 1, 24, 62)],
    "T_mod4": [("forward", 2, 41, 63), ("forward_enhance", 2, 38, 64), ("forward", 2, 36, 65), ("forward", 2, 35, 66)],
    "ragged_after_full": [("forward", 3, 40, 67), ("forward", 3, 44, 68), ("ragged", 3, 40, 69)],
    "audio_after_spectral": [("forward_enhance", 4, 50, 70), ("audio", 3, 45, 71)],
    "spectral_after_audio": [("audio", 4, 50, 72), ("ragged_enhance", 3, 45, 73)],
    "limited_after_unlimited": [("ragged_enhance", 3, 45, 74), ("enhance_lim", 3, 45, 75)],
    "window_after_wide": [("forward", 130, 20, 76), ("hook", 2, 70, 77)],
}


@pytest.mark.parametrize("model", ["lstm", "tcn", "cum_layer", "fsn_ws", "fsn_gru_cum"])
@pytest.mark.parametrize("history", list(HISTORIES))
def test_geometry_history(model, history, monkeypatch, nan_out):
    """A poisoned handle after calls at other geometries equals a fresh twin that ran only the last call"""
    cls, cfg, env = OFFLINE[model]
    P, Q = _pair(cls, cfg, monkeypatch, **env)
    calls = HISTORIES[history]
    if calls[-1][0] == "hook" and cfg["sequence_model"] == "TCN":
        pytest.skip("the sub-band hook runs the LSTM / GRU")
    for name, B, T, seed in calls[:-1]:
        _call(P, name, B, T, seed)
    _twin_calls(P, Q, calls[-1:], f"{model} {history}")


def test_window_history(monkeypatch, nan_out):
    """FSN_SB_WINDOW=32 with a cumulative norm: T' across multiples of 32 (a partial last window) on one handle"""
    cfg = _plus(norm_type="cumulative_layer_norm")
    P, Q = _pair(FullSubNet_Plus, cfg, monkeypatch, FSN_SB_WINDOW=32)
    for name, B, T, seed in [("forward", 2, 100, 80), ("forward", 3, 62, 81), ("ragged", 2, 95, 82)]:
        _call(P, name, B, T, seed)
    _twin_calls(P, Q, [("forward_enhance", 2, 45, 83)], "windows")


# ---------------------------------------------------------------------------------------------------------------------------------
# streaming (StreamingFullSubNet: fullsubnet.Model with a cumulative norm)
def _stream_cfg(**over):
    return _fsn(norm_type="cumulative_laplace_norm", **over)


def _stream_pair(monkeypatch, B, **env):
    cfg = _stream_cfg()
    p = _params(Model, cfg)
    ms = [_make(Model, cfg, p, monkeypatch, z, **env) for z in (True, False)]
    return ms, [StreamingFullSubNet(m, B, DEV) for m in ms]


def _mag(B, K, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B, F, K), generator=g) * 2 + 1e-3).to(DEV)


MASK_CALLS = [  # (kind, K, flags)
    ("chunk", 37, [START, START, START, START, HOLD, START]),
    ("slots", 1, [STEP, HOLD, STEP, STEP, START, STEP]),
    ("chunk", 1, [STEP, STEP, HOLD, STEP, STEP, HOLD]),
    ("chunk", 5, [STEP, START, STEP, HOLD, STEP, STEP]),
    ("chunk", 64, [STEP, STEP, STEP, START, HOLD, STEP]),
    ("slots", 1, [HOLD, STEP, STEP, STEP, STEP, START]),
    ("chunk", 3, [HOLD, HOLD, HOLD, HOLD, HOLD, HOLD]),
    ("chunk", 2, [STEP, STEP, START, STEP, START, STEP]),
]


def _run_mask(st, calls, seed):
    outs = []
    with torch.no_grad():
        for i, (kind, K, flags) in enumerate(calls):
            x = _mag(st.B, K, seed + i)
            outs += list(st.step_chunk(x, flags) if kind == "chunk" else st.step_slots(x[..., 0], flags))
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("path", ["generic", "layerwise_low_cap", "generic_no_ws", "layerwise_no_ws"])
def test_stream_mask_calls(path, monkeypatch, nan_out):
    """Per-frame slot and chunk calls with K varying per call (37, 1, 5, 64, ...) and STARTs / HOLDs, on both sub-band paths and
    both full-band kernels; then the lockstep per-frame call on a handle of its own"""
    env = {} if "no_ws" not in path else {"FSN_NO_WS": 1}
    if path.startswith("generic"):
        env["FSN_LSTM_IMPL"] = 1
    else:
        _, _, b = _lib.stream_chunk_plan(Model(**_stream_cfg())._cfg, 1, 16, 1e12)
        env["FSN_WS_CAP_GB"] = b / 1e9                          # K = 37, 64: windows; several sessions: sub-batches
    ms, (sp, sq) = _stream_pair(monkeypatch, 6, **env)
    _same(_run_mask(sp, MASK_CALLS, 100), _run_mask(sq, MASK_CALLS, 100), f"{path} slot / chunk calls")
    lp, lq = StreamingFullSubNet(ms[0], 3, DEV), StreamingFullSubNet(ms[1], 3, DEV)
    with torch.no_grad():
        for t in range(6):
            x = _mag(3, 1, 200 + t)[..., 0]
            a, b = lp.step(x), lq.step(x)
            assert (a is None) == (b is None)
            if a is not None:
                _same(a, b, f"{path} lockstep tick {t}")


AUDIO_HOP_CALLS = [  # (kind, K, flags, hops)
    ("hop", 1, [START, START, HOLD, START], None),
    ("hop", 1, [STEP, STEP, START, STEP], None),
    ("chunk", 3, [STEP, STEP, STEP, STEP], [3, 1, 2, 3]),
    ("chunk", 5, [FLUSH, STEP, STEP, HOLD], [2, 5, 3, 0]),
    ("chunk", 2, [FLUSH, FLUSH, STEP, START], [0, 1, 2, 2]),
    ("chunk", 4, [START, FLUSH, FLUSH, STEP], [1, 0, 1, 4]),
]
AUDIO_SAMPLE_CALLS = [  # (S, flags, counts)
    (100, [STEP, HOLD, START, STEP], [100, 0, 45, 7]),
    (80, [STEP, START, STEP, FLUSH], [61, 80, 13, 3]),
    (64, [FLUSH, STEP, STEP, START], [5, 64, 0, 50]),
    (40, [START, FLUSH, FLUSH, STEP], [40, 9, 1, 33]),
]


def _run_audio(st, seed):
    g = torch.Generator().manual_seed(seed)
    outs = []
    st.set_atten_lim([1], 9.0)
    with torch.no_grad():
        for kind, K, flags, hops in AUDIO_HOP_CALLS:
            x = (torch.randn((st.B, K * st.hop), generator=g) * 0.1).to(DEV)
            outs += list(st.step_audio(x, flags, return_mask=True) if kind == "hop" else st.step_audio_chunk(x, flags, hops, return_mask=True))
        for S, flags, counts in AUDIO_SAMPLE_CALLS:
            x = (torch.randn((st.B, S), generator=g) * 0.1).to(DEV)
            outs += list(st.step_audio_samples(x, counts, flags))
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("path", ["generic", "layerwise_low_cap", "no_ws"])
def test_stream_audio_calls(path, monkeypatch, nan_out):
    """Per-hop, K-hop (hop counts below K, FLUSHes) and sample-granular audio calls"""
    env = {"FSN_LSTM_IMPL": 1} if path == "generic" else {"FSN_NO_WS": 1} if path == "no_ws" else {}
    if path == "layerwise_low_cap":
        _, _, b = _lib.stream_chunk_plan(Model(**_stream_cfg())._cfg, 1, 2, 1e12)
        env["FSN_WS_CAP_GB"] = 1.5 * b / 1e9
    _, (sp, sq) = _stream_pair(monkeypatch, 4, **env)
    _same(_run_audio(sp, 300), _run_audio(sq, 300), f"{path} audio calls")


@pytest.mark.parametrize("path", ["generic", "layerwise"])
def test_stream_sessions_after_traffic(path, monkeypatch, nan_out):
    """A session started in a slot of a busy poisoned handle, and a saved session loaded into one, equal the same sessions on a fresh
    unpoisoned handle whose other slots never ran"""
    env = {"FSN_LSTM_IMPL": 1} if path == "generic" else {}
    ms, (sp, sq) = _stream_pair(monkeypatch, 6, **env)
    with torch.no_grad():
        for i, K in enumerate((40, 7, 1, 64)):                     # traffic on slots 0..4
            sp.step_chunk(_mag(6, K, 400 + i), [START if i == 0 else STEP] * 5 + [HOLD])
        mine = [START, STEP, STEP]
        got, want = [], []
        for i, K in enumerate((9, 33, 2)):
            x = _mag(6, K, 500 + i)
            busy = [STEP, STEP, HOLD, STEP, STEP, mine[i]]
            got.append(sp.step_chunk(x, busy)[0][5])
            want.append(sq.step_chunk(x, [HOLD] * 5 + [mine[i]])[0][5])
        state = sq.save_slots([5])
        sp.load_slots([2], state)
        fresh = StreamingFullSubNet(ms[1], 6, DEV)
        fresh.load_slots([2], state)
        for i, K in enumerate((5, 48)):
            x = _mag(6, K, 600 + i)
            got.append(sp.step_chunk(x, [STEP] * 6)[0][2])
            want.append(fresh.step_chunk(x, [HOLD, HOLD, STEP, HOLD, HOLD, HOLD])[0][2])
    torch.cuda.synchronize()
    _same(got, want, f"{path} sessions after traffic")


# ---------------------------------------------------------------------------------------------------------------------------------
# chunk sessions (ChunkStream: every completed chunk of every session through the offline audio call)
CHUNK_CALLS = [  # (S, flags, counts): completed rows 3, 1, 6, 0, 4, ...
    (900, [START, START, HOLD, START], [600, 300, 0, 900]),
    (300, [STEP, STEP, START, HOLD], [100, 250, 300, 0]),
    (1400, [STEP, STEP, STEP, STEP], [1400, 600, 700, 200]),
    (50, [STEP, HOLD, STEP, STEP], [50, 0, 10, 40]),
    (700, [FLUSH, STEP, FLUSH, STEP], [100, 700, 3, 500]),
    (400, [START, FLUSH, HOLD, FLUSH], [400, 0, 0, 77]),
]


@pytest.mark.parametrize("model", ["lstm", "tcn", "fsn_ws"])
def test_chunk_sessions(model, monkeypatch, nan_out):
    """Overlapped-chunk sessions with the completed-row count growing and shrinking from call to call, under a cap that splits the
    rows into sub-batches"""
    cls, cfg, _ = OFFLINE[model]
    c = cls(**cfg)._cfg
    cap = _lib.plan_audio(c, 2, 512 + 256, cap_bytes=1e12)[3]          # sub-batches of rows, or windows
    bs, tw, _, _ = _lib.plan_audio(c, 6, 512 + 256, cap_bytes=cap)
    assert bs < 6 or tw > 0
    P, Q = _pair(cls, cfg, monkeypatch, FSN_WS_CAP_GB=cap / 1e9)
    res = []
    for m in (P, Q):
        cs = ChunkStream(m, 4, 512, DEV)
        cs.set_atten_lim([3], 8.0)
        g = torch.Generator().manual_seed(700)
        outs = []
        with torch.no_grad():
            for S, flags, counts in CHUNK_CALLS:
                outs += list(cs.step((torch.randn((4, S), generator=g) * 0.1).to(DEV), counts, flags))
        torch.cuda.synchronize()
        res.append(outs)
        cs.close()
    _same(res[0], res[1], f"{model} chunk sessions")


# ---------------------------------------------------------------------------------------------------------------------------------
# metrics: the caller's workspace
def test_metrics_workspace():
    """SI-SDR and STOI with a workspace of 0xFF bytes equal those with a zeroed one, and the module's calls after a large NaN tensor
    went back to torch's cache"""
    lib = _lib.load_library()
    B, L, sr = 3, 24000, 16000
    ref = _wave(B, L, 800)
    est = (ref + 0.3 * _wave(B, L, 801)).contiguous()
    lens = [L, 17001, 9000]
    hl = (C.c_int64 * B)(*lens)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t: C.c_void_p(t.data_ptr())
    res = {}
    for name in ("si_sdr", "stoi"):
        nb = C.c_int64()
        if name == "si_sdr":
            _lib.check(lib.fsn_metric_si_sdr_workspace(B, L, hl, C.byref(nb)))
        else:
            _lib.check(lib.fsn_metric_stoi_workspace(B, L, hl, sr, C.byref(nb)))
        for fill in (0xFF, 0):
            work = torch.full((max(nb.value, 1),), fill, dtype=torch.uint8, device=DEV)
            out = torch.full((B,), float("nan"), dtype=torch.float64, device=DEV)
            if name == "si_sdr":
                _lib.check(lib.fsn_metric_si_sdr(p(ref), p(est), B, L, hl, p(work), nb.value, p(out), s))
            else:
                _lib.check(lib.fsn_metric_stoi(p(ref), p(est), B, L, hl, sr, p(work), nb.value, p(out), s))
            res[name, fill] = out
        _same(res[name, 0xFF], res[name, 0], f"{name}: 0xFF vs zeroed workspace")
        # NaN blocks of the workspace's and the scores' sizes, and a large one, freed into torch's cache for the module's call
        junk = [torch.full((n,), float("nan"), device=DEV) for n in (nb.value // 4 + 1, B * 2, 1 << 24)]
        del junk
        got = metrics.si_sdr(ref, est, lens) if name == "si_sdr" else metrics.stoi(ref, est, sr, lens)
        _same(got, res[name, 0], f"metrics.{name} after NaN in the cache")
    assert torch.isfinite(res["stoi", 0]).all() and torch.isfinite(res["si_sdr", 0]).all()
