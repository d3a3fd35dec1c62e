"""Every entry point keeps the caller's stream order (include/fsnplus_b200.h, "Stream order"; DESIGN.md §2, "Stream order").

The gate: on the stream under test a sleep kernel runs first and an event E is recorded behind it; then, on the same stream, the
inputs' final values are copied into buffers that held NaN, the call is made, and every output is copied into a fresh tensor.  A call
that does not synchronise must return with E still pending (else the case fails as inconclusive, naming the call: a call that waits
on the GPU breaks the promise too).  Right after the call returns, every host array it took is overwritten with other valid values.
The truth is the same calls on a fresh twin handle, ungated, on one stream.  Outputs must be bit-identical to the twin's.

Stream kinds: the legacy default stream (torch's default), cudaStreamPerThread (handle 2) and a non-blocking torch stream.  Every
shape runs once ungated first: a first call allocates, and a cudaFree on growth synchronises the device.

Cross-stream cases use identical shapes, lengths and slot sets, and fullsubnet.Model with FSN_NO_WS=1 (no grid barrier), so a wrong
order can change values but never an index, a length or a barrier.  Each gate sleeps about 50 ms.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from fsnplus_b200 import _lib
from fsnplus_b200.inference import EnhancePipeline
from fsnplus_b200.model import FullSubNet_Plus, Model
from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP, ChunkStream, StreamingFullSubNet
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F, HOP = 33, 32                                                  # n_fft 64
GATE_CYCLES = 90_000_000                                         # ~50 ms at the H100's clocks
KNOBS = ("FSN_NO_WS", "FSN_FRONT_OVERLAP", "FSN_POISON", "FSN_WS_CAP_GB", "FSN_SB_WINDOW", "FSN_SB_CHUNK", "FSN_LSTM_IMPL")
NAN = float("nan")
QUEUE_DEPTH = 4                                                  # PinnedStage::NSLOT: one slot per streaming call

# Which case covers each header function that takes a stream or creates, finalizes, loads or destroys a handle
# (tests/test_stream_order_cpu.py checks the header against this table).
CASES = {
    "test_offline_calls": ["fsn_model_forward", "fsn_model_forward_enhance", "fsn_model_forward_ragged",
                           "fsn_model_forward_enhance_ragged", "fsn_model_forward_enhance_lim", "fsn_model_enhance_audio",
                           "fsn_model_enhance_audio_lim", "fsn_apply_cirm", "fsn_model_get_stage", "fsn_model_sb_forward",
                           "fsn_gemm_f16"],
    "test_forward_host": ["fsn_model_forward_host"],
    "test_first_audio_call": ["fsn_model_create", "fsn_model_finalize", "fsn_model_destroy"],
    "test_model_file_load": ["fsn_model_load"],
    "test_full_subnet_plus": ["fsn_model_forward", "fsn_model_enhance_audio"],
    "test_pipeline": ["fsn_model_submit", "fsn_model_submit_enhance", "fsn_model_wait", "fsn_model_wait_lane",
                      "fsn_model_forward_host_async"],
    "test_streaming_calls": ["fsn_stream_step", "fsn_stream_step_slots", "fsn_stream_step_chunk", "fsn_stream_step_audio_slots",
                             "fsn_stream_step_audio_chunk", "fsn_stream_step_audio_samples", "fsn_stream_save_slots",
                             "fsn_stream_load_slots", "fsn_stream_get_stage"],
    "test_chunk_sessions": ["fsn_chunk_stream_step", "fsn_chunk_stream_save_slots", "fsn_chunk_stream_load_slots"],
    "test_metrics": ["fsn_metric_si_sdr", "fsn_metric_stoi", "fsn_metric_sdr"],
    "test_queue_depth": ["fsn_stream_step_chunk"],
    "test_create_under_busy_default_stream": ["fsn_stream_create", "fsn_chunk_stream_create"],
    "test_destroy_behind_gate": ["fsn_stream_destroy", "fsn_chunk_stream_destroy"],
    "test_cross_stream_plain_forwards": ["fsn_model_forward"],
    "test_cross_stream_chunk_and_offline": ["fsn_chunk_stream_step", "fsn_model_enhance_audio"],
    "test_cross_stream_stage_and_state": ["fsn_model_get_stage", "fsn_stream_save_slots", "fsn_stream_load_slots"],
    "test_enhance_pipeline": [],
    "test_tools_inference_streams": [],
}

LIB = None


def lib():
    global LIB
    if LIB is None:
        LIB = _lib.load_library()
    return LIB


def vp(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def sp(s):
    return C.c_void_p(s.cuda_stream)


def _stream(kind):
    if kind == "legacy":
        return torch.cuda.default_stream(DEV)
    if kind == "per_thread":
        return torch.cuda.ExternalStream(2, device=DEV)          # cudaStreamPerThread
    return torch.cuda.Stream(DEV)                                 # torch's pool streams are non-blocking


KINDS = ["legacy", "per_thread", "nonblocking"]


def _late(x):
    """x's value, written on the current stream into a buffer that held NaN (after the gate when one is pending)"""
    y = torch.full_like(x, NAN) if x.is_floating_point() or x.is_complex() else torch.full_like(x, -1)
    return y.copy_(x)


def _gate(s):
    """Sleep on stream s and return the event recorded behind it"""
    with torch.cuda.stream(s):
        torch.cuda._sleep(GATE_CYCLES)
        e = torch.cuda.Event()
        e.record(s)
    return e


_TRACE = {"e": None, "first": None}


def _mark(name):
    """Notes the first call after which the pending gate (set by _run_gated) had cleared"""
    e = _TRACE["e"]
    if e is not None and _TRACE["first"] is None and e.query():
        _TRACE["first"] = name


def _pending(e, what):
    first, _TRACE["e"], _TRACE["first"] = _TRACE["first"], None, None
    assert not e.query(), (f"inconclusive: the gate had cleared when {what} returned (the call waited on the GPU, or the gate is too "
                           f"short); first seen after {first}")


def _same(got, want, label, tol=None):
    if isinstance(got, (list, tuple)):
        assert len(got) == len(want), label
        for i, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"{label}[{i}]", tol)
        return
    if not torch.is_tensor(got):
        assert got == want, (label, got, want)
        return
    g, w = got.detach().cpu(), want.detach().cpu()
    assert g.shape == w.shape, (label, g.shape, w.shape)
    if g.is_complex():
        g, w = torch.view_as_real(g), torch.view_as_real(w)
    if tol is None:
        if torch.equal(g, w) or (g.is_floating_point() and torch.equal(torch.nan_to_num(g, 7.0), torch.nan_to_num(w, 7.0))
                                 and torch.equal(g.isnan(), w.isnan())):
            return
        bad = (g != w) & ~(g.isnan() & w.isnan()) if g.is_floating_point() else g != w
        raise AssertionError(f"{label}: {int(bad.sum())} elements differ from the twin, first at {tuple(bad.nonzero()[0].tolist())}")
    assert torch.isfinite(g).all(), f"{label}: non-finite output"
    d = (g.double() - w.double()).abs().max().item() / max(w.double().pow(2).mean().sqrt().item(), 1e-30)
    assert d <= tol, f"{label}: max |d| / RMS = {d:.3g} > {tol}"


def _model(cls, cfg, params, monkeypatch, **env):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
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


def _fsn_cfg():
    c = O.default_fsn_config()
    c.update(num_freqs=F, sb_num_neighbors=3, sb_model_hidden_size=64, fb_model_hidden_size=48, norm_type="cumulative_laplace_norm")
    return c


def _plus_cfg():
    c = O.default_plus_config()
    c.update(num_freqs=F, sb_num_neighbors=3, sb_model_hidden_size=64)
    return c


def _pair(monkeypatch, plus=False, **env):
    """A model and its twin: same weights, separate handles"""
    cls, cfg = (FullSubNet_Plus, _plus_cfg()) if plus else (Model, _fsn_cfg())
    p = (O.make_params_plus if plus else O.make_params_fsn)(cfg, seed=5)
    return _model(cls, cfg, p, monkeypatch, **env), _model(cls, cfg, p, monkeypatch, **env)


def _spec(B, T, seed):
    X = O.stft(O.synth_clips(B, num_samples=(T - 1) * HOP, seed0=seed), 2 * HOP, HOP, 2 * HOP)[..., :T]
    return tuple(torch.from_numpy(np.ascontiguousarray(a[:, None].astype(np.float32))).to(DEV) for a in (np.abs(X), X.real, X.imag))


def _wave(B, L, seed):
    return torch.from_numpy(O.synth_clips(B, num_samples=L, seed0=seed).astype(np.float32)).to(DEV)


def _i32(v):
    return (C.c_int32 * len(v))(*v)


def _i64(v):
    return (C.c_int64 * len(v))(*v)


def _f32(v):
    return (C.c_float * len(v))(*v)


def _overwrite(arr, vals):
    for i, v in enumerate(vals):
        arr[i] = v


def _run_gated(kind, calls, label):
    """calls(s): enqueue inputs, the call(s) and output copies on s; return the outputs.  Run once ungated (warm-up), then gated;
    every call must have returned with the gate pending.  The calls keep one forward geometry: a forward at another one reallocates
    part of the model's workspace, which synchronises the device (the header's "Queue depth")."""
    s = _stream(kind)
    with torch.cuda.stream(s):
        calls(s)
    torch.cuda.synchronize()
    e = _gate(s)
    _TRACE["e"], _TRACE["first"] = e, None
    with torch.cuda.stream(s):
        out = calls(s)
    _pending(e, label)
    torch.cuda.synchronize()
    return out


def _truth(calls):
    """calls run twice on the legacy stream, as _run_gated runs them (a warm-up, then the checked pass)"""
    s = torch.cuda.default_stream(DEV)
    with torch.cuda.stream(s):
        calls(s)
        out = calls(s)
    torch.cuda.synchronize()
    return out


# ---------------------------------------------------------------------------------------------------------------------------------
# offline
B, T = 3, 40
L = (T - 1) * HOP


def _offline_calls(m, ins, wave, x_sb, ga, gb, part):
    """Every offline device-buffer call of model m on the current stream; host arrays overwritten with other valid values on return"""
    h = m._handle
    mag, real, imag = ins
    crm0 = torch.randn((B, 2, F, T), generator=torch.Generator().manual_seed(9)).to(DEV)

    def calls(s):
        st = sp(s)
        a, r, i = (_late(t) for t in ins)
        outs = []
        o = torch.full((B, 2, F, T), NAN, device=DEV)
        if part == 3:
            return hook(st, o)
        _lib.check(lib().fsn_model_forward(h, vp(a), None, None, B, T, vp(o), st))
        _mark("fsn_model_forward")
        outs.append(o.clone())
        stage = torch.full((1 * B * F * (T + m._cfg.look_ahead),), NAN, device=DEV)
        _lib.check(lib().fsn_model_get_stage(h, b"fb_out", vp(stage), stage.numel(), st))
        _mark("fsn_model_get_stage")
        outs.append(stage.clone())
        e = torch.full((B, F, T, 2), NAN, device=DEV)
        _lib.check(lib().fsn_model_forward_enhance(h, vp(a), vp(r), vp(i), B, T, vp(e), st))
        _mark("fsn_model_forward_enhance")
        outs.append(e.clone())
        fr = _i32([T, T - 9, T - 17])
        _lib.check(lib().fsn_model_forward_ragged(h, vp(a), None, None, B, T, fr, vp(o), st))
        _mark("fsn_model_forward_ragged")
        _overwrite(fr, [T - 3, T, T - 1])
        outs.append(o.clone())
        fr = _i32([T - 5, T, T - 11])
        _lib.check(lib().fsn_model_forward_enhance_ragged(h, vp(a), vp(r), vp(i), B, T, fr, vp(e), st))
        _mark("fsn_model_forward_enhance_ragged")
        _overwrite(fr, [T, T - 2, T])
        outs.append(e.clone())
        fr, db = _i32([T, T - 13, T - 4]), _f32([6.0, float("inf"), 15.0])
        _lib.check(lib().fsn_model_forward_enhance_lim(h, vp(a), vp(r), vp(i), B, T, fr, db, vp(e), st))
        _mark("fsn_model_forward_enhance_lim")
        _overwrite(fr, [T - 1, T, T])
        _overwrite(db, [0.0, 3.0, float("inf")])
        outs.append(e.clone())
        if part == 0:
            return outs
        w = _late(wave)
        y = torch.full_like(wave, NAN)
        if part == 2:                                               # a limited call plans another workspace: a part of its own
            ln, db = _i64([L - 61, L, L - 2]), _f32([10.0, 4.0, float("inf")])
            _lib.check(lib().fsn_model_enhance_audio_lim(h, vp(w), B, L, ln, db, vp(y), st))
            _mark("fsn_model_enhance_audio_lim")
            _overwrite(ln, [L, L - 1, L])
            _overwrite(db, [0.0, 0.0, 0.0])
            return [y.clone()]
        ln = _i64([L, L - 100, L - 333])
        _lib.check(lib().fsn_model_enhance_audio(h, vp(w), B, L, ln, vp(y), st))
        _mark("fsn_model_enhance_audio")
        _overwrite(ln, [L - 50, L, L - 7])
        outs.append(y.clone())
        stft = torch.full((3 * B * F * T,), NAN, device=DEV)
        _lib.check(lib().fsn_model_get_stage(h, b"stft", vp(stft), stft.numel(), st))
        _mark("fsn_model_get_stage")
        outs.append(stft.clone())
        crm = _late(crm0)
        noisy = _late(torch.complex(real[:, 0], imag[:, 0]))
        ce = torch.full((B, F, T), NAN + 0j, dtype=torch.complex64, device=DEV)
        _lib.check(lib().fsn_apply_cirm(vp(crm), vp(noisy), vp(ce), B, F, T, st))
        _mark("fsn_apply_cirm")
        outs.append(ce.clone())
        A, Bm = _late(ga), _late(gb)
        gc = torch.full((ga.shape[0], gb.shape[0]), NAN, dtype=torch.float16, device=DEV)
        _lib.check(lib().fsn_gemm_f16(vp(A), vp(Bm), vp(gc), ga.shape[0], gb.shape[0], ga.shape[1], 0, st))
        _mark("fsn_gemm_f16")
        outs.append(gc.clone())
        return outs

    def hook(st, o):                                                # the hook plans its own geometry: a part of its own
        xs = _late(x_sb)
        fr = _i32([T, T - 6, T - 30])
        _lib.check(lib().fsn_model_sb_forward(h, vp(xs), B, T, 0, fr, vp(o), None, None, None, st))
        _mark("fsn_model_sb_forward")
        _overwrite(fr, [T, T, T])
        return [o.clone()]
    return calls


def _offline_inputs(m):
    ins = _spec(B, T, 21)
    wave = _wave(B, L, 22)
    isb = 2 * 3 + 1 + (2 * m._cfg.fb_num_neighbors + 1)
    x_sb = torch.rand((B * F, isb, T + m._cfg.look_ahead), generator=torch.Generator().manual_seed(23)).to(DEV)
    g = torch.Generator().manual_seed(24)
    ga = (torch.randn((256, 128), generator=g) * 0.1).half().to(DEV)
    gb = (torch.randn((256, 128), generator=g) * 0.1).half().to(DEV)
    return ins, wave, x_sb, ga, gb


@pytest.mark.parametrize("kind", KINDS)
def test_offline_calls(kind, monkeypatch):
    """forward, enhance, both ragged calls, the limited enhance, both audio calls, fsn_apply_cirm, get_stage right after the forward and
    the audio call, the sub-band hook and the GEMM hook, all behind one gate"""
    P, Q = _pair(monkeypatch)
    args = _offline_inputs(P)
    for part in (0, 1, 2, 3):                                       # each within the queue depth of the model's staging ring
        got = _run_gated(kind, _offline_calls(P, *args, part), f"the offline calls (part {part}) on the {kind} stream")
        _same(got, _truth(_offline_calls(Q, *args, part)), f"offline {kind} part {part}")


@pytest.mark.parametrize("kind", KINDS)
def test_forward_host(kind, monkeypatch):
    """fsn_model_forward_host synchronises: only its result is checked, behind a gate on its stream"""
    P, Q = _pair(monkeypatch)
    mag = _spec(B, T, 30)[0].cpu()
    res = []
    for m, gate in ((P, True), (Q, False)):
        s = _stream(kind) if gate else torch.cuda.default_stream(DEV)
        out = torch.full((B, 2, F, T), NAN)
        if gate:
            _gate(s)
        _lib.check(lib().fsn_model_forward_host(m._handle, vp(mag), None, None, B, T, vp(out), sp(s)))
        _mark("fsn_model_forward_host")
        res.append(out.clone())
    torch.cuda.synchronize()
    _same(res[0], res[1], f"forward_host {kind}")


def test_first_audio_call(monkeypatch):
    """The first audio call of a fresh handle, under a gated non-blocking stream: the audio tables and the weights are in place
    (they are uploaded and synchronised at finalize) and it equals its twin.  A first call allocates its workspace and staging, which
    may synchronise the device: that is reported, and only the result is checked then."""
    P, Q = _pair(monkeypatch)
    wave = _wave(B, L, 31)
    s = _stream("nonblocking")
    e = _gate(s)
    with torch.cuda.stream(s):
        w = _late(wave)
        y = torch.full_like(wave, NAN)
        _lib.check(lib().fsn_model_enhance_audio(P._handle, vp(w), B, L, None, vp(y), sp(s)))
        if e.query():
            print("the first fsn_model_enhance_audio of a fresh handle synchronised (allocation): result checked only")
    torch.cuda.synchronize()
    _same(y, Q.enhance_audio(wave), "first audio call")


def test_model_file_load(monkeypatch, tmp_path):
    """A handle from fsn_model_load runs its first forward on a gated non-blocking stream: the upload is complete when load returns"""
    P, Q = _pair(monkeypatch)
    path = str(tmp_path / "m.fsn")
    Q.save_model_file(path)
    h = C.c_void_p()
    _lib.check(lib().fsn_model_load(path.encode(), C.byref(h)))
    _mark("fsn_model_load")
    try:
        mag = _spec(B, T, 32)[0]
        s = _stream("nonblocking")
        e = _gate(s)
        with torch.cuda.stream(s):
            a = _late(mag)
            o = torch.full((B, 2, F, T), NAN, device=DEV)
            _lib.check(lib().fsn_model_forward(h, vp(a), None, None, B, T, vp(o), sp(s)))
            _mark("fsn_model_forward")
            _pending(e, "the first fsn_model_forward of a loaded handle")
        torch.cuda.synchronize()
        with torch.no_grad():
            _same(o, Q(mag), "loaded model")
    finally:
        lib().fsn_model_destroy(h)


def test_full_subnet_plus(monkeypatch):
    """FullSubNet+ forward and audio behind a gate on a non-blocking stream (its full-band TCN sums gLN statistics with fp64 atomics
    in varying order: max |d| / RMS <= 1e-5)"""
    P, Q = _pair(monkeypatch, plus=True)
    ins, wave = _spec(B, T, 33), _wave(B, L, 34)

    def calls(m):
        def run(s):
            a, r, i = (_late(t) for t in ins)
            o = torch.full((B, 2, F, T), NAN, device=DEV)
            _lib.check(lib().fsn_model_forward(m._handle, vp(a), vp(r), vp(i), B, T, vp(o), sp(s)))
            _mark("fsn_model_forward")
            w, y = _late(wave), torch.full_like(wave, NAN)
            ln = _i64([L, L - 40, L - 90])
            _lib.check(lib().fsn_model_enhance_audio(m._handle, vp(w), B, L, ln, vp(y), sp(s)))
            _mark("fsn_model_enhance_audio")
            _overwrite(ln, [L, L, L])
            return [o.clone(), y.clone()]
        return run
    _same(_run_gated("nonblocking", calls(P), "FullSubNet+ calls"), _truth(calls(Q)), "FullSubNet+", tol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------------------
# pipeline
@pytest.mark.parametrize("overlap", [0, 1])
def test_pipeline(overlap, monkeypatch):
    """Three batches submitted behind a gate (submit, submit_enhance), read on ANOTHER stream after fsn_model_wait on it; then a plain
    forward on the gated stream right after them; wait_lane; then forward_host_async + sync_host.  FSN_FRONT_OVERLAP 0 and 1
    (two lanes: FullSubNet+)"""
    P, Q = _pair(monkeypatch, plus=True, FSN_FRONT_OVERLAP=overlap)
    ins = [_spec(2, 36, 40 + k) for k in range(3)]
    host = [tuple(t.cpu().pin_memory() for t in _spec(2, 36, 50 + k)) for k in range(2)]

    def run(m, s1, s2, gate):
        h = m._handle
        outs = []
        for g in (False, True) if gate else (True,):               # an ungated warm-up pass, then the gated one
            e = _gate(s1) if g and gate else None
            with torch.cuda.stream(s1):
                res, keep = [], []                                  # inputs stay untouched until fsn_model_wait
                for k, x in enumerate(ins):
                    a, r, i = (_late(t) for t in x)
                    keep.append((a, r, i))
                    if k == 1:
                        o = torch.full((2, F, 36, 2), NAN, device=DEV)
                        _lib.check(lib().fsn_model_submit_enhance(h, vp(a), vp(r), vp(i), 2, 36, vp(o), sp(s1)))
                        _mark("fsn_model_submit_enhance")
                    else:
                        o = torch.full((2, 2, F, 36), NAN, device=DEV)
                        _lib.check(lib().fsn_model_submit(h, vp(a), vp(r), vp(i), 2, 36, vp(o), sp(s1)))
                        _mark("fsn_model_submit")
                    res.append(o)
                lane = lib().fsn_model_last_lane(h)
            _lib.check(lib().fsn_model_wait(h, sp(s2)))
            _mark("fsn_model_wait")
            with torch.cuda.stream(s2):
                read = [o.clone() for o in res]                      # the reader on the other stream
            with torch.cuda.stream(s1):
                a, r, i = (_late(t) for t in ins[0])
                o = torch.full((2, 2, F, 36), NAN, device=DEV)
                _lib.check(lib().fsn_model_forward(h, vp(a), vp(r), vp(i), 2, 36, vp(o), sp(s1)))
                _mark("fsn_model_forward")
                read.append(o.clone())
                o2 = torch.full((2, 2, F, 36), NAN, device=DEV)
                _lib.check(lib().fsn_model_submit(h, vp(a), vp(r), vp(i), 2, 36, vp(o2), sp(s1)))
                _mark("fsn_model_submit")
            _lib.check(lib().fsn_model_wait_lane(h, lib().fsn_model_last_lane(h), sp(s2)))
            _mark("fsn_model_wait_lane")
            with torch.cuda.stream(s2):
                read.append(o2.clone())
            if e is not None:
                _pending(e, "fsn_model_submit / _submit_enhance / wait / wait_lane")
            hres = [torch.full((2, 2, F, 36), NAN).pin_memory() for _ in host]
            for x, ho in zip(host, hres):
                _lib.check(lib().fsn_model_forward_host_async(h, *(vp(t) for t in x), 2, 36, vp(ho), sp(s1)))
                _mark("fsn_model_forward_host_async")
            _lib.check(lib().fsn_model_sync_host(h))
            _mark("fsn_model_sync_host")
            torch.cuda.synchronize()
            outs = read + [t.clone() for t in hres]
        return outs, lane
    s1, s2 = _stream("nonblocking"), _stream("nonblocking")
    got, lane = run(P, s1, s2, True)
    d = torch.cuda.default_stream(DEV)
    want, _ = run(Q, d, d, False)
    assert overlap or lane == 0
    _same(got, want, f"pipeline overlap={overlap}", tol=1e-5)


# ---------------------------------------------------------------------------------------------------------------------------------
# streaming
SB = 4


def _mag(K, seed):
    return (torch.rand((SB, F, K), generator=torch.Generator().manual_seed(seed)) * 2 + 1e-3).to(DEV)


def _stream_calls(mask_st, audio_st, part):
    """Every streaming call on two handles of one model (a mask handle, an audio handle); host arrays overwritten on return.  The
    sequence starts every slot, so a warm-up pass leaves nothing behind."""
    g = torch.Generator().manual_seed(65)
    xin = {"m1": _mag(1, 60)[..., 0].contiguous(), "m2": _mag(1, 61)[..., 0].contiguous(), "k7": _mag(7, 62), "k3": _mag(3, 63),
           "k2": _mag(2, 64), "a1": (torch.randn((SB, HOP), generator=g) * 0.1).to(DEV),
           "a4": (torch.randn((SB, 4 * HOP), generator=g) * 0.1).to(DEV), "s75": (torch.randn((SB, 75), generator=g) * 0.1).to(DEV)}

    def calls(s):
        st, outs = sp(s), []
        h, ha = mask_st._st, audio_st._st
        va = _i32([9] * SB)
        if part == 2:
            return audio(st, ha, va)
        if part == 1:
            return state(st, h, va)
        x = _late(xin["m1"])
        m1 = torch.full((SB, 2, F), NAN, device=DEV)
        fl, va = _i32([START] * SB), _i32([9] * SB)
        _lib.check(lib().fsn_stream_step_slots(h, vp(x), vp(m1), fl, va, st))
        _mark("fsn_stream_step_slots")
        _overwrite(fl, [HOLD] * SB)
        outs += [m1.clone(), list(va)]
        x = _late(xin["m2"])
        v = C.c_int32(9)
        _lib.check(lib().fsn_stream_step(h, vp(x), vp(m1), C.byref(v), st))
        _mark("fsn_stream_step")
        outs += [m1.clone(), v.value]
        K = 7
        x = _late(xin["k7"])
        mk = torch.full((SB, 2, F, K), NAN, device=DEV)
        fl = _i32([STEP, HOLD, STEP, STEP])
        _lib.check(lib().fsn_stream_step_chunk(h, vp(x), K, vp(mk), fl, va, st))
        _mark("fsn_stream_step_chunk")
        _overwrite(fl, [HOLD, STEP, HOLD, HOLD])
        outs += [mk.clone(), list(va)]
        stage = torch.full((SB * F * K,), NAN, device=DEV)
        _lib.check(lib().fsn_stream_get_stage(h, b"fb_out", vp(stage), stage.numel(), st))
        _mark("fsn_stream_get_stage")
        v = stage.view(SB, F, K)                                     # the held slot 1's row holds no frame of the call
        outs.append(torch.cat((v[:1], v[2:])))
        return outs

    def state(st, h, va):
        outs = []
        nb = int(lib().fsn_stream_state_bytes(h))
        pay = torch.zeros((2, nb), dtype=torch.uint8, device=DEV)
        meta = (_lib.FsnSlotMeta * 2)()
        sl = _i32([2, 0])
        _lib.check(lib().fsn_stream_save_slots(h, 2, sl, vp(pay), meta, st))
        _mark("fsn_stream_save_slots")
        _overwrite(sl, [1, 3])
        x = _late(xin["k3"])
        mk3 = torch.full((SB, 2, F, 3), NAN, device=DEV)
        _lib.check(lib().fsn_stream_step_chunk(h, vp(x), 3, vp(mk3), _i32([STEP] * SB), va, st))
        _mark("fsn_stream_step_chunk")
        sl = _i32([3, 1])
        _lib.check(lib().fsn_stream_load_slots(h, 2, sl, vp(pay), meta, st))
        _mark("fsn_stream_load_slots")
        _overwrite(sl, [0, 2])
        x = _late(xin["k2"])
        mk2 = torch.full((SB, 2, F, 2), NAN, device=DEV)
        _lib.check(lib().fsn_stream_step_chunk(h, vp(x), 2, vp(mk2), _i32([STEP] * SB), va, st))
        _mark("fsn_stream_step_chunk")
        outs += [mk3.clone(), mk2.clone(), list(va), [(q.frames, q.tick, q.hops) for q in meta]]
        return outs

    def audio(st, ha, va):
        outs = []
        xa = _late(xin["a1"])
        ya = torch.full((SB, HOP), NAN, device=DEV)
        ma = torch.full((SB, 2, F), NAN, device=DEV)
        fl = _i32([START] * SB)
        _lib.check(lib().fsn_stream_step_audio_slots(ha, vp(xa), vp(ya), fl, va, vp(ma), st))
        _mark("fsn_stream_step_audio_slots")
        _overwrite(fl, [HOLD] * SB)
        outs += [ya.clone(), ma.clone(), list(va)]
        K = 4
        xa = _late(xin["a4"])
        ya = torch.full((SB, K * HOP), NAN, device=DEV)
        ma = torch.full((SB, 2, F, K), NAN, device=DEV)
        fl, hp, no = _i32([STEP, STEP, HOLD, FLUSH]), _i32([4, 2, 0, 3]), _i32([9] * SB)
        _lib.check(lib().fsn_stream_step_audio_chunk(ha, vp(xa), K, fl, hp, vp(ya), no, vp(ma), st))
        _mark("fsn_stream_step_audio_chunk")
        _overwrite(fl, [HOLD] * SB)
        _overwrite(hp, [1, 1, 1, 1])
        outs += [ya.clone(), ma.clone(), list(no)]
        S = 75
        xs = _late(xin["s75"])
        ys = torch.full((SB, S + (audio_st.look_ahead + 3) * HOP), NAN, device=DEV)
        fl, cn = _i32([STEP, FLUSH, START, FLUSH]), _i32([75, 10, 60, 0])
        _lib.check(lib().fsn_stream_step_audio_samples(ha, vp(xs), S, fl, cn, vp(ys), no, st))
        _mark("fsn_stream_step_audio_samples")
        _overwrite(fl, [HOLD] * SB)
        _overwrite(cn, [0] * SB)
        outs += [ys.clone(), list(no)]
        return outs
    return calls


def _stream_handles(m):
    return StreamingFullSubNet(m, SB, DEV), StreamingFullSubNet(m, SB, DEV)


@pytest.mark.parametrize("kind", KINDS)
def test_streaming_calls(kind, monkeypatch):
    """step, step_slots, step_chunk, save / load, get_stage and the three audio calls behind one gate"""
    P, Q = _pair(monkeypatch)
    a, b = _stream_handles(P)
    c, d = _stream_handles(Q)
    for part in (0, 1, 2):                                          # each within the queue depth of a handle's staging ring
        got = _run_gated(kind, _stream_calls(a, b, part), f"the streaming calls (part {part}) on the {kind} stream")
        _same(got, _truth(_stream_calls(c, d, part)), f"streaming {kind} part {part}")


CHUNK_C = 512


# (S, flags, counts) of the two steps on the first handle: every step completes 4 chunk rows (chunk k completes when a session reaches
# k H + C samples, H = C / 2; a FLUSH completes the rest), so every forward of the sequence has one geometry
CHUNK_STEPS = ((767, [START] * SB, [600, 700, 767, 512]), (168, [STEP, STEP, STEP, FLUSH], [168, 100, 1, 0]))


def _chunk_calls(cs, cs2):
    g = torch.Generator().manual_seed(70)
    xin = [(torch.randn((SB, S), generator=g) * 0.1).to(DEV) for S in (767, 168, 512)]

    def calls(s):
        st, outs = sp(s), []
        no = _i32([9] * SB)
        for k, (S, flags, counts) in enumerate(CHUNK_STEPS):
            x = _late(xin[k])
            y = torch.full((SB, S + CHUNK_C), NAN, device=DEV)
            fl, cn = _i32(flags), _i32(counts)
            _lib.check(lib().fsn_chunk_stream_step(cs._cs, vp(x), S, fl, cn, vp(y), no, st))
            _mark("fsn_chunk_stream_step")
            _overwrite(fl, [HOLD] * SB)
            _overwrite(cn, [0] * SB)
            outs += [y.clone(), list(no)]
        nb, _ = _lib.chunk_state_layout(CHUNK_C)
        pay = torch.zeros((2, nb), dtype=torch.uint8, device=DEV)
        meta = (_lib.FsnChunkSlotMeta * 2)()
        sl = _i32([1, 0])
        _lib.check(lib().fsn_chunk_stream_save_slots(cs._cs, 2, sl, vp(pay), meta, st))
        _mark("fsn_chunk_stream_save_slots")
        _overwrite(sl, [2, 3])
        sl = _i32([2, 1])
        _lib.check(lib().fsn_chunk_stream_load_slots(cs2._cs, 2, sl, vp(pay), meta, st))
        _mark("fsn_chunk_stream_load_slots")
        _overwrite(sl, [0, 3])
        x = _late(xin[2])                                           # sessions at 768 and 800 samples: 2 rows each
        y = torch.full((SB, 512 + CHUNK_C), NAN, device=DEV)
        _lib.check(lib().fsn_chunk_stream_step(cs2._cs, vp(x), 512, _i32([HOLD, STEP, FLUSH, HOLD]), _i32([0, 512, 0, 0]), vp(y),
                                               no, st))
        outs += [[m.samples for m in meta], [m.chunks for m in meta], y.clone(), list(no)]
        return outs
    return calls


@pytest.mark.parametrize("kind", KINDS)
def test_chunk_sessions(kind, monkeypatch):
    """fsn_chunk_stream_step with rows completing, save on one handle, load into another and step and FLUSH there, behind one gate"""
    P, Q = _pair(monkeypatch)
    got = _run_gated(kind, _chunk_calls(ChunkStream(P, SB, CHUNK_C, DEV), ChunkStream(P, SB, CHUNK_C, DEV)), f"the chunk calls ({kind})")
    want = _truth(_chunk_calls(ChunkStream(Q, SB, CHUNK_C, DEV), ChunkStream(Q, SB, CHUNK_C, DEV)))
    _same(got, want, f"chunk sessions {kind}")


# ---------------------------------------------------------------------------------------------------------------------------------
# metrics
@pytest.mark.parametrize("kind", KINDS)
def test_metrics(kind):
    """SI-SDR, STOI and SDR with the caller's workspace and inputs written behind the gate, lengths overwritten on return"""
    Bm, Lm, sr = 3, 12000, 16000
    ref = _wave(Bm, Lm, 80)
    est = (ref + 0.3 * _wave(Bm, Lm, 81)).contiguous()
    lens = [Lm, 9001, 4000]

    def calls(s):
        st, outs = sp(s), []
        r, e = _late(ref), _late(est)
        for name in ("si_sdr", "stoi", "sdr"):
            hl, nb = _i64(lens), C.c_int64()
            if name == "stoi":
                _lib.check(lib().fsn_metric_stoi_workspace(Bm, Lm, hl, sr, C.byref(nb)))
                _mark("fsn_metric_stoi_workspace")
            else:
                _lib.check(getattr(lib(), f"fsn_metric_{name}_workspace")(Bm, Lm, hl, C.byref(nb)))
            work = torch.full((nb.value,), 0xFF, dtype=torch.uint8, device=DEV)
            out = torch.full((Bm,), NAN, dtype=torch.float64, device=DEV)
            if name == "stoi":
                _lib.check(lib().fsn_metric_stoi(vp(r), vp(e), Bm, Lm, hl, sr, vp(work), nb.value, vp(out), st))
                _mark("fsn_metric_stoi")
            else:
                _lib.check(getattr(lib(), f"fsn_metric_{name}")(vp(r), vp(e), Bm, Lm, hl, vp(work), nb.value, vp(out), st))
            _overwrite(hl, [Lm, Lm, Lm])
            outs.append(out.clone())
        return outs
    _same(_run_gated(kind, calls, f"the metrics on the {kind} stream"), _truth(calls), f"metrics {kind}")


# ---------------------------------------------------------------------------------------------------------------------------------
# queue depth (the header's "Queue depth")
def test_queue_depth(monkeypatch):
    """QUEUE_DEPTH streaming calls return with the gate pending; the next one blocks until the GPU has reached the first"""
    P, Q = _pair(monkeypatch)
    st = StreamingFullSubNet(P, SB, DEV)
    twin = StreamingFullSubNet(Q, SB, DEV)
    xs = [_mag(3, 90 + k) for k in range(QUEUE_DEPTH + 1)]
    s = _stream("nonblocking")
    with torch.cuda.stream(s):
        st.step_chunk(xs[0], [START] * SB)                          # warm-up: the scratch of K = 3
    torch.cuda.synchronize()
    e = _gate(s)
    got = []
    with torch.cuda.stream(s):
        for k, x in enumerate(xs):
            got.append(st.step_chunk(_late(x), [START] * SB if k == 0 else [STEP] * SB))
            if k < QUEUE_DEPTH:
                _pending(e, f"streaming call {k + 1} of {QUEUE_DEPTH}")
    assert e.query(), f"call {QUEUE_DEPTH + 1} returned before the GPU reached call 1: the staging ring is deeper than {QUEUE_DEPTH}"
    torch.cuda.synchronize()
    want = [twin.step_chunk(x, [START] * SB if k == 0 else [STEP] * SB) for k, x in enumerate(xs)]
    _same(got, want, "queue depth")


# ---------------------------------------------------------------------------------------------------------------------------------
# creation under a busy default stream, destroy behind a gate
def test_create_under_busy_default_stream(monkeypatch):
    """Handles created while the legacy stream sleeps, then stepped on a non-blocking stream: create's zero-fills must not land on
    the handle's state after the first step.  If create returns with the gate pending, the first step runs on the side stream and
    only that stream is synchronised (no kernel of the handle is in flight when the legacy stream wakes); then every mask must
    equal a twin's.  A create that waits for the gate is reported, and only its results are checked."""
    P, Q = _pair(monkeypatch, FSN_NO_WS=1)
    side = _stream("nonblocking")
    xm = [_mag(5, 100 + k) for k in range(3)]
    xa = [(torch.randn((SB, 700), generator=torch.Generator().manual_seed(110 + k)) * 0.1).to(DEV) for k in range(3)]
    torch.cuda.synchronize()
    for what in ("stream", "chunk"):
        e = _gate(torch.cuda.default_stream(DEV))
        h = StreamingFullSubNet(P, SB, DEV) if what == "stream" else ChunkStream(P, SB, CHUNK_C, DEV)
        if e.query():
            print(f"fsn_{what if what == 'stream' else 'chunk_stream'}_create synchronised: results checked only")
        twin = StreamingFullSubNet(Q, SB, DEV) if what == "stream" else ChunkStream(Q, SB, CHUNK_C, DEV)
        got, want = [], []
        for k in range(3):
            if what == "stream":
                x = xm[k]
                with torch.cuda.stream(side):
                    got.append(h.step_chunk(x, [START] * SB if k == 0 else [STEP] * SB))
                want.append(twin.step_chunk(x, [START] * SB if k == 0 else [STEP] * SB))
            else:
                x = xa[k]
                fl = [START] * SB if k == 0 else [STEP] * SB
                with torch.cuda.stream(side):
                    got.append(h.step(x, [700] * SB, fl))
                want.append(twin.step(x, [700] * SB, fl))
            if k == 0:
                side.synchronize()
                torch.cuda.synchronize()
        torch.cuda.synchronize()
        _same(got, want, f"{what} handle created under a busy default stream")


def test_destroy_behind_gate(monkeypatch):
    """A streaming and a chunk handle destroyed while their last call is still behind a gate: the outputs read after the gate are
    the twin's"""
    P, Q = _pair(monkeypatch)
    s = _stream("nonblocking")
    x = _mag(4, 120)
    xa = (torch.randn((SB, 900), generator=torch.Generator().manual_seed(121)) * 0.1).to(DEV)
    res = []
    for m, gate in ((P, True), (Q, False)):
        st, cs = StreamingFullSubNet(m, SB, DEV), ChunkStream(m, SB, CHUNK_C, DEV)
        with torch.cuda.stream(s):
            st.step_chunk(x, [START] * SB)                          # warm-up
            cs.step(xa, [900] * SB, [START] * SB)
        torch.cuda.synchronize()
        if gate:
            _gate(s)
        with torch.cuda.stream(s):
            a = st.step_chunk(_late(x), [START] * SB)
            b = cs.step(_late(xa), [900] * SB, [START] * SB)
        st.close()
        cs.close()
        torch.cuda.synchronize()
        res.append([a, b])
    _same(res[0], res[1], "destroy behind a gate")


# ---------------------------------------------------------------------------------------------------------------------------------
# one handle, two streams
def _plain(m, x, s):
    with torch.cuda.stream(s):
        a = _late(x)
        o = torch.full((B, 2, F, T), NAN, device=DEV)
        _lib.check(lib().fsn_model_forward(m._handle, vp(a), None, None, B, T, vp(o), sp(s)))
        _mark("fsn_model_forward")
    return o


@pytest.mark.parametrize("gated", ["s1", "s2", "both"])
def test_cross_stream_plain_forwards(gated, monkeypatch):
    """Two plain forwards of one model from s1 and s2 (same shapes, different inputs).  "both" is the case that shows a missing
    order: with equal gates on both streams the two forwards would run at the same time in one workspace unless the second waits for
    the first.  With one gate ("s1", "s2") the ungated forward ends before the gated one starts, so those two only pin that the
    results and the non-blocking promise hold whichever stream arrives first."""
    P, Q = _pair(monkeypatch, FSN_NO_WS=1)
    x1, x2 = _spec(B, T, 130)[0], _spec(B, T, 131)[0]
    s1, s2 = _stream("nonblocking"), _stream("nonblocking")
    _plain(P, x1, s1)
    torch.cuda.synchronize()
    e = _gate(s1 if gated != "s2" else s2)
    if gated == "both":
        _gate(s2)
    o1 = _plain(P, x1, s1)
    o2 = _plain(P, x2, s2)
    _pending(e, "two plain forwards on two streams")
    torch.cuda.synchronize()
    with torch.no_grad():
        _same([o1, o2], [Q(x1), Q(x2)], f"cross-stream forwards, gate on {gated}")


def test_cross_stream_chunk_and_offline(monkeypatch):
    """A chunk session step on s1 and an offline audio call of the same model on s2, behind equal gates: they share the model's
    workspace, so without an order they would run at the same time in it.  The offline batch has the chunk rows' geometry (8 rows of
    C + 256 samples: 900 samples complete chunks 0 and 1 of each of the 4 sessions), so neither call reallocates"""
    P, Q = _pair(monkeypatch, FSN_NO_WS=1)
    cs, twin = ChunkStream(P, SB, CHUNK_C, DEV), ChunkStream(Q, SB, CHUNK_C, DEV)
    x = (torch.randn((SB, 900), generator=torch.Generator().manual_seed(140)) * 0.1).to(DEV)
    wave = _wave(2 * SB, CHUNK_C + 256, 141)
    s1, s2 = _stream("nonblocking"), _stream("nonblocking")

    def offline(m, s):
        with torch.cuda.stream(s):
            w, y = _late(wave), torch.full_like(wave, NAN)
            _lib.check(lib().fsn_model_enhance_audio(m._handle, vp(w), 2 * SB, CHUNK_C + 256, None, vp(y), sp(s)))
        return y
    with torch.cuda.stream(s1):
        cs.step(x, [900] * SB, [START] * SB)
    offline(P, s2)
    torch.cuda.synchronize()
    e = _gate(s1)
    _gate(s2)
    with torch.cuda.stream(s1):
        a = cs.step(_late(x), [900] * SB, [START] * SB)
    o = offline(P, s2)
    _pending(e, "a chunk step and an offline audio call on two streams")
    torch.cuda.synchronize()
    _same([a, o], [twin.step(x, [900] * SB, [START] * SB), offline(Q, torch.cuda.default_stream(DEV))], "chunk step and offline call")


def test_cross_stream_stage_and_state(monkeypatch):
    """get_stage on another stream right after a gated forward; a streaming save on s1 (gated) and a load on s2"""
    P, Q = _pair(monkeypatch, FSN_NO_WS=1)
    x = _spec(B, T, 150)[0]
    s1, s2 = _stream("nonblocking"), _stream("nonblocking")
    n = B * F * (T + P._cfg.look_ahead)

    def stage(m, s):
        with torch.cuda.stream(s):
            t = torch.full((n,), NAN, device=DEV)
            _lib.check(lib().fsn_model_get_stage(m._handle, b"fb_in", vp(t), n, sp(s)))
            _mark("fsn_model_get_stage")
        return t
    _plain(P, x, s1)
    stage(P, s2)
    torch.cuda.synchronize()
    _plain(P, _spec(B, T, 151)[0], s1)                               # the stage must come from the gated forward, not this one
    torch.cuda.synchronize()
    e = _gate(s1)
    _plain(P, x, s1)
    got = stage(P, s2)
    _pending(e, "get_stage on another stream")
    torch.cuda.synchronize()
    with torch.no_grad():
        Q(x)
    _same(got, stage(Q, torch.cuda.default_stream(DEV)), "get_stage across streams")

    st, twin = StreamingFullSubNet(P, SB, DEV), StreamingFullSubNet(Q, SB, DEV)
    for h in (st, twin):
        h.step_chunk(_mag(6, 160), [START] * SB)
        h.save_slots([0, 1])                                         # warm-up of the slot list buffers
        h.load_slots([2, 3], h.save_slots([0, 1]))
    x6, x2 = _mag(6, 161), _mag(2, 162)
    torch.cuda.synchronize()
    e = _gate(s1)
    with torch.cuda.stream(s1):
        st.step_chunk(_late(x6), [STEP] * SB)
        saved = st.save_slots([0, 1])
    with torch.cuda.stream(s2):
        st.load_slots([2, 3], saved)
        got = st.step_chunk(_late(x2), [STEP] * SB)
    _pending(e, "save on s1, load on s2")
    torch.cuda.synchronize()
    twin.step_chunk(x6, [STEP] * SB)
    twin.load_slots([2, 3], twin.save_slots([0, 1]))
    _same(got, twin.step_chunk(x2, [STEP] * SB), "save on s1, load on s2")


# ---------------------------------------------------------------------------------------------------------------------------------
# Python layer
def test_enhance_pipeline(monkeypatch):
    """EnhancePipeline with its main stream gated (its post and copy streams see the batches in order) equals the same pipeline run
    ungated on a twin"""
    P, Q = _pair(monkeypatch)
    Xs = []
    for k in range(3):
        mag, real, imag = _spec(2, 36, 170 + k)
        Xs.append(torch.complex(real[:, 0], imag[:, 0]))
    length = 35 * HOP

    def run(m, gate):
        pipe = EnhancePipeline(m, length, n_fft=2 * HOP, hop_length=HOP, win_length=2 * HOP)
        for X in Xs:                                                # warm-up: the ring's buffers
            pipe.push(X)
        pipe.flush()
        s = _stream("nonblocking")
        e = _gate(s) if gate else None
        with torch.cuda.stream(s):
            for X in Xs:
                pipe.push(_late(X))
            if e is not None:
                _pending(e, "EnhancePipeline.push")
            out = [r.clone() for r in pipe.flush()]
        torch.cuda.synchronize()
        return out
    _same(run(P, True), run(Q, False), "EnhancePipeline")


def test_tools_inference_streams(monkeypatch, tmp_path):
    """tools.inference with three batches in flight, one per CUDA stream and model replica, writes the same files, byte for byte, as
    with one stream (fullsubnet.Model at the reference's n_fft 512)"""
    from scipy.io import wavfile

    from fsnplus_b200.tools import inference as T
    rng = np.random.default_rng(6)
    noisy = tmp_path / "noisy"
    noisy.mkdir()
    for i, n in enumerate([8000, 12000, 8000, 5000, 9000, 12000, 7000]):
        wavfile.write(noisy / f"f{i}.wav", 16000, (rng.standard_normal(n) * 0.05).astype(np.float32))
    cfg = T.load_toml(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inference_reference.toml"))
    cfg["dataset"]["args"]["dataset_dir_list"] = [str(noisy)]
    cfg["inferencer"]["type"] = "full_band_crm_mask"
    mcfg = O.default_fsn_config()
    mcfg.update(num_freqs=257, sb_model_hidden_size=64, fb_model_hidden_size=64)
    p = O.make_params_fsn(mcfg, seed=7)
    models = [_model(Model, mcfg, p, monkeypatch) for _ in range(3)]
    out = {}
    for n in (1, 3):
        logs = []
        T.run(cfg, tmp_path / "x.tar", tmp_path / f"s{n}", batch_size=1, device=DEV, log=logs.append, model_and_epoch=(models[0], 1),
              streams=n, replicas=models[1:n])
        assert any(f"{n} stream(s)" in line for line in logs), logs
        out[n] = {f.name: f.read_bytes() for f in (tmp_path / f"s{n}" / "enhanced_0001").iterdir()}
    assert sorted(out[1]) == [f"f{i}.wav" for i in range(7)]
    for name in out[1]:
        assert out[3][name] == out[1][name], name
