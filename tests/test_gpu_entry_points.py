"""The ten offline entry points of the C ABI share one argument check (fsn_api.cu: check_batch) and one setup.

  * every single-fault call of every entry point returns its code and message;
  * the host-buffer calls refuse a bad batch or frame count (zero or negative) with FSN_EINVAL before they stage or allocate anything;
  * the sub-band test hook decides its chained launches from its own batch, so it computes the same bits whatever forward ran before.
"""
import ctypes as C

import pytest
import torch

from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EINVAL, ESTATE = -1, -3
F, T = 33, 16


def _model(cfg=None):
    from fsnplus_b200.model import FullSubNet_Plus
    if cfg is None:
        cfg = O.default_plus_config()
        cfg.update(num_freqs=F, sb_num_neighbors=3, sb_model_hidden_size=64)
    m = FullSubNet_Plus(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in O.make_params_plus(cfg, seed=0).items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    return m


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p()


def _calls(lib, dev, host, s):
    """entry point -> call(handle, **fault) with every argument valid unless the fault names it"""
    def spec(fn, x, out, ragged=False):
        def call(h, mag=x, real=x, imag=x, B=1, T=T, frames=None, out=out):
            frames = frames or (T,)
            fr = [(C.c_int32 * len(frames))(*frames)] if ragged else []
            return fn(h, _p(mag), _p(real), _p(imag), B, T, *fr, _p(out), s)
        return call

    x = torch.rand(1, 1, F, T, device=dev) + 0.1
    mask, enh = torch.empty(1, 2, F, T, device=dev), torch.empty(1, F, T, dtype=torch.complex64, device=dev)
    hx = host[0]

    def audio(h, wave=torch.zeros(1, 256, device=dev), B=1, L=256, lengths=None, out=torch.empty(1, 256, device=dev)):
        hl = (C.c_int64 * len(lengths))(*lengths) if lengths is not None else None
        return lib.fsn_model_enhance_audio(h, _p(wave), B, L, hl, _p(out), s)

    isb = 2 * 3 + 1 + 3
    xr = torch.zeros(F, isb, T + 2, device=dev)

    def hook(h, x=xr, B=1, T=T, Tw=0, frames=None, out=mask):
        fr = (C.c_int32 * len(frames))(*frames) if frames is not None else None
        return lib.fsn_model_sb_forward(h, _p(x), B, T, Tw, fr, _p(out), None, None, None, s)

    return {
        "forward": spec(lib.fsn_model_forward, x, mask),
        "forward_enhance": spec(lib.fsn_model_forward_enhance, x, enh),
        "forward_ragged": spec(lib.fsn_model_forward_ragged, x, mask, ragged=True),
        "forward_enhance_ragged": spec(lib.fsn_model_forward_enhance_ragged, x, enh, ragged=True),
        "submit": spec(lib.fsn_model_submit, x, mask),
        "submit_enhance": spec(lib.fsn_model_submit_enhance, x, enh),
        "forward_host": spec(lib.fsn_model_forward_host, hx, host[1]),
        "forward_host_async": spec(lib.fsn_model_forward_host_async, hx, host[1]),
        "enhance_audio": audio,
        "sb_forward": hook,
    }


SPECTRAL = ["forward", "forward_enhance", "forward_ragged", "forward_enhance_ragged", "submit", "submit_enhance", "forward_host",
            "forward_host_async"]
# (entry points, fault, code, message needle)
FAULTS = [(SPECTRAL, dict(h=None), EINVAL, b"null argument"),
          (SPECTRAL, dict(mag=None), EINVAL, b"null argument"),
          (SPECTRAL, dict(out=None), EINVAL, b"null argument"),
          (SPECTRAL, dict(B=0), EINVAL, b"bad batch/frames"),
          (SPECTRAL, dict(T=0), EINVAL, b"bad batch/frames"),
          (SPECTRAL, dict(B=-1), EINVAL, b"bad batch/frames"),
          (SPECTRAL, dict(T=-1), EINVAL, b"bad batch/frames"),
          (SPECTRAL, dict(T=1), EINVAL, b"shorter than the TSSE kernel size"),
          (SPECTRAL, "unfinalized", ESTATE, b"fsn_model_finalize has not been called"),
          (["forward", "submit"], dict(real=None), EINVAL, b"FullSubNet_Plus.forward needs mag, real and imag"),
          (["forward_enhance", "forward_enhance_ragged", "submit_enhance"], dict(imag=None), EINVAL,
           b"the enhanced-spectrum output needs the noisy real and imaginary planes"),
          (["forward_host", "forward_host_async"], dict(real=None), EINVAL, b"missing input 1"),
          (["forward_ragged", "forward_enhance_ragged"], dict(frames=(0,)), EINVAL, b"frames[0] = 0 is outside 1..T = 16"),
          (["forward_ragged", "forward_enhance_ragged"], dict(frames=(T + 1,)), EINVAL, b"is outside 1..T"),
          (["forward_ragged", "forward_enhance_ragged"], dict(frames=(5,)), EINVAL, b"shorter than the TSSE kernel size 10"),
          (["enhance_audio"], dict(h=None), EINVAL, b"m is null"),
          (["enhance_audio"], dict(wave=None), EINVAL, b"d_wave is null"),
          (["enhance_audio"], dict(out=None), EINVAL, b"d_out is null"),
          (["enhance_audio"], dict(B=0), EINVAL, b"the batch needs at least one clip"),
          (["enhance_audio"], dict(L=0), EINVAL, b"the row length must be"),
          (["enhance_audio"], dict(lengths=(16,)), EINVAL, b"more than n_fft / 2"),
          (["enhance_audio"], dict(lengths=(300,)), EINVAL, b"exceeds the row length L = 256"),
          (["enhance_audio"], dict(L=64, lengths=(64,)), EINVAL, b"shorter than the TSSE kernel size"),
          (["enhance_audio"], "unfinalized", ESTATE, b"fsn_model_finalize has not been called"),
          (["sb_forward"], dict(h=None), EINVAL, b"null argument"),
          (["sb_forward"], dict(x=None), EINVAL, b"null argument"),
          (["sb_forward"], dict(out=None), EINVAL, b"null argument"),
          (["sb_forward"], dict(B=0), EINVAL, b"bad batch/frames"),
          (["sb_forward"], dict(Tw=48), EINVAL, b"multiple of 32 frames"),
          (["sb_forward"], dict(frames=(0,)), EINVAL, b"is outside 1..T"),
          (["sb_forward"], "unfinalized", ESTATE, b"fsn_model_finalize has not been called")]


def test_single_fault_table(built_lib):
    """Every entry point: a valid call succeeds; each single fault returns its code and message."""
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    m = _model()
    host = (torch.rand(1, 1, F, T).pin_memory() + 0.1, torch.empty(1, 2, F, T).pin_memory())
    s = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    calls = _calls(lib, DEV, host, s)
    raw = C.c_void_p()
    _lib.check(lib.fsn_model_create(C.byref(m._cfg), C.byref(raw)))
    try:
        for name, call in calls.items():
            assert call(m._handle) == 0, (name, lib.fsn_last_error())
        lib.fsn_model_sync_host(m._handle)
        torch.cuda.synchronize()
        n = 0
        for names, fault, code, needle in FAULTS:
            for name in names:
                rc = calls[name](raw) if fault == "unfinalized" else calls[name](**{"h": m._handle, **fault})
                msg = lib.fsn_last_error()
                assert rc == code and needle in msg, (name, fault, rc, msg)
                n += 1
        print(f"\n[entry points] {len(calls)} entry points, {n} single-fault calls")
    finally:
        lib.fsn_model_destroy(raw)
        lib.fsn_model_sync_host(m._handle)
        torch.cuda.synchronize()


@pytest.mark.parametrize("pipelined", [False, True])
@pytest.mark.parametrize("B,T_", [(0, T), (-1, T), (1, 0), (1, -1)])
def test_host_calls_check_before_staging(built_lib, pipelined, B, T_):
    """A bad batch or frame count: FSN_EINVAL "bad batch/frames" before any staging allocation, copy or synchronisation."""
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    m = _model()
    h = torch.zeros(1, 1, F, T).pin_memory()
    out = torch.empty(1, 2, F, T).pin_memory()
    before = lib.fsn_model_workspace_bytes(m._handle)
    fn = lib.fsn_model_forward_host_async if pipelined else lib.fsn_model_forward_host
    s = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    rc = fn(m._handle, _p(h), _p(h), _p(h), B, T_, _p(out), s)
    assert rc == EINVAL and b"bad batch/frames" in lib.fsn_last_error(), (rc, lib.fsn_last_error())
    assert lib.fsn_model_workspace_bytes(m._handle) == before


def test_hook_follows_its_own_batch(built_lib):
    """The hook after a forward of one clip (chained launches on) and after one of 64 clips (off at num_freqs 257): the same bits."""
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    cfg = O.default_plus_config()
    m = _model(cfg)
    Fd, Td, isb = cfg["num_freqs"], 24, 2 * cfg["sb_num_neighbors"] + 1 + 3
    g = torch.Generator(device=DEV).manual_seed(3)
    x = torch.randn(2 * Fd, isb, Td + cfg["look_ahead"], device=DEV, generator=g).half().float()
    s = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)

    def hook():
        out = torch.full((2, 2, Fd, Td), float("nan"), device=DEV)
        _lib.check(lib.fsn_model_sb_forward(m._handle, _p(x), 2, Td, 0, None, _p(out), None, None, None, s))
        torch.cuda.synchronize()
        return out

    outs = []
    for B in (1, 64):
        mag = torch.rand(B, 1, Fd, Td, device=DEV) + 0.1
        m(mag, mag, mag)
        outs.append(hook())
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])
