"""Objective scores of enhanced speech on the device, one per clip (C ABI: fsn_metric_si_sdr / fsn_metric_stoi, DESIGN.md §3.20;
fsn_metric_sdr, §3.21).

    from fsnplus_b200 import metrics
    enhanced = model.enhance_audio(noisy, lengths)
    scores = metrics.stoi(clean, enhanced, sr=16000, lengths=lengths)     # float64 [B] on the same device

Each takes the reference and the estimate as CUDA float32 ``[B, L]`` tensors with optional per-clip ``lengths`` (clip b is the first
lengths[b] samples of its row, as ``model.enhance_audio`` takes them), or as two lists of 1-D CUDA tensors, packed here into that
form.  A clip's score does not depend on the rest of the batch.  The workspace is allocated by torch on the tensors' device, and the
call runs on its current stream.
"""
import ctypes as C

import torch

from . import _lib


def pack(clips):
    """A list of 1-D tensors on one device as a zero-padded float32 ``[B, max length]`` batch and the list of their lengths."""
    if len(clips) == 0:
        raise ValueError("no clips")
    lengths = [int(c.numel()) for c in clips]
    out = torch.zeros((len(clips), max(lengths)), dtype=torch.float32, device=clips[0].device)
    for i, c in enumerate(clips):
        if c.dim() != 1:
            raise ValueError(f"clip {i} has shape {tuple(c.shape)}; list inputs are 1-D waveforms")
        out[i, :lengths[i]] = c
    return out, lengths


def _batch(ref, est, lengths):
    if isinstance(ref, (list, tuple)) or isinstance(est, (list, tuple)):
        if not (isinstance(ref, (list, tuple)) and isinstance(est, (list, tuple))):
            raise TypeError("ref and est must both be lists of 1-D tensors or both be [B, L] tensors")
        if lengths is not None:
            raise ValueError("lengths is given by the clips themselves when ref and est are lists")
        if len(ref) != len(est):
            raise ValueError(f"{len(ref)} reference clips and {len(est)} estimates")
        for i, (r, e) in enumerate(zip(ref, est)):
            if r.numel() != e.numel():
                raise ValueError(f"clip {i}: the reference has {r.numel()} samples and the estimate {e.numel()}")
        ref, lengths = pack(list(ref))
        est, _ = pack(list(est))
    for name, t in (("ref", ref), ("est", est)):
        if not torch.is_tensor(t) or not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor (fsnplus_b200 has no CPU path)")
        if t.dtype != torch.float32 or t.dim() != 2:
            raise ValueError(f"{name} must be float32 [B, L], got {t.dtype} {tuple(t.shape)}")
    if ref.shape != est.shape or ref.device != est.device:
        raise ValueError(f"ref {tuple(ref.shape)} on {ref.device} and est {tuple(est.shape)} on {est.device} differ")
    B, L = ref.shape
    return ref.contiguous(), est.contiguous(), B, L, _lib.lengths_arg(lengths, B)


def _run(ref, est, lengths, workspace, call):
    ref, est, B, L, hl = _batch(ref, est, lengths)
    lib = _lib.load_library()
    nbytes = C.c_int64()
    _lib.check(workspace(lib, B, L, hl, C.byref(nbytes)))
    with torch.cuda.device(ref.device):
        work = torch.empty(max(nbytes.value, 1), dtype=torch.uint8, device=ref.device)
        out = torch.empty(B, dtype=torch.float64, device=ref.device)
        stream = C.c_void_p(torch.cuda.current_stream(ref.device).cuda_stream)
        _lib.check(call(lib, C.c_void_p(ref.data_ptr()), C.c_void_p(est.data_ptr()), B, L, hl, C.c_void_p(work.data_ptr()), nbytes.value,
                        C.c_void_p(out.data_ptr()), stream))
    return out


def si_sdr(ref, est, lengths=None):
    """Scale-invariant SDR in dB of each clip of ``est`` against ``ref``: 10 log10(|a r|^2 / |e - a r|^2), a = <r, e> / <r, r>,
    accumulated in float64.  Returns a float64 CUDA tensor [B]."""
    return _run(ref, est, lengths, lambda lib, B, L, hl, nb: lib.fsn_metric_si_sdr_workspace(B, L, hl, nb),
                lambda lib, r, e, B, L, hl, w, nw, o, s: lib.fsn_metric_si_sdr(r, e, B, L, hl, w, nw, o, s))


def stoi(ref, est, sr=16000, lengths=None):
    """Classic STOI of each clip of ``est`` against ``ref`` at ``sr`` Hz (8000 .. 48000), as pystoi's stoi(ref, est, sr,
    extended=False); a clip with fewer than 30 frames left after silent-frame removal scores 1e-5.  Returns a float64 CUDA tensor [B]."""
    sr = int(sr)
    return _run(ref, est, lengths, lambda lib, B, L, hl, nb: lib.fsn_metric_stoi_workspace(B, L, hl, sr, nb),
                lambda lib, r, e, B, L, hl, w, nw, o, s: lib.fsn_metric_stoi(r, e, B, L, hl, sr, w, nw, o, s))


def sdr(ref, est, lengths=None):
    """BSS Eval v3 SDR in dB of each clip of ``est`` against ``ref``, as mir_eval's bss_eval_sources scores one source: the
    projection P of ``est`` onto the 512 delayed copies of ``ref`` (a 512-tap distortion filter, one Toeplitz solve per clip) and
    10 log10(|P|^2 / |e' - P|^2), all in float64.  No sample rate: SDR does not depend on it.  A silent reference or estimate gives
    NaN; scores above 100 dB measure rounding noise.  Returns a float64 CUDA tensor [B]."""
    return _run(ref, est, lengths, lambda lib, B, L, hl, nb: lib.fsn_metric_sdr_workspace(B, L, hl, nb),
                lambda lib, r, e, B, L, hl, w, nw, o, s: lib.fsn_metric_sdr(r, e, B, L, hl, w, nw, o, s))
