"""Frame-by-frame (causal) inference for BASELINE config #4: ``fsnplus_b200.model.Model`` (the original FullSubNet) with a
cumulative norm.  FullSubNet+ itself cannot stream: its TSSE attention pools over all time, its TCN is non-causal and
offline_laplace_norm uses the utterance mean (SURVEY.md 0.5).

The state carried between frames (running norm sums, (h, c) of both LSTMs) lives on the device behind the C ABI
(``fsn_stream_*`` in include/fsnplus_b200.h).  Algorithmic latency = look_ahead frames: the mask of frame n - look_ahead is
produced when frame n arrives, exactly as the reference's right zero-padding + output shift (fullsubnet.py:81,117) implies.

Independent sessions share one handle through ``step_slots``: each of the B slots serves its own session, which starts, pauses
and ends on its own schedule (flags HOLD / STEP / START per slot and tick, DESIGN.md §3.9).
"""
import ctypes as C

import torch

from . import _lib

HOLD, STEP, START = 0, 1, 2            # FSN_SLOT_* of include/fsnplus_b200.h


class StreamingFullSubNet:
    def __init__(self, model, batch_size=1, device="cuda:0"):
        self.model, self.B, self.device = model, batch_size, torch.device(device)
        self.look_ahead = model.look_ahead
        with torch.cuda.device(self.device):
            self.lib = model._ensure_handle(self.device)
            h = C.c_void_p()
            _lib.check(self.lib.fsn_stream_create(model._handle, batch_size, C.byref(h)))
        self._st = h
        self.F = model._cfg.num_freqs

    def step(self, mag_frame):
        """mag_frame [B, F] float32 CUDA -> mask [B, 2, F] of frame (n - look_ahead), or None while the look-ahead fills."""
        assert mag_frame.shape == (self.B, self.F) and mag_frame.is_cuda
        x = mag_frame.contiguous().float()
        out = torch.empty((self.B, 2, self.F), dtype=torch.float32, device=self.device)
        valid = C.c_int32(0)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_step(self._st, C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), C.byref(valid), stream))
        return out if valid.value else None

    def step_slots(self, mag_frame, flags):
        """One tick of independent sessions.  mag_frame [B, F] float32 CUDA (rows of held slots are never read); flags: B values of
        HOLD / STEP / START (a sequence or a CPU integer tensor).  Returns (mask [B, 2, F], valid bool CPU tensor [B]): valid[b] when
        slot b stepped and has consumed more than look_ahead frames since its START, its mask row being that of frame n_b - look_ahead;
        every other row is zero.  End a session with look_ahead zero frames stepped, then HOLD the slot until a START reuses it."""
        assert mag_frame.shape == (self.B, self.F) and mag_frame.is_cuda
        f = torch.as_tensor(flags, dtype=torch.int32)
        assert f.device.type == "cpu" and f.shape == (self.B,), "flags: B host values"
        f = f.contiguous()
        x = mag_frame.contiguous().float()
        out = torch.empty((self.B, 2, self.F), dtype=torch.float32, device=self.device)
        valid = torch.zeros(self.B, dtype=torch.int32)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_step_slots(self._st, C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()),
                                                      C.c_void_p(f.data_ptr()), C.c_void_p(valid.data_ptr()), stream))
        return out, valid.bool()

    def flush(self):
        """Feed look_ahead zero frames (the reference's right padding) and return the remaining masks."""
        z = torch.zeros((self.B, self.F), dtype=torch.float32, device=self.device)
        return [self.step(z) for _ in range(self.look_ahead)]

    def close(self):
        if self._st is not None:
            self.lib.fsn_stream_destroy(self._st)
            self._st = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
