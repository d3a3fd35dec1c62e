"""Frame-by-frame (causal) inference for BASELINE config #4: ``fsnplus_b200.model.Model`` (the original FullSubNet) with a
cumulative norm.  FullSubNet+ itself cannot stream: its TSSE attention pools over all time, its TCN is non-causal and
offline_laplace_norm uses the utterance mean (SURVEY.md 0.5).

The state carried between frames (running norm sums, (h, c) of both LSTMs) lives on the device behind the C ABI
(``fsn_stream_*`` in include/fsnplus_b200.h).  Algorithmic latency = look_ahead frames: the mask of frame n - look_ahead is
produced when frame n arrives, exactly as the reference's right zero-padding + output shift (fullsubnet.py:81,117) implies.

Independent sessions share one handle through ``step_slots``: each of the B slots serves its own session, which starts, pauses
and ends on its own schedule (flags HOLD / STEP / START per slot and tick, DESIGN.md §3.9).

``step_chunk`` advances the same sessions K frames per call, with the sub-band LSTM on the offline forward's tensor-core kernels
where the configuration takes them (DESIGN.md §3.13); it mixes freely with ``step_slots`` on one handle.

``step_audio`` serves the same sessions with audio in and out: one hop of samples per slot and tick goes in, one hop of enhanced
audio comes out, with the STFT, the cIRM and the overlap-add iSTFT on the device (flag FLUSH ends a session, DESIGN.md §3.10).
``step_audio_chunk`` advances audio sessions many hops per call: each slot brings its own number of hops, and the call equals that
many ``step_audio`` ticks on the slot (DESIGN.md §3.14).  ``step_audio_samples`` takes any number of samples per slot and call and
ends a session at any length, with ``ChunkStream.step``'s arguments (DESIGN.md §3.19).  A handle serves either the mask calls or the
audio calls.

``save_slots`` / ``load_slots`` park, resume and move sessions (DESIGN.md §3.11): a ``SessionState`` holds the saved state of some
slots, and loading it into any slot of a handle of the same model -- this one, one with another B, or one on another GPU -- continues
each session where it was saved.

``ChunkStream`` serves live audio to the models that cannot stream frame by frame -- FullSubNet+ and ``Model`` with an offline norm --
by the reference's overlapped-chunk inferencer: chunks of C samples with 50 % overlap, each enhanced by the offline audio call, the
halves cross-faded with a Hann window; the latency is C / 2 to C samples (DESIGN.md §3.16).  Its ``save_slots`` / ``load_slots`` park,
resume and move those sessions between chunk handles of the same C, whatever their model (DESIGN.md §3.17).
"""
import ctypes as C

import torch

from . import _lib

HOLD, STEP, START, FLUSH = 0, 1, 2, 3  # FSN_SLOT_* of include/fsnplus_b200.h (FLUSH: audio call only)


def _slot_array(slots):
    s = torch.as_tensor(slots, dtype=torch.int32).reshape(-1).contiguous()
    assert s.device.type == "cpu" and s.numel() >= 1, "slots: host slot indices"
    return s


class SessionState:
    """Saved streaming sessions: ``payload`` [n, stride] uint8 (a CUDA tensor, or pinned host memory after ``.to("cpu")``) and
    ``meta``, a ctypes array of n ``fsn_slot_meta`` (StreamingFullSubNet) or ``fsn_chunk_slot_meta`` (ChunkStream), whose element
    type the selections and copies keep.  ``len()``, indexing / selection (``state[2]``, ``state[[0, 3]]``, slices) and
    ``.to(device)`` return new SessionState objects; the payload format is that of this library version only."""

    def __init__(self, payload, meta):
        assert payload.dtype == torch.uint8 and payload.dim() == 2 and payload.shape[0] == len(meta)
        self.payload, self.meta = payload, meta

    def __len__(self):
        return self.payload.shape[0]

    @property
    def device(self):
        return self.payload.device

    @property
    def _meta_type(self):
        return self.meta._type_

    def __getitem__(self, idx):
        if isinstance(idx, slice):
            ids = list(range(len(self)))[idx]
        elif torch.is_tensor(idx):
            ids = [int(i) for i in idx.reshape(-1).tolist()]
        elif isinstance(idx, int):
            ids = [idx]
        else:
            ids = [int(i) for i in idx]
        ids = [i + len(self) if i < 0 else i for i in ids]
        if any(i < 0 or i >= len(self) for i in ids):
            raise IndexError(f"session index out of range (0..{len(self) - 1})")
        meta = (self._meta_type * len(ids))(*[self.meta[i] for i in ids])
        sel = torch.tensor(ids, dtype=torch.long, device=self.payload.device)
        payload = self.payload.index_select(0, sel)
        if payload.device.type == "cpu" and self.payload.is_pinned():
            payload = payload.pin_memory()
        return SessionState(payload, meta)

    def to(self, device):
        """A copy on `device`: "cpu" gives pinned host memory, a CUDA device a plain copy (this object itself if it is there already)."""
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        if device == self.payload.device:
            return self
        if device.type == "cpu":
            payload = torch.empty(self.payload.shape, dtype=torch.uint8).pin_memory()
            payload.copy_(self.payload)
        else:
            payload = self.payload.to(device)
        return SessionState(payload, (self._meta_type * len(self))(*self.meta))


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
        _, meta_bytes = _lib.state_layout(model._cfg, _lib.STATE_MODE_MASK)
        if meta_bytes != C.sizeof(_lib.FsnSlotMeta):
            raise _lib.FsnError(f"fsn_slot_meta is {meta_bytes} bytes in the library, {C.sizeof(_lib.FsnSlotMeta)} in the ctypes mirror")

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

    def step_chunk(self, mag, flags):
        """K ticks of independent sessions in one call (DESIGN.md §3.13).  mag [B, F, K] float32 CUDA: each slot's next K frames
        (rows of held slots are never read); flags: B values of HOLD / STEP / START, which STEP or START K frames.  Returns (mask
        [B, 2, F, K], nvalid int32 CPU tensor [B]): column k of slot b is the mask of its frame n_b + k - look_ahead (n_b: frames
        consumed since its START before this call), and the nvalid[b] valid columns are the trailing ones; every other column and
        every held row is zero."""
        assert mag.dim() == 3 and mag.shape[:2] == (self.B, self.F) and mag.is_cuda
        K = mag.shape[2]
        f = torch.as_tensor(flags, dtype=torch.int32)
        assert f.device.type == "cpu" and f.shape == (self.B,), "flags: B host values"
        f = f.contiguous()
        x = mag.contiguous().float()
        out = torch.empty((self.B, 2, self.F, K), dtype=torch.float32, device=self.device)
        nvalid = torch.zeros(self.B, dtype=torch.int32)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_step_chunk(self._st, C.c_void_p(x.data_ptr()), K, C.c_void_p(out.data_ptr()),
                                                      C.c_void_p(f.data_ptr()), C.c_void_p(nvalid.data_ptr()), stream))
        return out, nvalid

    @property
    def hop(self):
        """Samples per hop of the audio call: n_fft / 2 = num_freqs - 1."""
        return self.F - 1

    def step_audio(self, samples, flags, return_mask=False):
        """One tick of independent audio sessions.  samples [B, hop] float32 CUDA: one hop per slot (rows of HOLD and FLUSH slots are
        never read); flags: B values of HOLD / STEP / START / FLUSH.  Returns (audio [B, hop], valid bool CPU tensor [B]), plus the
        masks [B, 2, F] with return_mask: valid[b] when audio[b] is hop q of the slot's session, which comes out at the slot's tick
        q + look_ahead + 2 (HOLD ticks not counted); every other row is zero.  A session of K >= 2 hops ends with look_ahead + 2
        FLUSH ticks (other lengths: ``step_audio_samples``); at slot tick k the mask row is that of frame k - look_ahead - 1 (zero before frame 0)."""
        assert samples.shape == (self.B, self.hop) and samples.is_cuda
        f = torch.as_tensor(flags, dtype=torch.int32)
        assert f.device.type == "cpu" and f.shape == (self.B,), "flags: B host values"
        f = f.contiguous()
        x = samples.contiguous().float()
        out = torch.empty((self.B, self.hop), dtype=torch.float32, device=self.device)
        mask = torch.empty((self.B, 2, self.F), dtype=torch.float32, device=self.device) if return_mask else None
        valid = torch.zeros(self.B, dtype=torch.int32)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_step_audio_slots(self._st, C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()),
                                                            C.c_void_p(f.data_ptr()), C.c_void_p(valid.data_ptr()),
                                                            C.c_void_p(mask.data_ptr() if return_mask else None), stream))
        return (out, valid.bool(), mask) if return_mask else (out, valid.bool())

    def step_audio_chunk(self, samples, flags, hops, return_mask=False):
        """Up to K hops per slot in one call (DESIGN.md §3.14).  samples [B, K hop] float32 CUDA: slot b's hops[b] new hops at the front
        of its row (nothing else is read); flags, hops: B values each (sequences or CPU integer tensors).  For slot b the call is K
        ``step_audio`` ticks: HOLD x K; START, STEP x (n - 1), HOLD...; STEP x n, HOLD...; or STEP x n, FLUSH... (n = hops[b], 1..K,
        or 0..K for FLUSH).  Returns (audio [B, K hop], nout int32 CPU tensor [B]): the nout[b] hops the ticks emitted at the front of
        row b, zero after them; plus the masks [B, 2, F, K] with return_mask, column i being tick i's mask row."""
        assert samples.dim() == 2 and samples.shape[0] == self.B and samples.shape[1] % self.hop == 0 and samples.is_cuda
        K = samples.shape[1] // self.hop
        f = torch.as_tensor(flags, dtype=torch.int32)
        n = torch.as_tensor(hops, dtype=torch.int32)
        assert f.device.type == "cpu" and f.shape == (self.B,), "flags: B host values"
        assert n.device.type == "cpu" and n.shape == (self.B,), "hops: B host values"
        f, n = f.contiguous(), n.contiguous()
        x = samples.contiguous().float()
        out = torch.empty((self.B, K * self.hop), dtype=torch.float32, device=self.device)
        mask = torch.empty((self.B, 2, self.F, K), dtype=torch.float32, device=self.device) if return_mask else None
        nout = torch.zeros(self.B, dtype=torch.int32)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_step_audio_chunk(self._st, C.c_void_p(x.data_ptr()), K, C.c_void_p(f.data_ptr()),
                                                            C.c_void_p(n.data_ptr()), C.c_void_p(out.data_ptr()),
                                                            C.c_void_p(nout.data_ptr()),
                                                            C.c_void_p(mask.data_ptr() if return_mask else None), stream))
        return (out, nout, mask) if return_mask else (out, nout)

    def step_audio_samples(self, samples, counts, flags):
        """Any number of samples per slot (DESIGN.md §3.19; C: fsn_stream_step_audio_samples).  samples [B, S] float32 CUDA: slot b's
        counts[b] new samples at the front of its row (nothing else is read); counts, flags: B values each (sequences or CPU integer
        tensors), flags HOLD / STEP / START / FLUSH (FLUSH consumes, then ends the session).  Returns (out [B, S + (look_ahead + 3)
        hop], nout int32 CPU tensor [B]): slot b's nout[b] newly final samples at the front of its row, zero after them.  A session's
        outputs concatenated over its calls are its offline enhancement (``enhance_audio``), as long as its input."""
        assert samples.dim() == 2 and samples.shape[0] == self.B and samples.is_cuda
        S = samples.shape[1]
        f = torch.as_tensor(flags, dtype=torch.int32)
        n = torch.as_tensor(counts, dtype=torch.int32)
        assert f.device.type == "cpu" and f.shape == (self.B,), "flags: B host values"
        assert n.device.type == "cpu" and n.shape == (self.B,), "counts: B host values"
        f, n = f.contiguous(), n.contiguous()
        x = samples.contiguous().float()
        out = torch.empty((self.B, S + (self.look_ahead + 3) * self.hop), dtype=torch.float32, device=self.device)
        nout = torch.zeros(self.B, dtype=torch.int32)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_step_audio_samples(self._st, C.c_void_p(x.data_ptr()), S, C.c_void_p(f.data_ptr()),
                                                              C.c_void_p(n.data_ptr()), C.c_void_p(out.data_ptr()),
                                                              C.c_void_p(nout.data_ptr()), stream))
        return out, nout

    def _slot_array(self, slots):
        return _slot_array(slots)

    def save_slots(self, slots):
        """Snapshot the sessions of `slots` (a sequence or a CPU integer tensor) into a SessionState on this handle's device.  The slots
        are unchanged: they may keep stepping (a fork) or START other sessions.  Ordered on the current stream like the step calls."""
        s = self._slot_array(slots)
        n = s.numel()
        with torch.cuda.device(self.device):
            stride = int(self.lib.fsn_stream_state_bytes(self._st))
            _lib.check(stride if stride < 0 else 0)
            payload = torch.empty((n, stride), dtype=torch.uint8, device=self.device)
            meta = (_lib.FsnSlotMeta * n)()
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_save_slots(self._st, n, C.c_void_p(s.data_ptr()), C.c_void_p(payload.data_ptr()), meta, stream))
        return SessionState(payload, meta)

    def load_slots(self, slots, state):
        """Load session i of `state` into slot slots[i] (distinct slots), replacing a START: the slot's next tick continues the session
        where it was saved.  The state is copied to this handle's device first if it lives elsewhere."""
        s = self._slot_array(slots)
        assert s.numel() == len(state), f"{s.numel()} slots for {len(state)} sessions"
        state = state.to(self.device)
        payload = state.payload.contiguous()
        if payload.data_ptr() % 256:
            payload = payload.clone()
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_load_slots(self._st, s.numel(), C.c_void_p(s.data_ptr()), C.c_void_p(payload.data_ptr()),
                                                      state.meta, stream))

    def set_atten_lim(self, slots, db):
        """Attenuation limit of `slots` (a sequence or a CPU integer tensor) in dB -- one number for all of them or one per slot,
        float('inf') = no limit (DESIGN.md §3.18; C: fsn_stream_set_atten_lim).  ``step_audio`` / ``step_audio_chunk`` apply it to every
        frame they synthesise from now on; the masks are unchanged.  The limit belongs to the slot, not to the session: START and
        ``load_slots`` keep it, and ``save_slots`` does not carry it."""
        s = self._slot_array(slots)
        _lib.check(self.lib.fsn_stream_set_atten_lim(self._st, s.numel(), C.cast(s.data_ptr(), C.POINTER(C.c_int32)),
                                                     _lib.atten_arg(db, s.numel())))

    def get_stage(self, name, shape):
        """Test hook (C: fsn_stream_get_stage): a float32 CUDA tensor of `shape` with the intermediate `name` ("fb_in", "fb_out",
        "sb_img", "mag", "mask", "spec") of the last call that stepped the model, ordered on the current stream like the step calls.
        "spec" is complex: `shape` is its [B, K, F] and the tensor complex64."""
        cplx = name == "spec"
        t = torch.empty(tuple(shape) + ((2,) if cplx else ()), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_stream_get_stage(self._st, name.encode(), C.c_void_p(t.data_ptr()), t.numel(), stream))
        if cplx:
            return torch.view_as_complex(t)
        return t

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


class ChunkStream:
    """Live audio for any model ``enhance_audio`` runs -- FullSubNet+ (any attention, norm or sub-band model) and ``Model`` with any
    norm -- by the reference's overlapped-chunk inferencer (DESIGN.md §3.16; C: ``fsn_chunk_stream_*``).  Each of the B slots serves
    its own session: its input is cut into chunks of ``chunk_samples`` (C, even) with 50 % overlap and 256 samples of pre-context,
    each chunk is enhanced by the offline audio call, and the halves are cross-faded with a periodic Hann window of C.  Every chunk
    completed by every slot in one ``step`` runs as one batch.  The output lags the input by C / 2 to C samples."""

    def __init__(self, model, batch_size=1, chunk_samples=16000, device="cuda:0"):
        self.model, self.B, self.C, self.device = model, batch_size, chunk_samples, torch.device(device)
        model._check_call()
        with torch.cuda.device(self.device):
            self.lib = model._ensure_handle(self.device)
            h = C.c_void_p()
            _lib.check(self.lib.fsn_chunk_stream_create(model._handle, batch_size, chunk_samples, C.byref(h)))
        self._cs = h

    def step(self, samples, counts, flags):
        """One call.  samples [B, S] float32 CUDA: slot b's counts[b] new samples at the front of its row (nothing else is read);
        counts, flags: B values each (sequences or CPU integer tensors), flags HOLD / STEP / START / FLUSH (FLUSH consumes, then ends
        the session).  Returns (out [B, S + C], nout int32 CPU tensor [B]): slot b's nout[b] newly final output samples at the front
        of its row, zero after them.  A session's outputs concatenated over its calls are its enhanced audio, as long as its input."""
        assert samples.dim() == 2 and samples.shape[0] == self.B and samples.is_cuda
        S = samples.shape[1]
        f = torch.as_tensor(flags, dtype=torch.int32)
        n = torch.as_tensor(counts, dtype=torch.int32)
        assert f.device.type == "cpu" and f.shape == (self.B,), "flags: B host values"
        assert n.device.type == "cpu" and n.shape == (self.B,), "counts: B host values"
        f, n = f.contiguous(), n.contiguous()
        x = samples.contiguous().float()
        out = torch.empty((self.B, S + self.C), dtype=torch.float32, device=self.device)
        nout = torch.zeros(self.B, dtype=torch.int32)
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_chunk_stream_step(self._cs, C.c_void_p(x.data_ptr()), S, C.c_void_p(f.data_ptr()),
                                                      C.c_void_p(n.data_ptr()), C.c_void_p(out.data_ptr()),
                                                      C.c_void_p(nout.data_ptr()), stream))
        return out, nout

    def save_slots(self, slots):
        """Snapshot the sessions of `slots` (a sequence or a CPU integer tensor) into a SessionState on this handle's device (DESIGN.md
        §3.17).  The slots are unchanged: they may keep stepping (a fork) or START other sessions; a slot without a session saves as
        samples = -1.  Ordered on the current stream like ``step``."""
        s = _slot_array(slots)
        n = s.numel()
        stride, _ = _lib.chunk_state_layout(self.C)
        payload = torch.empty((n, stride), dtype=torch.uint8, device=self.device)
        meta = (_lib.FsnChunkSlotMeta * n)()
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_chunk_stream_save_slots(self._cs, n, C.c_void_p(s.data_ptr()), C.c_void_p(payload.data_ptr()), meta,
                                                            stream))
        return SessionState(payload, meta)

    def load_slots(self, slots, state):
        """Load session i of `state` into slot slots[i] (distinct slots), replacing a START: the slot's next STEP or FLUSH continues the
        session where it was saved, with this handle's model for the chunks still to come.  The state may come from any chunk handle of
        the same C -- another B, another device (it is copied to this handle's device first), another model."""
        s = _slot_array(slots)
        assert s.numel() == len(state), f"{s.numel()} slots for {len(state)} sessions"
        if state._meta_type is not _lib.FsnChunkSlotMeta:
            raise TypeError("state holds frame-by-frame sessions (StreamingFullSubNet.save_slots), not chunk sessions")
        state = state.to(self.device)
        payload = state.payload.contiguous()
        if payload.data_ptr() % 256:
            payload = payload.clone()
        with torch.cuda.device(self.device):
            stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
            _lib.check(self.lib.fsn_chunk_stream_load_slots(self._cs, s.numel(), C.c_void_p(s.data_ptr()), C.c_void_p(payload.data_ptr()),
                                                            state.meta, stream))

    def set_atten_lim(self, slots, db):
        """Attenuation limit of `slots` in dB, as ``StreamingFullSubNet.set_atten_lim`` (C: fsn_chunk_stream_set_atten_lim): every chunk a
        slot completes from now on is enhanced with its limit (``enhance_audio(..., atten_lim_db)``)."""
        s = _slot_array(slots)
        _lib.check(self.lib.fsn_chunk_stream_set_atten_lim(self._cs, s.numel(), C.cast(s.data_ptr(), C.POINTER(C.c_int32)),
                                                           _lib.atten_arg(db, s.numel())))

    def close(self):
        if self._cs is not None:
            self.lib.fsn_chunk_stream_destroy(self._cs)
            self._cs = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
