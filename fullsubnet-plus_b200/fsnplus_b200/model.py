"""Host-side mirror of the reference model classes for the one path this package accelerates.

``FullSubNet_Plus`` mirrors speech_enhance/fullsubnet_plus/model/fullsubnet_plus.py:16-209 and ``Model``
mirrors speech_enhance/fullsubnet/model/fullsubnet.py:12-118: same constructor keywords, same
``state_dict`` keys/shapes (so reference checkpoints load with ``strict=True``), same forward signature and
``[B, 2, F, T]`` float32 output.  The sub-modules below are *parameter containers only*: all arithmetic of
``forward`` runs in the sm_90a CUDA library behind the C ABI of include/fsnplus_b200.h.  There is no
PyTorch/CPU fallback -- CPU tensors, training mode or a missing library raise.
"""
import ctypes as C

import torch
import torch.nn as nn

from . import _lib

TCN_DILATIONS = (1, 2, 5, 9, 1, 2, 5, 9)      # reference sequence_model.py:47-58
TCN_HIDDEN = 512                               # reference causal_conv.py:68


class _NoForward(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter container; run the parent model's forward "
                           "(CUDA library), there is no PyTorch fallback")


class ChannelTimeSenseSELayer(_NoForward):
    """Parameters of the TSSE attention (reference attention_model.py:49-76)."""

    def __init__(self, num_channels, reduction_ratio=2, kersize=(3, 5, 10)):
        super().__init__()
        def branch(k):
            return nn.Sequential(nn.Conv1d(num_channels, num_channels, kernel_size=k, groups=num_channels),
                                 nn.AdaptiveAvgPool1d(1), nn.ReLU(inplace=True))
        self.smallConv1d = branch(kersize[0])
        self.middleConv1d = branch(kersize[1])
        self.largeConv1d = branch(kersize[2])
        self.feature_concate_fc = nn.Linear(3, 1, bias=True)
        self.fc1 = nn.Linear(num_channels, num_channels // reduction_ratio, bias=True)
        self.fc2 = nn.Linear(num_channels // reduction_ratio, num_channels, bias=True)


class ChannelSELayer(_NoForward):
    """Parameters of the SE attention (reference attention_model.py:6-23)."""

    def __init__(self, num_channels, reduction_ratio=2):
        super().__init__()
        self.reduction_ratio = reduction_ratio
        self.fc1 = nn.Linear(num_channels, num_channels // reduction_ratio, bias=True)
        self.fc2 = nn.Linear(num_channels // reduction_ratio, num_channels, bias=True)


class ChannelCBAMLayer(ChannelSELayer):
    """Parameters of the CBAM attention (reference attention_model.py:296-315): same two Linear layers as SE."""


class ChannelECAlayer(_NoForward):
    """Parameters of the ECA attention (reference attention_model.py:337-347)."""

    def __init__(self, channel, k_size=3):
        super().__init__()
        self.conv = nn.Conv1d(1, 1, kernel_size=k_size, padding=(k_size - 1) // 2, bias=False)


class TCNBlock(_NoForward):
    """Parameters of one TCN block (reference causal_conv.py:67-80)."""

    def __init__(self, channels, hidden, dilation):
        super().__init__()
        self.conv1x1 = nn.Conv1d(channels, hidden, 1)
        self.prelu1 = nn.PReLU()
        self.norm1 = nn.GroupNorm(1, hidden, eps=1e-8)
        self.depthwise_conv = nn.Conv1d(hidden, hidden, kernel_size=3, groups=hidden, padding=dilation, dilation=dilation)
        self.prelu2 = nn.PReLU()
        self.norm2 = nn.GroupNorm(1, hidden, eps=1e-8)
        self.sconv = nn.Conv1d(hidden, channels, 1)


class SequenceModel(_NoForward):
    """Parameters of the reference SequenceModel (sequence_model.py:5-93) for the LSTM and TCN cores."""

    def __init__(self, input_size, output_size, hidden_size, num_layers, sequence_model, output_activate_function):
        super().__init__()
        if sequence_model in ("LSTM", "GRU"):                                   # sequence_model.py:31-46
            self.sequence_model = getattr(nn, sequence_model)(input_size=input_size, hidden_size=hidden_size,
                                                              num_layers=num_layers, batch_first=True, bidirectional=False)
            self.fc_output_layer = nn.Linear(hidden_size, output_size)
        elif sequence_model == "TCN":
            blocks = [TCNBlock(input_size, TCN_HIDDEN, d) for d in TCN_DILATIONS]
            self.sequence_model = nn.Sequential(*blocks, nn.ReLU())
            self.fc_output_layer = nn.Linear(input_size, output_size)
        else:
            raise NotImplementedError(f"Not implemented {sequence_model}")                           # sequence_model.py:70
        if output_activate_function not in _lib.ACT:
            raise NotImplementedError(f"Not implemented activation function {output_activate_function}")
        self.output_activate_function = output_activate_function


def _reference_weight_init(m):
    """Same initialisation rule as BaseModel.weight_init (reference base_model.py:332-397) for the module
    types this model contains."""
    if isinstance(m, nn.Conv1d):
        nn.init.normal_(m.weight.data)
        if m.bias is not None:
            nn.init.normal_(m.bias.data)
    elif isinstance(m, nn.Linear):
        nn.init.xavier_normal_(m.weight.data)
        nn.init.normal_(m.bias.data)
    elif isinstance(m, (nn.LSTM, nn.GRU)):
        for p in m.parameters():
            (nn.init.orthogonal_ if p.dim() >= 2 else nn.init.normal_)(p.data)


class _B200Model(nn.Module):
    """Shared machinery: C-ABI handle, lazy parameter push, forward dispatch."""

    _kind = None
    _subband_runs = True

    def _setup(self, num_freqs, look_ahead, sb_num_neighbors, fb_num_neighbors, fb_hidden, sb_hidden, num_layers,
               output_size, fb_act, sb_act, norm_type, kersize, lstm_impl, fast_math, channel_attention="TSSE",
               rnn="LSTM", subband_num=1, tcn_causal=False, sb_tcn=False):
        if norm_type not in _lib.NORM:
            raise NotImplementedError("You must set up a type of Norm. e.g. offline_laplace_norm, "
                                      "cumulative_laplace_norm, forgetting_norm, etc.")       # base_model.py:328-329
        cfg = _lib.FsnConfig()
        cfg.model_kind = self._kind
        cfg.num_freqs, cfg.look_ahead = num_freqs, look_ahead
        cfg.sb_num_neighbors, cfg.fb_num_neighbors = sb_num_neighbors, fb_num_neighbors
        cfg.fb_hidden, cfg.sb_hidden, cfg.num_layers, cfg.output_size = fb_hidden, sb_hidden, num_layers, output_size
        cfg.fb_act, cfg.sb_act = _lib.ACT[fb_act], _lib.ACT[sb_act]
        cfg.norm_type = _lib.NORM[norm_type]
        for i in range(3):
            cfg.kersize[i] = int(kersize[i])
        cfg.lstm_impl = _lib.LSTM_IMPL[lstm_impl]
        cfg.fast_math = int(bool(fast_math))
        cfg.channel_attention = _lib.ATTENTION[channel_attention]
        cfg.rnn_type = _lib.RNN[rnn]
        cfg.subband_num = int(subband_num)
        cfg.tcn_causal = int(bool(tcn_causal))
        cfg.sb_tcn = int(bool(sb_tcn))
        self._cfg = cfg
        self._handle = None
        self._handle_device = None
        self._pushed_version = None
        self._inflight, self._inflight_host = [], []

    # -- handle management ---------------------------------------------------------------------
    def _param_version(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def _ensure_handle(self, device):
        lib = _lib.load_library()
        if self._handle is not None and self._handle_device != device:
            self._release()
        if self._handle is None:
            h = C.c_void_p()
            _lib.check(lib.fsn_model_create(C.byref(self._cfg), C.byref(h)))
            self._handle, self._handle_device, self._pushed_version = h, device, None
        ver = self._param_version()
        if ver != self._pushed_version:
            sd = self.state_dict()
            n = lib.fsn_model_num_params(self._handle)
            for i in range(n):
                key, numel = C.c_char_p(), C.c_int64()
                _lib.check(lib.fsn_model_param_info(self._handle, i, C.byref(key), C.byref(numel)))
                k = key.value.decode()
                if k not in sd:
                    raise _lib.FsnError(f"state_dict has no entry {k}")
                t = self._host_param(sd[k])
                if t.numel() != numel.value:
                    raise _lib.FsnError(f"size mismatch for {k}: {tuple(t.shape)} vs {numel.value} elements")
                _lib.check(lib.fsn_model_set_param(self._handle, key.value, C.c_void_p(t.data_ptr()), t.numel()))
            _lib.check(lib.fsn_model_finalize(self._handle))
            self._pushed_version = ver
        return lib

    @staticmethod
    def _host_param(t):
        """A state_dict tensor as the library takes it: contiguous float32 on the host."""
        return t.detach().to(device="cpu", dtype=torch.float32).contiguous()

    def save_model_file(self, path):
        """Write the configuration and parameters to the model file ``path`` (C ABI: fsn_model_file_write; format in
        include/fsnplus_b200.h), which ``fsn_model_load`` turns into a ready handle in a C or C++ program.  Host only: the model may
        live on any device and no GPU is needed.  A handle loaded from the file has this model's ``weights_id()``."""
        sd = self.state_dict()
        _lib.write_model_file(path, self._cfg, {k: self._host_param(v) for k, v in sd.items()})

    def _release(self):
        if getattr(self, "_handle", None) is not None:
            _lib.load_library().fsn_model_destroy(self._handle)
            self._handle = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    # -- forward -------------------------------------------------------------------------------
    def _check_call(self, x=None):
        """What every entry point needs before it creates a handle: a subband_num the reference forward runs (FullSubNet_Plus), eval
        mode and, for ``x`` (the input tensor; None for the host-buffer call), a CUDA device."""
        if not self._subband_runs:
            raise RuntimeError(f"subband_num={self.subband_num}: the attention was built for {self.num_channels} channels but the "
                               "real/imag branches have num_freqs channels (the reference forward raises here too, "
                               "fullsubnet_plus.py:157-163); only channel_attention_model='ECA' runs with subband_num > 1")
        if self.training:
            raise NotImplementedError("fsnplus_b200 implements the inference (eval) forward only; call .eval()")
        if x is not None and not x.is_cuda:
            raise RuntimeError("fsnplus_b200 has no CPU fallback: move the model and its inputs to a CUDA (H100) device")

    def enhance_spectrum(self, noisy_mag, noisy_real, noisy_imag, pipelined=False, out=None, hold=True, frames=None, atten_lim_db=None):
        """Model forward + decompress_cIRM + complex multiply with the noisy spectrum in ONE call (C ABI: fsn_model_forward_enhance /
        fsn_model_submit_enhance; reference inferencer.py:149-157): [B, 1, F, T] x3 -> enhanced spectrum complex64 [B, F, T], the
        argument of the inferencer's iSTFT.  The cIRM never goes to memory (fused into the sub-band LSTM's epilogue).
        ``pipelined=True``: like ``submit()`` -- valid after ``wait()`` / ``wait_lane()``.  ``frames``: as in ``forward()``.
        ``atten_lim_db``: None, one number or B numbers -- no bin of clip b loses more than atten_lim_db[b] dB (C ABI:
        fsn_model_forward_enhance_lim, DESIGN.md §3.18; float('inf'): no limit).  The pipelined call takes no limit (ValueError)."""
        if atten_lim_db is not None and pipelined:
            raise ValueError("atten_lim_db is not supported with pipelined=True (the pipelined entry points take no limit)")
        return self._run(noisy_mag, noisy_real, noisy_imag, enhance=True, pipelined=pipelined, out=out, hold=hold, frames=frames,
                         atten_lim_db=atten_lim_db)

    def enhance_audio(self, wave, lengths=None, atten_lim_db=None):
        """Waveforms in, enhanced waveforms out in ONE call (C ABI: fsn_model_enhance_audio): torch.stft -> model -> decompress_cIRM x
        spectrum -> torch.istft(length = L_b) per clip, with both transforms on the device (what ``inference.enhance_batch`` /
        ``enhance_ragged`` compute).  ``wave``: [B, L] float32 CUDA; ``lengths``: None (every clip is L samples) or B sample counts (a
        sequence or a 1-D CPU integer tensor), clip b being the first lengths[b] samples of its row.  Returns [B, L], zero past each
        clip's length.  n_fft = 2 (num_freqs - 1), hop = n_fft / 2, periodic Hann window.  ``atten_lim_db``: None, one number or B
        numbers -- no bin of clip b loses more than atten_lim_db[b] dB (C ABI: fsn_model_enhance_audio_lim, DESIGN.md §3.18;
        float('inf'): no limit)."""
        if wave.dim() != 2:
            raise ValueError(f"enhance_audio: wave must be [B, L], got {tuple(wave.shape)}")
        self._check_call(wave)
        B, L = wave.shape
        hl = _lib.lengths_arg(lengths, B)
        ha = _lib.atten_arg(atten_lim_db, B)
        x = wave.detach().to(dtype=torch.float32).contiguous()
        with torch.cuda.device(x.device):
            lib = self._ensure_handle(x.device)
            out = torch.empty((B, L), dtype=torch.float32, device=x.device)
            stream = C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)
            if ha is None:
                _lib.check(lib.fsn_model_enhance_audio(self._handle, C.c_void_p(x.data_ptr()), B, L, hl, C.c_void_p(out.data_ptr()), stream))
            else:
                _lib.check(lib.fsn_model_enhance_audio_lim(self._handle, C.c_void_p(x.data_ptr()), B, L, hl, ha, C.c_void_p(out.data_ptr()),
                                                           stream))
        return out

    @staticmethod
    def _frames_arg(frames, B):
        """``frames`` (a sequence of ints or a CPU integer tensor of length B) as a C int32 array."""
        if isinstance(frames, torch.Tensor):
            if frames.is_cuda or frames.is_floating_point() or frames.is_complex() or frames.dim() != 1:
                raise ValueError("frames must be a 1-D CPU integer tensor or a sequence of ints")
            frames = frames.tolist()
        frames = [int(n) for n in frames]
        if len(frames) != B:
            raise ValueError(f"frames has {len(frames)} entries for a batch of {B}")
        return (C.c_int32 * B)(*frames)

    def _run(self, mag, real, imag, enhance=False, pipelined=False, out=None, hold=True, frames=None, atten_lim_db=None):
        assert mag.dim() == 4                                            # fullsubnet_plus.py:136
        B, Cn, F, T = mag.shape
        if frames is not None and pipelined:
            raise ValueError("frames (ragged batches) is not supported with pipelined=True / submit()")
        hframes = self._frames_arg(frames, B) if frames is not None else None
        hatten = _lib.atten_arg(atten_lim_db, B)
        assert Cn == 1, f"{self.__class__.__name__} takes the mag feature as inputs."      # :141
        self._check_call(mag)
        if F != self._cfg.num_freqs:
            raise ValueError(f"expected {self._cfg.num_freqs} frequency bins, got {F}")
        ins = [x.detach().to(dtype=torch.float32).contiguous() if x is not None else None for x in (mag, real, imag)]
        with torch.cuda.device(mag.device):
            lib = self._ensure_handle(mag.device)
            if out is None:
                out = (torch.empty((B, F, T), dtype=torch.complex64, device=mag.device) if enhance else
                       torch.empty((B, self._cfg.output_size, F, T), dtype=torch.float32, device=mag.device))
            ptr = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p()
            stream = C.c_void_p(torch.cuda.current_stream(mag.device).cuda_stream)
            if hatten is not None:                                          # enhance only (enhance_spectrum)
                _lib.check(lib.fsn_model_forward_enhance_lim(self._handle, ptr(ins[0]), ptr(ins[1]), ptr(ins[2]), B, T, hframes, hatten,
                                                             ptr(out), stream))
                return out
            if hframes is not None:
                fn = lib.fsn_model_forward_enhance_ragged if enhance else lib.fsn_model_forward_ragged
                _lib.check(fn(self._handle, ptr(ins[0]), ptr(ins[1]), ptr(ins[2]), B, T, hframes, ptr(out), stream))
                return out
            fn = {(False, False): lib.fsn_model_forward, (True, False): lib.fsn_model_forward_enhance,
                  (False, True): lib.fsn_model_submit, (True, True): lib.fsn_model_submit_enhance}[(enhance, pipelined)]
            _lib.check(fn(self._handle, ptr(ins[0]), ptr(ins[1]), ptr(ins[2]), B, T, ptr(out), stream))
            if pipelined:
                if hold:                                                        # hold=False: the caller keeps the buffers alive itself (EnhancePipeline's ring)
                    self._inflight.append((ins, out))
                self.last_lane = int(lib.fsn_model_last_lane(self._handle))     # ticket for wait_lane()
        return out

    def submit(self, mag, real=None, imag=None, out=None, hold=True):
        """Pipelined forward for STREAMS of batches (C ABI: fsn_model_submit): same inputs as forward(), returns the output tensor
        immediately; it is valid on the current stream after ``wait()``.  The full-band front end of this batch runs while the
        sub-band LSTM of the previously submitted batch is still running (two internal streams, two workspace lanes).  The inputs
        must not be modified before ``wait()``; references to them are held until then."""
        return self._run(mag, real, imag, enhance=False, pipelined=True, out=out, hold=hold)

    def wait_lane(self, lane, stream=None):
        """Make ``stream`` (default: the current stream) wait for the batch most recently submitted into workspace lane ``lane``
        (``self.last_lane`` right after its ``submit()``); valid until the next submit into the same lane, i.e. two submits later."""
        with torch.cuda.device(self._handle_device):
            st = stream if stream is not None else torch.cuda.current_stream(self._handle_device)
            _lib.check(_lib.load_library().fsn_model_wait_lane(self._handle, int(lane), C.c_void_p(st.cuda_stream)))

    def wait(self):
        """Make the current stream wait for every ``submit()`` issued so far (does not block the host)."""
        if self._handle is not None:
            with torch.cuda.device(self._handle_device):
                stream = C.c_void_p(torch.cuda.current_stream(self._handle_device).cuda_stream)
                _lib.check(_lib.load_library().fsn_model_wait(self._handle, stream))
                # the tensors may now be freed: torch's caching allocator orders reuse on the current stream, which waits for them
                for ins, out in self._inflight:
                    for t in ins + [out]:
                        if t is not None and t.is_cuda:
                            t.record_stream(torch.cuda.current_stream(self._handle_device))
        self._inflight = []

    @staticmethod
    def _check_host(name, t, shape):
        if not isinstance(t, torch.Tensor) or t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
            raise ValueError(f"forward_host: {name} must be a contiguous CPU float32 tensor of shape {tuple(shape)}, got "
                             f"{type(t).__name__} {getattr(t, 'device', '')} {getattr(t, 'dtype', '')} {tuple(getattr(t, 'shape', ()))}")

    def forward_host(self, mag, real=None, imag=None, out=None, device="cuda:0", pipelined=False):
        """Same forward through the HOST-buffer entry point of the C ABI (H2D + forward + D2H in one call).
        ``mag/real/imag``: CPU float32 tensors [B, 1, F, T] (pinned for best bandwidth); returns a CPU tensor.
        ``pipelined=True`` uses the double-buffered async entry point (copies and the front end of the next batch overlap the
        sub-band LSTM of the previous one); it needs PINNED buffers, the returned tensor is valid after ``sync_host()`` and the
        inputs/outputs are kept referenced until then."""
        self._check_call()
        if mag.dim() != 4:
            raise ValueError("forward_host: mag must be [B, 1, F, T]")
        B, _, F, T = mag.shape
        shape = (B, 1, self._cfg.num_freqs, T)
        self._check_host("mag", mag, shape)
        if self._kind == _lib.KIND_PLUS:
            self._check_host("real", real, shape)
            self._check_host("imag", imag, shape)
        else:
            real = imag = None
        if out is None:
            out = torch.empty((B, self._cfg.output_size, F, T), dtype=torch.float32).pin_memory()
        self._check_host("out", out, (B, self._cfg.output_size, F, T))
        if pipelined and not all(t.is_pinned() for t in (mag, real, imag, out) if t is not None):
            raise ValueError("forward_host(pipelined=True) needs pinned host tensors (the copies are asynchronous)")
        dev = torch.device(device)
        with torch.cuda.device(dev):
            lib = self._ensure_handle(dev)
            ptr = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p()
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            fn = lib.fsn_model_forward_host_async if pipelined else lib.fsn_model_forward_host
            _lib.check(fn(self._handle, ptr(mag), ptr(real), ptr(imag), B, T, ptr(out), stream))
        if pipelined:
            self._inflight_host.append((mag, real, imag, out))     # the async copies read / write these after the call returns
        return out

    def sync_host(self):
        """Wait for every forward_host(..., pipelined=True) / submit() issued so far (their outputs are then valid)."""
        if self._handle is not None:
            _lib.check(_lib.load_library().fsn_model_sync_host(self._handle))
        self._inflight_host = []
        self._inflight = []

    # -- introspection used by tests / bench -----------------------------------------------------
    def last_lstm_impl(self):
        return {0: "none", 1: "mma", 2: "tcgen05", 3: "tcn"}[_lib.load_library().fsn_model_last_lstm_impl(self._handle)] if self._handle else "none"

    def last_lstm_ms(self):
        return float(_lib.load_library().fsn_model_last_lstm_ms(self._handle)) if self._handle else -1.0

    def lstm_ms_history(self, n=32):
        buf = (C.c_float * n)()
        k = _lib.load_library().fsn_model_lstm_ms_history(self._handle, buf, n) if self._handle else 0
        return [float(buf[i]) for i in range(k)]

    def timeline(self, n=32):
        """[(front start, front end, LSTM start, LSTM end)] in ms for the last n forwards, relative to the first one's front start."""
        buf = (C.c_float * (4 * n))()
        k = _lib.load_library().fsn_model_timeline(self._handle, buf, n) if self._handle else 0
        return [tuple(float(buf[4 * i + j]) for j in range(4)) for i in range(k)]

    def last_launch_count(self):
        return int(_lib.load_library().fsn_model_last_launch_count(self._handle)) if self._handle else 0

    def weights_id(self):
        """fsn_model_weights_id: 64-bit hash of the parameters last pushed to the handle (0 before the first forward / stream)."""
        return int(_lib.load_library().fsn_model_weights_id(self._handle)) if self._handle else 0

    def workspace_bytes(self):
        """Bytes this model currently holds in forward workspaces (both lanes and the sub-band scratch; parameters excluded)."""
        return int(_lib.load_library().fsn_model_workspace_bytes(self._handle)) if self._handle else 0

    def last_plan(self):
        """(clips per sub-batch, sub-band window in frames) of the last plain forward; window 0 = unwindowed."""
        if not self._handle:
            return (0, 0)
        bs, tw = C.c_int32(), C.c_int32()
        _lib.check(_lib.load_library().fsn_model_last_plan(self._handle, C.byref(bs), C.byref(tw)))
        return (bs.value, tw.value)

    def plan(self, B, T):
        """(clips per sub-batch, sub-band window in frames or 0, workspace bytes) that this model's next plain forward of B clips of
        T frames will use (C ABI: fsn_model_plan, with the FSN_* knobs the handle read at creation).  Creates the handle if needed, so
        the model must be on its CUDA device; enqueues no GPU work."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("plan() needs the model on its CUDA device (the plan is the handle's)")
        with torch.cuda.device(dev):
            lib = self._ensure_handle(dev)
        bs, tw, nb = C.c_int32(), C.c_int32(), C.c_int64()
        _lib.check(lib.fsn_model_plan(self._handle, int(B), int(T), C.byref(bs), C.byref(tw), C.byref(nb)))
        return bs.value, tw.value, nb.value

    def last_plan_bins(self):
        """(clips per sub-batch, sub-band window in frames, sub-band TCN bins per chunk) of the last plain forward; 0 = unwindowed /
        unchunked."""
        if not self._handle:
            return (0, 0, 0)
        bs, tw, fc = C.c_int32(), C.c_int32(), C.c_int32()
        _lib.check(_lib.load_library().fsn_model_last_plan_bins(self._handle, C.byref(bs), C.byref(tw), C.byref(fc)))
        return (bs.value, tw.value, fc.value)

    def plan_bins(self, B, T):
        """plan() with the sub-band TCN's bin chunk: (clips per sub-batch, window or 0, bins per chunk or 0, workspace bytes) of this
        model's next plain forward (C ABI: fsn_model_plan_bins, with the FSN_* knobs the handle read at creation, FSN_SB_CHUNK among
        them).  Creates the handle if needed, so the model must be on its CUDA device; enqueues no GPU work."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("plan_bins() needs the model on its CUDA device (the plan is the handle's)")
        with torch.cuda.device(dev):
            lib = self._ensure_handle(dev)
        bs, tw, fc, nb = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
        _lib.check(lib.fsn_model_plan_bins(self._handle, int(B), int(T), C.byref(bs), C.byref(tw), C.byref(fc), C.byref(nb)))
        return bs.value, tw.value, fc.value, nb.value

    def release_workspace(self):
        """Free every forward workspace this model holds (synchronises the device); the next forward allocates again."""
        if self._handle:
            _lib.check(_lib.load_library().fsn_model_release_workspace(self._handle))

    def get_stage(self, name, shape, device):
        t = torch.empty(shape, dtype=torch.float32, device=device)
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
        _lib.check(_lib.load_library().fsn_model_get_stage(self._handle, name.encode(), C.c_void_p(t.data_ptr()), t.numel(), stream))
        return t


class FullSubNet_Plus(_B200Model):
    """Drop-in for fullsubnet_plus.model.fullsubnet_plus.FullSubNet_Plus (config/inference.toml:27)."""

    _kind = _lib.KIND_PLUS

    def __init__(self, num_freqs, look_ahead, sequence_model, fb_num_neighbors, sb_num_neighbors,
                 fb_output_activate_function, sb_output_activate_function, fb_model_hidden_size, sb_model_hidden_size,
                 channel_attention_model="SE", norm_type="offline_laplace_norm", num_groups_in_drop_band=2,
                 output_size=2, subband_num=1, kersize=[3, 5, 10], weight_init=True,
                 num_layers=2, lstm_impl="auto", fast_math=True, causal_tcn=False):
        """Reference keywords (fullsubnet_plus.py:17-34) + additive ones: num_layers (LSTM depth), lstm_impl, fast_math,
        causal_tcn (TCNBlock(causal=True) in the full-band models, causal_conv.py:74-75,104-105; parameters unchanged).
        With sequence_model="TCN" the sub-band model is the reference's 8-block TCN of hidden width 512: like the reference, it
        ignores sb_model_hidden_size and num_layers, and lstm_impl / fast_math have no effect."""
        super().__init__()
        assert sequence_model in ("GRU", "LSTM", "TCN"), f"{self.__class__.__name__} only support GRU, LSTM and TCN."
        if channel_attention_model not in _lib.ATTENTION:                                       # fullsubnet_plus.py:69-70
            raise NotImplementedError(f"Not implemented channel attention model {channel_attention_model}")
        # fullsubnet_plus.py:47-50.  With subband_num > 1 the reference builds all three attentions for F // subband_num + 1
        # channels but applies the real / imag ones to F channels (:157-163), so its forward only runs with the
        # channel-agnostic ECA; the containers keep the reference's shapes and every entry point raises like the reference
        # forward otherwise (_check_call).
        self.num_channels = num_freqs if subband_num == 1 else num_freqs // subband_num + 1
        self._subband_runs = subband_num == 1 or channel_attention_model == "ECA"
        for sfx in ("", "_real", "_imag"):
            setattr(self, "channel_attention" + sfx,                                               # fullsubnet_plus.py:52-68
                    {"TSSE": lambda: ChannelTimeSenseSELayer(self.num_channels, kersize=kersize),
                     "SE": lambda: ChannelSELayer(self.num_channels), "CBAM": lambda: ChannelCBAMLayer(self.num_channels),
                     "ECA": lambda: ChannelECAlayer(self.num_channels)}[channel_attention_model]())
        for sfx in ("", "_real", "_imag"):                      # full-band models are TCNs (fullsubnet_plus.py:72-100)
            setattr(self, "fb_model" + sfx, SequenceModel(num_freqs, num_freqs, fb_model_hidden_size, 2, "TCN",
                                                          fb_output_activate_function))
        self.sb_model = SequenceModel((sb_num_neighbors * 2 + 1) + 3 * (fb_num_neighbors * 2 + 1), output_size,
                                      sb_model_hidden_size, num_layers, sequence_model, sb_output_activate_function)
        self.subband_num = subband_num
        self.sb_num_neighbors = sb_num_neighbors
        self.fb_num_neighbors = fb_num_neighbors
        self.look_ahead = look_ahead
        self.num_groups_in_drop_band = num_groups_in_drop_band      # read by the reference trainer (trainer.py:335)
        self.output_size = output_size
        self._setup(num_freqs, look_ahead, sb_num_neighbors, fb_num_neighbors, fb_model_hidden_size, sb_model_hidden_size,
                    num_layers, output_size, fb_output_activate_function, sb_output_activate_function, norm_type, kersize,
                    lstm_impl, fast_math, channel_attention_model, "LSTM" if sequence_model == "TCN" else sequence_model,
                    subband_num if self._subband_runs else 1, causal_tcn, sb_tcn=sequence_model == "TCN")
        self.causal_tcn = bool(causal_tcn)
        if weight_init:
            self.apply(_reference_weight_init)

    def forward(self, noisy_mag, noisy_real, noisy_imag, *, frames=None):
        """[B, 1, F, T] x3 -> [B, 2, F, T] (reference fullsubnet_plus.py:122-209, eval semantics per sample).
        ``frames`` (additive, keyword-only): the frame count of every clip of a ragged batch, 1 <= frames[b] <= T.  Clip b is then
        its first frames[b] frames; its output equals that clip's own forward there and is zero after (C ABI:
        fsn_model_forward_ragged)."""
        return self._run(noisy_mag, noisy_real, noisy_imag, frames=frames)


class Model(_B200Model):
    """Drop-in for fullsubnet.model.fullsubnet.Model (config/inference.toml:28)."""

    _kind = _lib.KIND_FSN

    def __init__(self, num_freqs, look_ahead, sequence_model, fb_num_neighbors, sb_num_neighbors,
                 fb_output_activate_function, sb_output_activate_function, fb_model_hidden_size, sb_model_hidden_size,
                 norm_type="offline_laplace_norm", num_groups_in_drop_band=2, weight_init=True,
                 num_layers=2, lstm_impl="auto", fast_math=True):
        super().__init__()
        assert sequence_model in ("GRU", "LSTM"), f"{self.__class__.__name__} only support GRU and LSTM."
        self.fb_model = SequenceModel(num_freqs, num_freqs, fb_model_hidden_size, num_layers, sequence_model,
                                      fb_output_activate_function)
        self.sb_model = SequenceModel((sb_num_neighbors * 2 + 1) + (fb_num_neighbors * 2 + 1), 2, sb_model_hidden_size,
                                      num_layers, sequence_model, sb_output_activate_function)
        self.sb_num_neighbors = sb_num_neighbors
        self.fb_num_neighbors = fb_num_neighbors
        self.look_ahead = look_ahead
        self.num_groups_in_drop_band = num_groups_in_drop_band
        self._setup(num_freqs, look_ahead, sb_num_neighbors, fb_num_neighbors, fb_model_hidden_size, sb_model_hidden_size,
                    num_layers, 2, fb_output_activate_function, sb_output_activate_function, norm_type, (3, 5, 10),
                    lstm_impl, fast_math, "TSSE", sequence_model)
        if weight_init:
            self.apply(_reference_weight_init)

    def forward(self, noisy_mag, *, frames=None):
        """[B, 1, F, T] -> [B, 2, F, T] (reference fullsubnet.py:68-118, eval semantics per sample).  ``frames``: as in
        FullSubNet_Plus.forward."""
        return self._run(noisy_mag, None, None, frames=frames)
