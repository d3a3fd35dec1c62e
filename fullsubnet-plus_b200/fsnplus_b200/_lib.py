"""ctypes binding of the C ABI declared in include/fsnplus_b200.h (the drop-in boundary)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

KIND_PLUS, KIND_FSN = 0, 1
ACT = {None: 0, False: 0, "": 0, "ReLU": 1, "Tanh": 2, "ReLU6": 3}
NORM = {"offline_laplace_norm": 0, "cumulative_laplace_norm": 1, "offline_gaussian_norm": 2, "cumulative_layer_norm": 3}
LSTM_IMPL = {"auto": 0, "mma": 1, "tcgen05": 2}
RNN = {"LSTM": 0, "GRU": 1}                                  # FSN_RNN_* (reference sequence_model.py:31-46)
ATTENTION = {"TSSE": 0, "SE": 1, "CBAM": 2, "ECA": 3}     # FSN_ATTN_* (reference fullsubnet_plus.py:52-70)

# every symbol include/fsnplus_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "fsn_version", "fsn_last_error", "fsn_model_create", "fsn_model_destroy", "fsn_model_set_param",
    "fsn_model_num_params", "fsn_model_param_info", "fsn_model_finalize", "fsn_model_forward",
    "fsn_model_forward_host", "fsn_model_forward_host_async", "fsn_model_sync_host", "fsn_model_submit", "fsn_model_wait", "fsn_model_forward_enhance", "fsn_model_submit_enhance", "fsn_model_forward_ragged", "fsn_model_forward_enhance_ragged", "fsn_model_last_lane", "fsn_model_wait_lane", "fsn_apply_cirm", "fsn_stream_create", "fsn_stream_step", "fsn_stream_destroy", "fsn_model_get_stage", "fsn_model_last_launch_count", "fsn_model_last_lstm_impl", "fsn_model_last_fb_ws", "fsn_model_last_lstm_ms", "fsn_model_lstm_ms_history", "fsn_model_timeline",
    "fsn_plan_forward", "fsn_model_workspace_bytes", "fsn_model_last_plan", "fsn_model_plan", "fsn_model_release_workspace",
    "fsn_plan_forward_bins", "fsn_model_plan_bins", "fsn_model_last_plan_bins",
    "fsn_sw128_offset", "fsn_tc5_weight_stream_bytes", "fsn_tc5_pack_weights", "fsn_tc5_gate_row", "fsn_tc5r_weight_stream_bytes", "fsn_tc5r_pack_layer",
    "fsn_gemm_f16", "fsn_gemm_f16_tile_n",
    "fsn_tc5r_gin_weights", "fsn_tc5r_ring_stages", "fsn_lstm_mma_rows", "fsn_model_sb_forward",
    "fsn_stream_step_slots", "fsn_stream_step_audio_slots",
    "fsn_stream_state_bytes", "fsn_stream_state_layout", "fsn_model_weights_id", "fsn_stream_save_slots", "fsn_stream_load_slots",
    "fsn_model_enhance_audio", "fsn_plan_audio",
    "fsn_stream_step_chunk", "fsn_stream_chunk_plan", "fsn_stream_step_audio_chunk",
    "fsn_model_file_write", "fsn_model_file_config", "fsn_model_load",
    "fsn_chunk_stream_create", "fsn_chunk_stream_step", "fsn_chunk_stream_destroy",
    "fsn_chunk_stream_state_layout", "fsn_chunk_stream_save_slots", "fsn_chunk_stream_load_slots",
    "fsn_model_forward_enhance_lim", "fsn_model_enhance_audio_lim", "fsn_stream_set_atten_lim", "fsn_chunk_stream_set_atten_lim",
    "fsn_stream_get_stage", "fsn_stream_fb_ws", "fsn_stream_step_audio_samples",
    "fsn_metric_si_sdr_workspace", "fsn_metric_si_sdr", "fsn_metric_stoi_workspace", "fsn_metric_stoi",
    "fsn_metric_sdr_workspace", "fsn_metric_sdr",
]


class FsnError(RuntimeError):
    pass


class FsnConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("model_kind", "num_freqs", "look_ahead", "sb_num_neighbors", "fb_num_neighbors",
                                          "fb_hidden", "sb_hidden", "num_layers", "output_size", "fb_act", "sb_act",
                                          "norm_type")] + [("kersize", C.c_int32 * 3), ("lstm_impl", C.c_int32),
                                                           ("fast_math", C.c_int32), ("channel_attention", C.c_int32), ("rnn_type", C.c_int32), ("subband_num", C.c_int32), ("tcn_causal", C.c_int32),
                                                           ("sb_tcn", C.c_int32)]


STATE_MODE_MASK, STATE_MODE_AUDIO = 1, 2                    # FSN_STATE_MODE_*
SLOT_STATE_MAGIC, SLOT_STATE_VERSION = 0x534E5346, 1        # FSN_SLOT_STATE_MAGIC ('F' 'S' 'N' 'S'), FSN_SLOT_STATE_VERSION


class FsnSlotMeta(C.Structure):
    """fsn_slot_meta: the host-side description of one saved streaming session (include/fsnplus_b200.h)."""
    _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("cfg", FsnConfig), ("weights_id", C.c_uint64), ("mode", C.c_int32),
                ("frames", C.c_int32), ("tick", C.c_int32), ("hops", C.c_int32), ("payload_bytes", C.c_int64)]


CHUNK_STATE_MAGIC, CHUNK_STATE_VERSION = 0x434E5346, 1      # FSN_CHUNK_STATE_MAGIC ('F' 'S' 'N' 'C'), FSN_CHUNK_STATE_VERSION


class FsnChunkSlotMeta(C.Structure):
    """fsn_chunk_slot_meta: the host-side description of one saved overlapped-chunk session (include/fsnplus_b200.h)."""
    _fields_ = [("magic", C.c_uint32), ("version", C.c_uint32), ("chunk_samples", C.c_int32), ("pre_context", C.c_int32),
                ("num_freqs", C.c_int32), ("model_kind", C.c_int32), ("weights_id", C.c_uint64), ("samples", C.c_int64),
                ("chunks", C.c_int64), ("payload_bytes", C.c_int64)]


def chunk_state_layout(chunk_samples):
    """fsn_chunk_stream_state_layout: (payload bytes per session, sizeof(fsn_chunk_slot_meta)) of chunk sessions of chunk_samples.
    Host only; needs no GPU."""
    lib = load_library()
    nb, mb = C.c_int64(), C.c_int32()
    check(lib.fsn_chunk_stream_state_layout(int(chunk_samples), C.byref(nb), C.byref(mb)))
    return nb.value, mb.value


def state_layout(cfg, mode):
    """fsn_stream_state_layout: (payload bytes per session, sizeof(fsn_slot_meta)) of a configuration in mode STATE_MODE_MASK or
    STATE_MODE_AUDIO.  Host only; needs no GPU."""
    lib = load_library()
    nb, mb = C.c_int64(), C.c_int32()
    check(lib.fsn_stream_state_layout(C.byref(cfg), int(mode), C.byref(nb), C.byref(mb)))
    return nb.value, mb.value


def write_model_file(path, cfg, params):
    """fsn_model_file_write: ``cfg`` and ``params`` ({state_dict key: contiguous float32 CPU tensor}) to the model file ``path``.  Host
    only; needs no GPU."""
    keys = list(params)
    n = len(keys)
    ckeys = (C.c_char_p * n)(*[k.encode() for k in keys])
    data = (C.c_void_p * n)(*[params[k].data_ptr() for k in keys])
    numel = (C.c_int64 * n)(*[params[k].numel() for k in keys])
    check(load_library().fsn_model_file_write(os.fsencode(path), C.byref(cfg), n, ckeys, data, numel))


def model_file_config(path):
    """fsn_model_file_config: the FsnConfig of the model file ``path``, after verifying the whole file.  Host only; needs no GPU."""
    cfg = FsnConfig()
    check(load_library().fsn_model_file_config(os.fsencode(path), C.byref(cfg)))
    return cfg


def lib_path():
    """The in-tree library; FSN_B200_LIB points at another build of the same sources (e.g. a -DFSN_MBAR_DEBUG build)."""
    return os.environ.get("FSN_B200_LIB") or os.path.join(_HERE, "libfsnplus_b200.so")


def load_library():
    """Load the in-tree CUDA library.  There is no fallback: a missing build is an error."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise FsnError(f"{path} not found: run `python __graft_entry__.py` (nvcc, sm_90a) first; "
                       "fsnplus_b200 has no CPU or PyTorch fallback")
    lib = C.CDLL(path)
    vp, i32, i64, fp = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_float)
    lib.fsn_version.restype = C.c_int
    lib.fsn_last_error.restype = C.c_char_p
    lib.fsn_model_create.argtypes = [C.POINTER(FsnConfig), C.POINTER(vp)]
    lib.fsn_model_destroy.argtypes = [vp]
    lib.fsn_model_destroy.restype = None
    lib.fsn_model_set_param.argtypes = [vp, C.c_char_p, vp, i64]
    lib.fsn_model_num_params.argtypes = [vp]
    lib.fsn_model_param_info.argtypes = [vp, C.c_int, C.POINTER(C.c_char_p), C.POINTER(i64)]
    lib.fsn_model_finalize.argtypes = [vp]
    lib.fsn_model_forward.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.fsn_model_forward_host.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.fsn_model_forward_host_async.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.fsn_model_sync_host.argtypes = [vp]
    lib.fsn_model_submit.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.fsn_model_wait.argtypes = [vp, vp]
    lib.fsn_model_forward_enhance.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.fsn_model_submit_enhance.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
    lib.fsn_model_forward_ragged.argtypes = [vp, vp, vp, vp, i32, i32, C.POINTER(i32), vp, vp]
    lib.fsn_model_forward_enhance_ragged.argtypes = [vp, vp, vp, vp, i32, i32, C.POINTER(i32), vp, vp]
    lib.fsn_model_last_lane.argtypes = [vp]
    lib.fsn_model_wait_lane.argtypes = [vp, i32, vp]
    lib.fsn_stream_create.argtypes = [vp, i32, C.POINTER(vp)]
    lib.fsn_stream_step.argtypes = [vp, vp, vp, C.POINTER(i32), vp]
    lib.fsn_stream_step_slots.argtypes = [vp, vp, vp, vp, vp, vp]
    lib.fsn_stream_step_audio_slots.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.fsn_stream_step_chunk.argtypes = [vp, vp, i32, vp, vp, vp, vp]
    lib.fsn_stream_step_audio_chunk.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp, vp]
    lib.fsn_stream_step_audio_samples.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    lib.fsn_stream_chunk_plan.argtypes = [C.POINTER(FsnConfig), i32, i32, C.c_double, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
    lib.fsn_stream_destroy.argtypes = [vp]
    lib.fsn_stream_destroy.restype = None
    lib.fsn_stream_state_bytes.argtypes = [vp]
    lib.fsn_stream_state_bytes.restype = i64
    lib.fsn_stream_state_layout.argtypes = [C.POINTER(FsnConfig), i32, C.POINTER(i64), C.POINTER(i32)]
    lib.fsn_model_weights_id.argtypes = [vp]
    lib.fsn_model_weights_id.restype = C.c_uint64
    lib.fsn_stream_save_slots.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.fsn_stream_load_slots.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.fsn_apply_cirm.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    lib.fsn_model_get_stage.argtypes = [vp, C.c_char_p, vp, i64, vp]
    lib.fsn_stream_get_stage.argtypes = [vp, C.c_char_p, vp, i64, vp]
    lib.fsn_stream_fb_ws.argtypes = [vp]
    lib.fsn_model_last_launch_count.argtypes = [vp]
    lib.fsn_model_last_launch_count.restype = i64
    lib.fsn_model_last_lstm_impl.argtypes = [vp]
    lib.fsn_model_last_fb_ws.argtypes = [vp]
    lib.fsn_model_last_lstm_ms.argtypes = [vp]
    lib.fsn_model_last_lstm_ms.restype = C.c_float
    lib.fsn_model_lstm_ms_history.argtypes = [vp, fp, i32]
    lib.fsn_model_timeline.argtypes = [vp, fp, i32]
    lib.fsn_plan_forward.argtypes = [C.POINTER(FsnConfig), i32, i32, C.c_double, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
    lib.fsn_model_workspace_bytes.argtypes = [vp]
    lib.fsn_model_workspace_bytes.restype = i64
    lib.fsn_model_last_plan.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
    lib.fsn_model_plan.argtypes = [vp, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
    lib.fsn_model_release_workspace.argtypes = [vp]
    lib.fsn_plan_forward_bins.argtypes = [C.POINTER(FsnConfig), i32, i32, C.c_double, i32, i32, C.POINTER(i32), C.POINTER(i32),
                                          C.POINTER(i32), C.POINTER(i64)]
    lib.fsn_model_plan_bins.argtypes = [vp, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i64)]
    lib.fsn_model_last_plan_bins.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    lib.fsn_sw128_offset.argtypes = [C.c_uint32, C.c_uint32]
    lib.fsn_sw128_offset.restype = C.c_uint32
    lib.fsn_tc5_weight_stream_bytes.argtypes = [i32, i32]
    lib.fsn_tc5_weight_stream_bytes.restype = i64
    lib.fsn_tc5_pack_weights.argtypes = [i32, i32, vp, vp, vp, vp, vp]
    lib.fsn_tc5_gate_row.argtypes = [i32, i32, i32]
    lib.fsn_tc5r_weight_stream_bytes.argtypes = [i32]
    lib.fsn_tc5r_weight_stream_bytes.restype = i64
    lib.fsn_tc5r_pack_layer.argtypes = [i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, vp]
    lib.fsn_tc5_gate_row.restype = i32
    lib.fsn_gemm_f16.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp]
    lib.fsn_gemm_f16_tile_n.argtypes = [i64, i32, i32, i32]
    lib.fsn_gemm_f16_tile_n.restype = i32
    lib.fsn_tc5r_gin_weights.argtypes = [i32, i32, i32, vp, vp]
    lib.fsn_tc5r_ring_stages.argtypes = [i32, i32, i32]
    lib.fsn_tc5r_ring_stages.restype = i32
    lib.fsn_lstm_mma_rows.argtypes = [i32, i32, i32, i32]
    lib.fsn_lstm_mma_rows.restype = i32
    lib.fsn_model_sb_forward.argtypes = [vp, vp, i32, i32, i32, C.POINTER(i32), vp, vp, vp, vp, vp]
    lib.fsn_model_enhance_audio.argtypes = [vp, vp, i32, i64, C.POINTER(i64), vp, vp]
    lib.fsn_plan_audio.argtypes = [C.POINTER(FsnConfig), i32, i64, C.POINTER(i64), C.c_double, i32, i32, C.POINTER(i32), C.POINTER(i32),
                                   C.POINTER(i32), C.POINTER(i64)]
    lib.fsn_model_file_write.argtypes = [C.c_char_p, C.POINTER(FsnConfig), i32, C.POINTER(C.c_char_p), C.POINTER(vp), C.POINTER(i64)]
    lib.fsn_model_file_config.argtypes = [C.c_char_p, C.POINTER(FsnConfig)]
    lib.fsn_model_load.argtypes = [C.c_char_p, C.POINTER(vp)]
    lib.fsn_chunk_stream_create.argtypes = [vp, i32, i32, C.POINTER(vp)]
    lib.fsn_chunk_stream_step.argtypes = [vp, vp, i32, vp, vp, vp, vp, vp]
    lib.fsn_chunk_stream_destroy.argtypes = [vp]
    lib.fsn_chunk_stream_destroy.restype = None
    lib.fsn_chunk_stream_state_layout.argtypes = [i32, C.POINTER(i64), C.POINTER(i32)]
    lib.fsn_chunk_stream_save_slots.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.fsn_chunk_stream_load_slots.argtypes = [vp, i32, vp, vp, vp, vp]
    lib.fsn_model_forward_enhance_lim.argtypes = [vp, vp, vp, vp, i32, i32, C.POINTER(i32), fp, vp, vp]
    lib.fsn_model_enhance_audio_lim.argtypes = [vp, vp, i32, i64, C.POINTER(i64), fp, vp, vp]
    lib.fsn_stream_set_atten_lim.argtypes = [vp, i32, C.POINTER(i32), fp]
    lib.fsn_chunk_stream_set_atten_lim.argtypes = [vp, i32, C.POINTER(i32), fp]
    lib.fsn_metric_si_sdr_workspace.argtypes = [i32, i64, C.POINTER(i64), C.POINTER(i64)]
    lib.fsn_metric_si_sdr.argtypes = [vp, vp, i32, i64, C.POINTER(i64), vp, i64, vp, vp]
    lib.fsn_metric_stoi_workspace.argtypes = [i32, i64, C.POINTER(i64), i32, C.POINTER(i64)]
    lib.fsn_metric_stoi.argtypes = [vp, vp, i32, i64, C.POINTER(i64), i32, vp, i64, vp, vp]
    lib.fsn_metric_sdr_workspace.argtypes = [i32, i64, C.POINTER(i64), C.POINTER(i64)]
    lib.fsn_metric_sdr.argtypes = [vp, vp, i32, i64, C.POINTER(i64), vp, i64, vp, vp]
    _LIB = lib
    return lib


def check(rc):
    if rc != 0:
        raise FsnError(f"fsnplus_b200 error {rc}: {load_library().fsn_last_error().decode()}")


DEFAULT_WS_CAP = 24e9


def ws_cap_bytes():
    """The workspace cap of a model created now: FSN_WS_CAP_GB (GB, > 0) or the default 24 GB (read by fsn_model_create)."""
    try:
        v = float(os.environ.get("FSN_WS_CAP_GB", ""))
    except ValueError:
        return DEFAULT_WS_CAP
    return v * 1e9 if v > 0 else DEFAULT_WS_CAP


def plan_forward(cfg, B, T, cap_bytes=None, force_window=0):
    """fsn_plan_forward: (clips per sub-batch, sub-band window in frames or 0, workspace bytes) of a plain forward of B clips of
    T frames under the cap (default: ws_cap_bytes()).  Computed on the host from the configuration; needs no GPU."""
    lib = load_library()
    bs, tw, nb = C.c_int32(), C.c_int32(), C.c_int64()
    cap = ws_cap_bytes() if cap_bytes is None else float(cap_bytes)
    check(lib.fsn_plan_forward(C.byref(cfg), int(B), int(T), cap, int(force_window), C.byref(bs), C.byref(tw), C.byref(nb)))
    return bs.value, tw.value, nb.value


def plan_forward_bins(cfg, B, T, cap_bytes=None, force_window=0, force_bins=0):
    """fsn_plan_forward_bins: plan_forward's (clips per sub-batch, window, workspace bytes) with the sub-band TCN's bin chunk, as
    (Bs, Tw, Fc, bytes); Fc = 0 means unchunked (always for LSTM / GRU).  force_bins: 0, or the FSN_SB_CHUNK value.  Needs no GPU."""
    lib = load_library()
    bs, tw, fc, nb = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
    cap = ws_cap_bytes() if cap_bytes is None else float(cap_bytes)
    check(lib.fsn_plan_forward_bins(C.byref(cfg), int(B), int(T), cap, int(force_window), int(force_bins), C.byref(bs), C.byref(tw),
                                    C.byref(fc), C.byref(nb)))
    return bs.value, tw.value, fc.value, nb.value


def stream_chunk_plan(cfg, n_active, K, cap_bytes=None):
    """fsn_stream_chunk_plan: (sessions per sub-batch, window in frames or 0, scratch bytes of one sub-batch) of a streaming chunk call
    with n_active stepping sessions of K frames under the cap (default: ws_cap_bytes()).  Needs no GPU."""
    lib = load_library()
    bs, tw, nb = C.c_int32(), C.c_int32(), C.c_int64()
    cap = ws_cap_bytes() if cap_bytes is None else float(cap_bytes)
    check(lib.fsn_stream_chunk_plan(C.byref(cfg), int(n_active), int(K), cap, C.byref(bs), C.byref(tw), C.byref(nb)))
    return bs.value, tw.value, nb.value


def lengths_arg(lengths, B):
    """``lengths`` (None, a sequence of ints or a 1-D CPU integer tensor of length B) as a C int64 array, or None."""
    if lengths is None:
        return None
    if hasattr(lengths, "is_cuda"):
        if lengths.is_cuda or lengths.is_floating_point() or lengths.is_complex() or lengths.dim() != 1:
            raise ValueError("lengths must be a 1-D CPU integer tensor or a sequence of ints")
        lengths = lengths.tolist()
    lengths = [int(n) for n in lengths]
    if len(lengths) != B:
        raise ValueError(f"lengths has {len(lengths)} entries for a batch of {B}")
    return (C.c_int64 * B)(*lengths)


def atten_arg(atten_lim_db, B):
    """An attenuation limit in dB (DESIGN.md §3.18) as a C float array of B values, or None: ``atten_lim_db`` is None (no limit), one
    number (every clip or slot) or B numbers (a sequence or a 1-D CPU tensor).  float('inf') is no limit; the library refuses a negative
    or NaN value, naming the clip or slot."""
    if atten_lim_db is None:
        return None
    if hasattr(atten_lim_db, "is_cuda"):
        if atten_lim_db.is_cuda or atten_lim_db.is_complex() or atten_lim_db.dim() > 1:
            raise ValueError("atten_lim_db must be a number, a sequence of numbers or a 0-/1-D CPU tensor")
        atten_lim_db = atten_lim_db.tolist()
    if isinstance(atten_lim_db, (int, float)):
        vals = [float(atten_lim_db)] * B
    else:
        vals = [float(v) for v in atten_lim_db]
        if len(vals) != B:
            raise ValueError(f"atten_lim_db has {len(vals)} entries for {B} clips / slots")
    return (C.c_float * B)(*vals)


def atten_floor(db):
    """The floor lam = 10^(-db / 20) of an attenuation limit of ``db`` dB, computed in double and rounded to float32 as the library
    does (float('inf'): 0.0, no limit)."""
    import numpy as np
    return float(np.float32(10.0 ** (-float(db) / 20.0)))


def plan_audio(cfg, B, L, lengths=None, cap_bytes=None, force_window=0, force_bins=0):
    """fsn_plan_audio: the (Bs, Tw, Fc, bytes) plan of the audio call (fsn_model_enhance_audio) for B clips in rows of L samples, each
    ``lengths[b]`` long (None: L), after the call's own checks (FsnError with its message).  Needs no GPU."""
    lib = load_library()
    bs, tw, fc, nb = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
    cap = ws_cap_bytes() if cap_bytes is None else float(cap_bytes)
    check(lib.fsn_plan_audio(C.byref(cfg), int(B), int(L), lengths_arg(lengths, B), cap, int(force_window), int(force_bins),
                             C.byref(bs), C.byref(tw), C.byref(fc), C.byref(nb)))
    return bs.value, tw.value, fc.value, nb.value
