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
    "fsn_model_forward_host", "fsn_model_forward_host_async", "fsn_model_sync_host", "fsn_model_submit", "fsn_model_wait", "fsn_model_forward_enhance", "fsn_model_submit_enhance", "fsn_model_forward_ragged", "fsn_model_forward_enhance_ragged", "fsn_model_last_lane", "fsn_model_wait_lane", "fsn_apply_cirm", "fsn_stream_create", "fsn_stream_step", "fsn_stream_destroy", "fsn_model_get_stage", "fsn_model_last_launch_count", "fsn_model_last_lstm_impl", "fsn_model_last_lstm_ms", "fsn_model_lstm_ms_history", "fsn_model_timeline",
    "fsn_plan_forward", "fsn_model_workspace_bytes", "fsn_model_last_plan", "fsn_model_plan", "fsn_model_release_workspace",
    "fsn_plan_forward_bins", "fsn_model_plan_bins", "fsn_model_last_plan_bins",
    "fsn_sw128_offset", "fsn_tc5_weight_stream_bytes", "fsn_tc5_pack_weights", "fsn_tc5_gate_row", "fsn_tc5r_weight_stream_bytes", "fsn_tc5r_pack_layer",
    "fsn_gemm_f16", "fsn_gemm_f16_tile_n",
]


class FsnError(RuntimeError):
    pass


class FsnConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("model_kind", "num_freqs", "look_ahead", "sb_num_neighbors", "fb_num_neighbors",
                                          "fb_hidden", "sb_hidden", "num_layers", "output_size", "fb_act", "sb_act",
                                          "norm_type")] + [("kersize", C.c_int32 * 3), ("lstm_impl", C.c_int32),
                                                           ("fast_math", C.c_int32), ("channel_attention", C.c_int32), ("rnn_type", C.c_int32), ("subband_num", C.c_int32), ("tcn_causal", C.c_int32),
                                                           ("sb_tcn", C.c_int32)]


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
    lib.fsn_stream_destroy.argtypes = [vp]
    lib.fsn_stream_destroy.restype = None
    lib.fsn_apply_cirm.argtypes = [vp, vp, vp, i32, i32, i32, vp]
    lib.fsn_model_get_stage.argtypes = [vp, C.c_char_p, vp, i64, vp]
    lib.fsn_model_last_launch_count.argtypes = [vp]
    lib.fsn_model_last_launch_count.restype = i64
    lib.fsn_model_last_lstm_impl.argtypes = [vp]
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
