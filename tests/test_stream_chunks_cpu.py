"""CPU: the plan of the streaming chunk call (fsn_stream_chunk_plan, DESIGN.md §3.13) -- its byte count from the buffer shapes, the cap
respected, sub-batches before windows -- its error messages, and the ctypes signature of fsn_stream_step_chunk.  No GPU needed."""
import ctypes as C

import pytest


def _cfg(F=257, L=2, rnn="LSTM", la=2, fb=512, sb=384, norm="cumulative_laplace_norm", kind=1, impl="auto"):
    from fsnplus_b200 import _lib
    c = _lib.FsnConfig()
    c.model_kind, c.num_freqs, c.look_ahead = kind, F, la
    c.sb_num_neighbors, c.fb_num_neighbors = 7, 0
    c.fb_hidden, c.sb_hidden, c.num_layers, c.output_size = fb, sb, L, 2
    c.fb_act, c.sb_act, c.norm_type = 1, 0, _lib.NORM[norm]
    c.rnn_type = _lib.RNN[rnn]
    c.lstm_impl = _lib.LSTM_IMPL[impl]
    c.fast_math = 1
    return c


def _bytes(F, L, H, bs, K, tw):
    """The layer-wise scratch of one sub-batch from the buffer shapes: images [tile pairs, tw, 128, 64] fp16, Gin [M, 4H] and the
    layer output [M, H] fp16 (layers > 0), the h carry [L, tile pairs x 128, H] fp16, the c carry [L, tile pairs x 128, H] fp32 and
    the compact masks [bs, 2, F, K] fp32."""
    tp = ((bs * F + 127) // 128 + 1) // 2 * 2
    M = tp * tw * 128
    gin = M * 4 * H * 2 + M * H * 2 if L > 1 else 0
    return tp * tw * 16384 + gin + L * tp * 128 * H * 2 + L * tp * 128 * H * 4 + bs * 2 * F * K * 4


@pytest.mark.parametrize("F,H,L", [(257, 384, 2), (65, 64, 2), (65, 128, 1), (129, 192, 3)])
@pytest.mark.parametrize("K", [1, 3, 4, 32, 37, 64])
def test_plan_bytes_and_cap(built_lib, F, H, L, K):
    from fsnplus_b200 import _lib
    c = _cfg(F=F, sb=H, L=L, fb=96 if F != 257 else 512)
    for n in (1, 3, 80, 700, 1280):
        bs, tw, nb = _lib.stream_chunk_plan(c, n, K, cap_bytes=1e15)
        assert (bs, tw) == (n, 0) and nb == _bytes(F, L, H, n, K, K)
        for cap in (24e9, 2e9, 1e8):
            bs, tw, nb = _lib.stream_chunk_plan(c, n, K, cap_bytes=cap)
            assert nb == _bytes(F, L, H, bs, K, tw or K)
            if tw == 0:
                assert nb <= cap or bs == 1
                nsub = -(-n // bs)
                assert bs == -(-n // nsub)                               # equal sub-batches
                if bs < n:                                               # the next larger equal split would not fit
                    assert _bytes(F, L, H, -(-n // (nsub - 1)), K, K) > cap
            else:
                assert bs == 1 and tw % 4 == 0 and tw < K and _bytes(F, L, H, 1, K, K) > cap


def test_plan_default_geometry(built_lib):
    """Config #4 at K = 32: ~1 MB per session-frame, so about 700 sessions per sub-batch under the default 24 GB cap; under a cap below
    one session's 32 frames the chunk runs one session at a time in windows."""
    from fsnplus_b200 import _lib
    c = _cfg()
    per = _bytes(257, 2, 384, 100, 32, 32) / (100 * 32)
    assert 0.9e6 < per < 1.2e6
    bs, tw, nb = _lib.stream_chunk_plan(c, 1280, 32, cap_bytes=24e9)
    assert 600 <= bs <= 720 and tw == 0 and nb <= 24e9
    bs, tw, nb = _lib.stream_chunk_plan(c, 4, 32, cap_bytes=12e6)
    assert bs == 1 and 0 < tw < 32 and tw % 4 == 0 and nb <= 12e6


def test_plan_generic_path(built_lib):
    """lstm_impl = "mma" or a geometry the layer-wise kernels do not take: one piece, the images of the sessions."""
    from fsnplus_b200 import _lib
    for c in (_cfg(impl="mma"), _cfg(F=65, sb=96, fb=96)):
        F = c.num_freqs
        for n, K in ((1, 1), (80, 37), (1280, 64)):
            assert _lib.stream_chunk_plan(c, n, K, cap_bytes=1e6) == (n, 0, (n * F + 127) // 128 * K * 16384)


def test_plan_rejects(built_lib):
    from fsnplus_b200 import _lib
    lib = built_lib
    bs, tw, nb = C.c_int32(), C.c_int32(), C.c_int64()

    def call(cfg, n, K, cap=24e9):
        return lib.fsn_stream_chunk_plan(cfg if cfg is None else C.byref(cfg), n, K, cap, C.byref(bs), C.byref(tw), C.byref(nb))

    def err():
        return lib.fsn_last_error().decode()

    assert call(_cfg(kind=_lib.KIND_PLUS), 4, 8) == -1 and "FullSubNet+" in err()
    assert call(_cfg(norm="offline_laplace_norm"), 4, 8) == -1 and "cumulative" in err()
    for K in (0, -3):
        assert call(_cfg(), 4, K) == -1 and f"K = {K}" in err() and "at least 1 frame" in err()
    assert call(_cfg(), 0, 8) == -1 and "n_active = 0" in err()
    assert call(_cfg(), 4, 65535 * 256 - 3) == -1 and "chunk limit" in err()
    assert call(_cfg(), 4, 65535 * 256 - 4) == -1 and "num_freqs x K" in err() and "2^31 - 1" in err()
    assert call(_cfg(F=65, fb=96, sb=64), 1, 65535 * 256 - 4) == 0
    assert call(_cfg(), 4, 8, 0.0) == -1 and "cap" in err()
    assert call(None, 4, 8) == -1 and "cfg is null" in err()


def test_entry_point_signature(built_lib):
    from fsnplus_b200 import _lib
    lib = built_lib
    assert "fsn_stream_step_chunk" in _lib.SYMBOLS and "fsn_stream_chunk_plan" in _lib.SYMBOLS
    vp, i32 = C.c_void_p, C.c_int32
    assert lib.fsn_stream_step_chunk.argtypes == [vp, vp, i32, vp, vp, vp, vp]
    assert lib.fsn_stream_step_chunk(None, None, 4, None, None, None, None) == -1 and "st is null" in lib.fsn_last_error().decode()
