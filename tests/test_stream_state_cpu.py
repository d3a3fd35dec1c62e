"""CPU: the payload layout of saved streaming sessions (fsn_stream_state_layout, DESIGN.md §3.11) follows its formula -- segments in a
fixed order at 16-byte aligned offsets, a stride that is a multiple of 256 -- the configurations that cannot stream are rejected, and
the ctypes mirror of fsn_slot_meta has the library's size.  No GPU needed."""
import ctypes as C

import pytest


def _cfg(F=257, L=2, rnn="LSTM", la=2, fb=512, sb=384, norm="cumulative_laplace_norm", kind=1):
    from fsnplus_b200 import _lib
    c = _lib.FsnConfig()
    c.model_kind, c.num_freqs, c.look_ahead = kind, F, la
    c.sb_num_neighbors, c.fb_num_neighbors = 7, 0
    c.fb_hidden, c.sb_hidden, c.num_layers, c.output_size = fb, sb, L, 2
    c.fb_act, c.sb_act, c.norm_type = 1, 0, _lib.NORM[norm]
    c.rnn_type = _lib.RNN[rnn]
    c.fast_math = 1
    return c


def _formula(F, L, la, fb, sb, mode):
    """Payload offsets of every segment and the stride, from the handle's buffer shapes."""
    H = F - 1
    seg = [16, F * 16, L * fb * 2, L * fb * 4, L * F * sb * 2, L * F * sb * 4]       # cum_in, cum_sb, fb h, fb c, sb h, sb c
    if mode == 2:
        seg += [3 * H * 4, (la + 1) * F * 8, H * 4]                                  # history ring, spectrum ring, overlap tail
    off, o = [], 0
    for s in seg:
        off.append(o)
        o += (s + 15) // 16 * 16
    return off, (o + 255) // 256 * 256, sum(seg)


@pytest.mark.parametrize("F", [33, 65, 257, 513])
@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("rnn", ["LSTM", "GRU"])
@pytest.mark.parametrize("mode", [1, 2])
def test_layout_matches_formula(built_lib, F, L, rnn, mode):
    from fsnplus_b200 import _lib
    for la in range(4):
        fb, sb = (512, 384) if F == 257 else (96, 64)
        stride, meta = _lib.state_layout(_cfg(F, L, rnn, la, fb, sb), mode)
        off, want, raw = _formula(F, L, la, fb, sb, mode)
        assert stride == want and stride % 256 == 0 and stride >= raw and all(o % 16 == 0 for o in off)
        assert meta == C.sizeof(_lib.FsnSlotMeta)


def test_default_payload_bytes(built_lib):
    """Config #4 (F 257, full-band H 512, sub-band H 384, 2 layers, look-ahead 2): 1 194 528 state bytes per mask session, 1 204 792
    per audio session, rounded up to the 256-byte stride."""
    from fsnplus_b200 import _lib
    for mode, raw in ((1, 1194528), (2, 1204792)):
        assert _formula(257, 2, 2, 512, 384, mode)[2] == raw
        assert _lib.state_layout(_cfg(), mode)[0] == {1: 1194752, 2: 1204992}[mode]


def test_meta_mirror_size(built_lib):
    from fsnplus_b200 import _lib
    assert _lib.state_layout(_cfg(), 1)[1] == C.sizeof(_lib.FsnSlotMeta) == 128


def test_layout_rejects(built_lib):
    from fsnplus_b200 import _lib
    lib = built_lib
    nb, mb = C.c_int64(), C.c_int32()

    def call(cfg, mode):
        return lib.fsn_stream_state_layout(C.byref(cfg), mode, C.byref(nb), C.byref(mb))

    assert call(_cfg(kind=_lib.KIND_PLUS), 1) == -1 and "FullSubNet+" in lib.fsn_last_error().decode()
    for norm in ("offline_laplace_norm", "offline_gaussian_norm"):
        assert call(_cfg(norm=norm), 1) == -1 and "cumulative" in lib.fsn_last_error().decode()
    for mode in (0, 3, -1):
        assert call(_cfg(), mode) == -1 and f"mode {mode}" in lib.fsn_last_error().decode()
    assert call(_cfg(F=100, fb=96, sb=64), 1) == 0                                 # masks stream at any num_freqs ...
    assert call(_cfg(F=100, fb=96, sb=64), 2) == -1 and "num_freqs 100" in lib.fsn_last_error().decode()   # ... audio needs a power-of-two n_fft
    assert lib.fsn_stream_state_layout(None, 1, C.byref(nb), C.byref(mb)) == -1
    assert call(_cfg(norm="cumulative_layer_norm"), 2) == 0
