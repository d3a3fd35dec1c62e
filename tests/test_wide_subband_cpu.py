"""CPU: wide sub-band inputs (64 < Isb <= 128, DESIGN.md §3.3).  The fp64 oracle against the reference's goldens, the workspace the
plan counts for a wide input (the 128-half input rows and layer 0's Gin), and the create-time limits.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from oracle import fsn_oracle as O

# golden: (model kind, config changes, small geometry)
GOLDENS = {
    "plus_small_wide70": ("plus", dict(sb_num_neighbors=3, fb_num_neighbors=10), True),
    "plus_small_wide128": ("plus", dict(sb_num_neighbors=2, fb_num_neighbors=20), True),
    "plus_small_wide70_GRU": ("plus", dict(sb_num_neighbors=3, fb_num_neighbors=10, sequence_model="GRU"), True),
    "fsn_small_wide66": ("fsn", dict(sb_num_neighbors=20, fb_num_neighbors=12), True),
    "fsn_small_wide128": ("fsn", dict(sb_num_neighbors=31, fb_num_neighbors=32), True),
    "plus_default_wide124": ("plus", dict(sb_num_neighbors=15, fb_num_neighbors=15), False),
}


def golden_cfg(name):
    """The configuration of a wide golden (tests/golden/make_golden_wide.py)."""
    kind, extra, small = GOLDENS[name]
    if kind == "plus":
        c = O.default_plus_config()
        if small:
            c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    else:
        c = O.default_fsn_config()
        c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64, fb_model_hidden_size=48, norm_type="cumulative_laplace_norm")
    c.update(extra)
    return kind, c


def isb(kind, c):
    return 2 * c["sb_num_neighbors"] + 1 + (3 if kind == "plus" else 1) * (2 * c["fb_num_neighbors"] + 1)


def golden_inputs(golden, name):
    """(mag, real, imag) of a wide golden: plus_small's inputs, or plus_default's 3 s clip"""
    src = golden("plus_small" if GOLDENS[name][2] else "plus_default")
    return src["mag"], src["real"], src["imag"]


def oracle(golden, name):
    kind, c = golden_cfg(name)
    g = golden(name)
    m, r, i = golden_inputs(golden, name)
    if kind == "plus":
        p = O.make_params_plus(c, seed=int(g["seed"]), lstm_scale=float(g["lstm_scale"]) if "lstm_scale" in g else 1.0)
        return O.fullsubnet_plus_forward(p, c, m, r, i), g["out"]
    p = O.make_params_fsn(c, seed=int(g["seed"]), lstm_scale=float(g["lstm_scale"]) if "lstm_scale" in g else 1.0)
    return O.fullsubnet_forward(p, c, m), g["out"]


@pytest.mark.parametrize("name", list(GOLDENS))
def test_oracle_matches_reference(golden, name):
    kind, c = golden_cfg(name)
    assert 64 < isb(kind, c) <= 128
    got, want = oracle(golden, name)
    err = O.rel_l2(got, want)
    print(f"{name}: Isb {isb(kind, c)} oracle-vs-reference rel-L2 {err:.2e}")
    assert err < 1e-6                                                   # the goldens are stored in fp32


def _cfg(kind="plus", **over):
    from fsnplus_b200.model import FullSubNet_Plus, Model
    c = (O.default_plus_config() if kind == "plus" else O.default_fsn_config())
    c.update(over)
    return (FullSubNet_Plus if kind == "plus" else Model)(**c)._cfg


def _bytes(cfg, B, T, Tw=0):
    """Exact workspace of (B, T, Tw): a forced (or no) window under an unlimited cap keeps the whole batch."""
    from fsnplus_b200 import _lib
    bs, tw, n = _lib.plan_forward(cfg, B, T, 1e18, Tw)
    assert (bs, tw) == (B, Tw)
    return n


@pytest.mark.parametrize("kind,sb,fb,L,B,T,Tw", [
    ("plus", 15, 15, 2, 4, 188, 0),          # Isb 124: default FullSubNet+ neighbourhood at 15 / 15
    ("plus", 15, 6, 1, 3, 100, 0),           # Isb 70, one layer: layer 0's Gin is the only one
    ("plus", 2, 20, 3, 2, 300, 64),          # Isb 128, windowed: the window's rows only
    ("fsn", 20, 12, 2, 5, 77, 0),            # fullsubnet.Model, Isb 66
    ("fsn", 31, 32, 1, 1, 400, 96),          # fullsubnet.Model, Isb 128, one layer, windowed
])
def test_plan_counts_the_wide_input(built_lib, kind, sb, fb, L, B, T, Tw):
    """A wide model's plan holds the narrow model's workspace plus the wider input rows and (one layer) layer 0's Gin."""
    wide = _cfg(kind, sb_num_neighbors=sb, fb_num_neighbors=fb, num_layers=L)
    narrow = _cfg(kind, sb_num_neighbors=sb, fb_num_neighbors=0, num_layers=L)
    F, H = wide.num_freqs, wide.sb_hidden
    assert isb(kind, dict(sb_num_neighbors=sb, fb_num_neighbors=fb)) > 64 >= isb(kind, dict(sb_num_neighbors=sb, fb_num_neighbors=0))
    ntp = ((B * F + 127) // 128 + 1) // 2 * 2                          # whole pairs of 128-row tiles
    frames = Tw if Tw else T + wide.look_ahead
    rows = ntp * frames * 128                                           # the GEMM's M: (tile, frame, row)
    extra = rows * (256 - 128)                                          # input rows of 128 halves instead of 64
    if L == 1:
        extra += rows * 4 * H * 2                                       # layer 0's Gin (deeper layers already hold one)
    assert _bytes(wide, B, T, Tw) - _bytes(narrow, B, T, Tw) == extra


# fsn_plan_forward bytes of Isb <= 64 configurations, as the release before wide inputs computed them
NARROW = [
    (dict(kind="plus"), 4, 188, 0, 988753168),
    (dict(kind="plus", sb_num_neighbors=10, fb_num_neighbors=1), 3, 100, 0, 425400588),
    (dict(kind="plus", num_layers=1), 2, 300, 64, 24112008),
    (dict(kind="fsn", norm_type="cumulative_laplace_norm"), 5, 77, 0, 491319552),
    (dict(kind="fsn", sb_num_neighbors=31, fb_num_neighbors=0, num_layers=1), 1, 400, 96, 23716852),
]


@pytest.mark.parametrize("over,B,T,Tw,want", NARROW)
def test_plan_of_narrow_inputs_unchanged(built_lib, over, B, T, Tw, want):
    over = dict(over)
    assert _bytes(_cfg(over.pop("kind"), **over), B, T, Tw) == want


def _create(cfg):
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    h = C.c_void_p()
    rc = lib.fsn_model_create(C.byref(cfg), C.byref(h))
    if rc == 0:
        lib.fsn_model_destroy(h)
    return rc, lib.fsn_last_error().decode()


def test_limits(built_lib):
    # Isb = 2 (sb + k fb) + k + 1 is even for both model kinds (k = 1, 3), so 130 is the smallest input refused: on every path, and the
    # message names 128
    rc, msg = _create(_cfg("fsn", sb_num_neighbors=32, fb_num_neighbors=32))           # 65 + 65
    assert rc == -1 and "130" in msg and "128" in msg, msg
    rc, msg = _create(_cfg("plus", sb_num_neighbors=3, fb_num_neighbors=20))           # 7 + 3 * 41
    assert rc == -1 and "130" in msg and "128" in msg, msg
    rc, msg = _create(_cfg("fsn", sb_num_neighbors=32, fb_num_neighbors=31, lstm_impl="mma"))   # 65 + 63 = 128: accepted
    assert rc != -1, msg
    # a sub-band TCN keeps its own limit of 64 (Isb 66 = 9 + 3 * 19), with a message that names the TCN
    rc, msg = _create(_cfg("plus", sequence_model="TCN", sb_num_neighbors=4, fb_num_neighbors=9, num_freqs=33))
    assert rc == -1 and "66" in msg and "64" in msg and "TCN" in msg, msg


def test_state_payload_does_not_depend_on_isb(built_lib):
    """A streaming session's saved state is H, the norm sums and the audio rings: the same bytes at Isb 128 as at Isb 32."""
    from fsnplus_b200 import _lib
    for mode in (_lib.STATE_MODE_MASK, _lib.STATE_MODE_AUDIO):
        wide = _lib.state_layout(_cfg("fsn", sb_num_neighbors=31, fb_num_neighbors=32, norm_type="cumulative_laplace_norm"), mode)
        narrow = _lib.state_layout(_cfg("fsn", sb_num_neighbors=15, fb_num_neighbors=0, norm_type="cumulative_laplace_norm"), mode)
        assert wide == narrow and wide[0] > 0
