"""Attenuation limits (DESIGN.md §3.18) without a GPU: the dB -> floor conversion, the Python wrappers' argument handling, the
--atten_lim_db flag of tools.inference, and the ctypes declarations of the new calls against include/fsnplus_b200.h."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ["fsn_model_forward_enhance_lim", "fsn_model_enhance_audio_lim", "fsn_stream_set_atten_lim", "fsn_chunk_stream_set_atten_lim"]


def test_floor_conversion():
    from fsnplus_b200 import _lib
    assert _lib.atten_floor(0.0) == 1.0
    assert _lib.atten_floor(float("inf")) == 0.0
    for db in (3.0, 6.0, 12.0, 20.0, 40.0, 100.0):
        lam = _lib.atten_floor(db)
        assert lam == float(np.float32(10.0 ** (-db / 20.0)))
        assert abs(20.0 * math.log10(lam) + db) < 1e-5                  # the floor is L dB below unity, to float32 rounding
    assert _lib.atten_floor(2000.0) == 0.0                               # underflows to no limit
    assert abs(_lib.atten_floor(6.0) - 0.5011872) < 1e-7


def test_atten_arg():
    from fsnplus_b200 import _lib
    assert _lib.atten_arg(None, 4) is None
    a = _lib.atten_arg(6, 3)
    assert list(a) == [6.0, 6.0, 6.0] and isinstance(a, C.Array) and a._type_ is C.c_float
    assert list(_lib.atten_arg([1, float("inf"), 0], 3)) == [1.0, float("inf"), 0.0]
    assert list(_lib.atten_arg(torch.tensor([2.0, 3.0]), 2)) == [2.0, 3.0]
    assert list(_lib.atten_arg(torch.tensor(5.0), 2)) == [5.0, 5.0]
    # a bad value passes through: the library refuses it with the clip or slot named
    assert math.isnan(_lib.atten_arg([float("nan")], 1)[0]) and _lib.atten_arg([-1.0], 1)[0] == -1.0
    with pytest.raises(ValueError, match="2 entries for 3"):
        _lib.atten_arg([1.0, 2.0], 3)
    with pytest.raises(ValueError):
        _lib.atten_arg(torch.zeros(2, 2), 4)


def test_wrappers_refuse_before_the_device():
    """enhance_spectrum(pipelined=True) with a limit is a ValueError; enhance_batch with a limit needs the library on CUDA."""
    from fsnplus_b200 import inference as inf
    from fsnplus_b200.model import FullSubNet_Plus
    from oracle import fsn_oracle as O
    cfg = O.default_plus_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    m = FullSubNet_Plus(**cfg).eval()
    x = torch.zeros(1, 1, 33, 8)
    with pytest.raises(ValueError, match="pipelined"):
        m.enhance_spectrum(x, x, x, pipelined=True, atten_lim_db=6.0)
    with pytest.raises(ValueError, match="CUDA"):
        inf.enhance_batch(lambda *a, **k: None, torch.zeros(1, 4096), 64, 32, 64, atten_lim_db=6.0)
    with pytest.raises(ValueError, match="CUDA"):
        inf.enhance_ragged(lambda *a, **k: None, [torch.zeros(4096)], 64, 32, 64, atten_lim_db=6.0)


def test_inference_flag(monkeypatch):
    from fsnplus_b200.tools import inference as tool
    seen = {}
    monkeypatch.setattr(tool, "load_toml", lambda p: {"dataset": {"args": {"dataset_dir_list": []}}})
    monkeypatch.setattr(tool, "run", lambda *a, **k: seen.update(k))
    tool.main(["-C", "c.toml", "-M", "m.tar", "-O", "out"])
    assert seen["atten_lim_db"] is None                                  # default: no limit, today's output
    tool.main(["-C", "c.toml", "-M", "m.tar", "-O", "out", "--atten_lim_db", "12"])
    assert seen["atten_lim_db"] == 12.0
    tool.main(["-C", "c.toml", "-M", "m.tar", "-O", "out", "--atten_lim_db", "inf"])
    assert seen["atten_lim_db"] == float("inf")
    for bad in ("-3", "nan"):
        with pytest.raises(SystemExit):
            tool.main(["-C", "c.toml", "-M", "m.tar", "-O", "out", "--atten_lim_db", bad])


def _header_args(name):
    text = open(os.path.join(ROOT, "include", "fsnplus_b200.h")).read()
    m = re.search(r"int\s+" + name + r"\(([^;]*)\);", text)
    assert m, name
    return [a.strip() for a in m.group(1).replace("\n", " ").split(",")]


def test_ctypes_match_header():
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    host = {"float*": C.POINTER(C.c_float), "int32_t*": C.POINTER(C.c_int32), "int64_t*": C.POINTER(C.c_int64)}
    scalar = {"int32_t": C.c_int32, "int64_t": C.c_int64}
    for name in NEW:
        assert name in _lib.SYMBOLS
        fn = getattr(lib, name)
        args = _header_args(name)
        assert len(fn.argtypes) == len(args), name
        for a, t in zip(args, fn.argtypes):
            m = re.fullmatch(r"(?:const\s+)?([A-Za-z_0-9]+\s*\**)\s*([A-Za-z_0-9]+)", a)
            typ, arg = m.group(1).replace(" ", ""), m.group(2)
            if arg.startswith("h_"):                                    # host arrays: typed pointers
                assert t == host[typ], (name, a, t)
            elif typ.endswith("*"):                                     # handles, device buffers, the stream
                assert t == C.c_void_p, (name, a, t)
            else:
                assert t == scalar[typ], (name, a, t)


def test_limits_are_refused_without_a_gpu():
    """The setters check their arguments on the host: a null handle is refused with a message, without touching a device."""
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    s = (C.c_int32 * 1)(0)
    v = (C.c_float * 1)(6.0)
    assert lib.fsn_stream_set_atten_lim(None, 1, s, v) == -1 and b"st is null" in lib.fsn_last_error()
    assert lib.fsn_chunk_stream_set_atten_lim(None, 1, s, v) == -1 and b"cs is null" in lib.fsn_last_error()
