"""FullSubNet+ with a TCN sub-band model (sequence_model = "TCN", reference fullsubnet_plus.py:45,102-110): the parts that need no GPU.

The state-dict contract of the Python mirror, the configuration checks of fsn_model_create, the numpy oracle and the CPU torch port
against the goldens made from the unmodified reference, and the inference CLI building the model from a TOML.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))


def _small_tcn(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, sequence_model="TCN")
    c.update(over)
    return c


@pytest.mark.parametrize("hidden", [32, 384, 7])
def test_state_dict_contract(hidden):
    """The oracle's TCN parameters load strict=True; like the reference, sb_model_hidden_size is unused (any value constructs)."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _small_tcn(sb_model_hidden_size=hidden)
    params = S.make_params(cfg, seed=15)
    m = FullSubNet_Plus(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    sd = m.state_dict()
    isb = 7 + 3
    assert sd["sb_model.sequence_model.0.conv1x1.weight"].shape == (512, isb, 1)
    assert sd["sb_model.sequence_model.7.sconv.weight"].shape == (isb, 512, 1)
    assert sd["sb_model.fc_output_layer.weight"].shape == (2, isb)
    assert m._cfg.sb_tcn == 1 and m._cfg.rnn_type == 0


def test_flops_include_the_tcn_term():
    """28.41 GFLOP per 3 s clip (T' = 190) at the default geometry: T' F [8 (2 * 2 Isb 512 + 2 * 3 * 512) + 2 Isb O]."""
    f = S.flops(dict(O.default_plus_config(), sequence_model="TCN"), 188)
    assert f == 190 * 257 * (8 * (2 * 2 * 34 * 512 + 2 * 3 * 512) + 2 * 34 * 2)
    assert abs(f / 1e9 - 28.41) < 0.01


def test_create_accepts_tcn_and_checks_the_input_size(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus

    def create(cfg_kw, **over):
        cfg = _lib.FsnConfig.from_buffer_copy(FullSubNet_Plus(**cfg_kw)._cfg)
        for k, v in over.items():
            setattr(cfg, k, v)
        h = C.c_void_p()
        rc = built_lib.fsn_model_create(C.byref(cfg), C.byref(h))
        if rc == 0:
            built_lib.fsn_model_destroy(h)
        return rc, built_lib.fsn_last_error()

    dflt = dict(O.default_plus_config(), sequence_model="TCN")
    for over in ({}, {"sb_hidden": 100}, {"sb_hidden": 0}):             # the TCN has no hidden-size constraint
        rc, msg = create(dflt, **over)
        assert rc == 0 if torch.cuda.is_available() else (rc == -2 and b"no CPU fallback" in msg), (over, rc, msg)
    rc, msg = create(dict(dflt, sb_num_neighbors=15, fb_num_neighbors=2))   # Isb = 31 + 3 * 5 = 46 <= 64
    assert rc == 0 if torch.cuda.is_available() else rc == -2, msg
    rc, msg = create(dict(dflt, fb_num_neighbors=3))                     # Isb = 31 + 3 * 7 = 52
    assert rc == 0 if torch.cuda.is_available() else rc == -2, msg
    rc, msg = create(dict(dflt, fb_num_neighbors=6))                     # Isb = 31 + 3 * 13 = 70
    assert rc == -1 and b"sub-band input size 70 > 64" in msg
    rc, msg = create(dflt, sb_tcn=2)
    assert rc == -1 and b"sb_tcn" in msg
    rc, msg = create(dflt, model_kind=_lib.KIND_FSN)
    assert rc == -1 and b"FullSubNet_Plus" in msg


def test_oracle_matches_reference_goldens(golden):
    g = golden("plus_small_sbTCN")
    gi = golden("plus_small")
    cfg = _small_tcn()
    params = S.make_params(cfg, seed=int(g["seed"]))
    st = {}
    out = S.forward(params, cfg, gi["mag"], gi["real"], gi["imag"], stages=st)
    assert O.rel_l2(out, g["out"]) < 1e-6
    assert O.rel_l2(st["fb_out"], g["fb_out"]) < 1e-6
    assert O.rel_l2(st["sb_in"], g["sb_in"]) < 1e-6


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-4), (torch.float64, 1e-6)])
def test_torch_port_matches_reference_goldens(golden, dtype, tol):
    cfg = _small_tcn()
    g, gi = golden("plus_small_sbTCN"), golden("plus_small")
    port = S.TcnPort(S.make_params(cfg, seed=int(g["seed"])), cfg, dtype=dtype)
    out = np.concatenate([port.forward(*(torch.from_numpy(gi[k][b:b + 1]).to(dtype) for k in ("mag", "real", "imag"))).numpy()
                          for b in range(gi["mag"].shape[0])])
    assert O.rel_l2(out, g["out"]) < tol


def test_torch_port_default_geometry_golden(golden):
    """One 3 s clip at the default geometry (F = 257, Isb = 34) through the fp32 port, in chunks of bins."""
    g, gd = golden("plus_default_sbTCN"), golden("plus_default")
    cfg = dict(O.default_plus_config(), sequence_model="TCN")
    port = S.TcnPort(S.make_params(cfg, seed=int(g["seed"])), cfg)
    out = port.forward(*(torch.from_numpy(gd[k]) for k in ("mag", "real", "imag"))).numpy()
    assert out.shape == g["out"].shape == (1, 2, 257, 188)
    assert O.rel_l2(out, g["out"]) < 1e-4


def test_cli_builds_a_tcn_model_from_toml(tmp_path):
    """The inference command line builds the drop-in class from a TOML whose [model.args] say sequence_model = "TCN" and loads a
    reference-format checkpoint of it strictly."""
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200.tools import inference as cli
    src = open(os.path.join(HERE, "golden", "inference_reference.toml")).read()
    assert 'sequence_model = "LSTM"' in src
    p = tmp_path / "tcn.toml"
    p.write_text(src.replace('sequence_model = "LSTM"', 'sequence_model = "TCN"'))
    config = cli.load_toml(str(p))
    params = S.make_params(dict(O.default_plus_config(), sequence_model="TCN"), seed=0)
    ckpt = tmp_path / "tcn.tar"
    torch.save({"model": {k: torch.from_numpy(v) for k, v in params.items()}, "epoch": 3}, str(ckpt))
    model, epoch = cli.build_model(config["model"], str(ckpt), "cpu")
    assert isinstance(model, FullSubNet_Plus) and epoch == 3
    assert model._cfg.sb_tcn == 1
    assert torch.equal(model.state_dict()["sb_model.sequence_model.7.sconv.weight"],
                       torch.from_numpy(params["sb_model.sequence_model.7.sconv.weight"]))
