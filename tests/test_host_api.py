"""CPU: the C-ABI library loads and exports every symbol include/fsnplus_b200.h declares, the host-side
mirror reproduces the reference's constructor / state_dict contract, the kernel-layout packers are correct,
and the product path fails loudly without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(built_lib):
    header = open(os.path.join(ROOT, "include", "fsnplus_b200.h")).read()
    declared = set(re.findall(r"\b(fsn_[a-z0-9_]+)\s*\(", header))
    from fsnplus_b200 import _lib
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for name in declared:
        assert getattr(built_lib, name) is not None
    assert built_lib.fsn_version() >= 100


def test_state_dict_contract_plus():
    """Keys and shapes must equal the reference's state_dict (tests/golden/make_golden.py loaded the same
    dict into the unmodified reference with strict=True)."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    m = FullSubNet_Plus(**cfg)
    ref = O.make_params_plus(cfg, seed=0)
    sd = m.state_dict()
    assert set(sd.keys()) == set(ref.keys())
    for k, v in ref.items():
        assert tuple(sd[k].shape) == v.shape, k
    m.load_state_dict({k: torch.from_numpy(v) for k, v in ref.items()}, strict=True)
    assert sum(p.numel() for p in m.parameters()) == 8675102           # SURVEY.md section 6
    assert m.num_groups_in_drop_band == 2 and m.look_ahead == 2


@pytest.mark.parametrize("attn", ["SE", "ECA", "CBAM"])
def test_state_dict_contract_other_attentions(attn):
    """SE is the reference constructor's default (fullsubnet_plus.py:27); the same parameter dicts were loaded into the
    unmodified reference with strict=True by tests/golden/make_golden.py."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = dict(O.default_plus_config(), channel_attention_model=attn)
    if attn == "SE":
        del cfg["channel_attention_model"]                              # constructor default
    m = FullSubNet_Plus(**cfg)
    ref = O.make_params_plus(dict(cfg, channel_attention_model=attn), seed=0)
    sd = m.state_dict()
    assert set(sd.keys()) == set(ref.keys())
    for k, v in ref.items():
        assert tuple(sd[k].shape) == v.shape, k


def test_subband_num_mirrors_reference():
    """subband_num > 1: attention containers get F // subband_num + 1 channels (fullsubnet_plus.py:47-50); the forward raises
    for every attention but ECA, as the reference's does (shape mismatch on the real / imag branches, :157-163)."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = dict(O.default_plus_config(), subband_num=2)
    m = FullSubNet_Plus(**cfg)
    assert m.num_channels == 129
    assert tuple(m.state_dict()["channel_attention_real.fc1.weight"].shape) == (64, 129)
    assert tuple(m.state_dict()["channel_attention.smallConv1d.0.weight"].shape) == (129, 1, 3)
    x = torch.zeros(1, 1, 257, 8)
    with pytest.raises(RuntimeError):
        m(x, x, x)
    e = FullSubNet_Plus(**dict(cfg, channel_attention_model="ECA"))
    assert tuple(e.state_dict()["channel_attention.conv.weight"].shape) == (1, 1, 3)


def test_state_dict_contract_gru():
    from fsnplus_b200.model import FullSubNet_Plus, Model
    cfg = dict(O.default_plus_config(), sequence_model="GRU")
    sd, ref = FullSubNet_Plus(**cfg).state_dict(), O.make_params_plus(cfg, seed=0)
    assert set(sd.keys()) == set(ref.keys())
    assert all(tuple(sd[k].shape) == v.shape for k, v in ref.items())
    assert tuple(sd["sb_model.sequence_model.weight_hh_l1"].shape) == (3 * 384, 384)
    cfg = dict(O.default_fsn_config(), sequence_model="GRU")
    sd, ref = Model(**cfg).state_dict(), O.make_params_fsn(cfg, seed=0)
    assert set(sd.keys()) == set(ref.keys())
    assert all(tuple(sd[k].shape) == v.shape for k, v in ref.items())


def test_state_dict_contract_fsn():
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    m = Model(**cfg)
    ref = O.make_params_fsn(cfg, seed=1)
    sd = m.state_dict()
    assert set(sd.keys()) == set(ref.keys())
    for k, v in ref.items():
        assert tuple(sd[k].shape) == v.shape, k
    assert sum(p.numel() for p in m.parameters()) == 5637635


def test_constructor_errors_mirror_reference():
    from fsnplus_b200.model import FullSubNet_Plus, Model
    cfg = O.default_plus_config()
    with pytest.raises(AssertionError):
        FullSubNet_Plus(**{**cfg, "sequence_model": "RNN"})             # fullsubnet_plus.py:45
    with pytest.raises(NotImplementedError):
        FullSubNet_Plus(**{**cfg, "channel_attention_model": "XYZ"})    # fullsubnet_plus.py:70
    with pytest.raises(NotImplementedError):
        FullSubNet_Plus(**{**cfg, "norm_type": "forgetting_norm"})      # base_model.py:328
    with pytest.raises(AssertionError):
        Model(**{**O.default_fsn_config(), "sequence_model": "TCN"})    # fullsubnet.py:37


def test_no_cpu_fallback(built_lib):
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200 import _lib
    cfg = O.default_plus_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32)
    m = FullSubNet_Plus(**cfg).eval()
    x = torch.rand(1, 1, 33, 20)
    with pytest.raises(RuntimeError):
        m(x, x, x)                                                       # CPU tensors are refused
    with pytest.raises(AssertionError):
        m(x[0], x[0], x[0])                                              # dim() == 4 (fullsubnet_plus.py:136)
    with pytest.raises(NotImplementedError):
        m.train()(x, x, x)
    if not torch.cuda.is_available():
        h = C.c_void_p()
        rc = built_lib.fsn_model_create(C.byref(m._cfg), C.byref(h))
        assert rc == -2 and b"no CPU fallback" in built_lib.fsn_last_error()


def test_create_validates_the_configuration(built_lib):
    """fsn_model_create rejects bad configurations with FSN_EINVAL (-1) and a message before it ever touches a device."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus

    def create(**over):
        cfg = _lib.FsnConfig.from_buffer_copy(FullSubNet_Plus(**O.default_plus_config())._cfg)
        for k, v in over.items():
            setattr(cfg, k, v)
        h = C.c_void_p()
        rc = built_lib.fsn_model_create(C.byref(cfg), C.byref(h))
        if rc == 0:
            built_lib.fsn_model_destroy(h)
        return rc, built_lib.fsn_last_error()

    for over, needle in (({"model_kind": 7}, b"model_kind"), ({"num_freqs": 2}, b"geometry"), ({"sb_num_neighbors": 300}, b"reflect"),
                         ({"num_layers": 5}, b"num_layers"), ({"sb_hidden": 100}, b"multiple of 16"), ({"output_size": 0}, b"output_size"),
                         ({"norm_type": 9}, b"norm_type"), ({"channel_attention": 4}, b"channel_attention"), ({"rnn_type": 2}, b"rnn_type"),
                         ({"subband_num": 2}, b"ECA"), ({"channel_attention": _lib.ATTENTION["ECA"], "subband_num": 200}, b"subband_num")):
        rc, msg = create(**over)
        assert rc == -1 and needle in msg, (over, rc, msg)
    rc, msg = create()                                                   # a valid configuration gets as far as the device check
    assert rc == 0 if torch.cuda.is_available() else (rc == -2 and b"no CPU fallback" in msg)


def test_sw128_offsets(built_lib):
    seen = set()
    for r in range(128):
        for k in range(64):
            off = built_lib.fsn_sw128_offset(r, k)
            assert off == r * 128 + ((((k >> 3) ^ (r & 7)) & 7) << 4) + ((k & 7) << 1)
            seen.add(off)
    assert len(seen) == 128 * 64 and max(seen) == 128 * 128 - 2


def test_tc5_weight_stream_layout(built_lib):
    """The stream must hold, stage by stage in consumption order, 128 gate columns x 64 k tiles whose un-swizzled
    content is the slice of [W_ih | W_hh] the kernel's MMA schedule expects (gate column n of 32-unit chunk j =
    gates i,f,g,o of units 32 j + 8 (n // 32) + n % 8)."""
    I, H = 34, 128
    rng = np.random.default_rng(0)
    w = [rng.standard_normal(s).astype(np.float32) for s in ((4 * H, I), (4 * H, H), (4 * H, H), (4 * H, H))]
    nbytes = built_lib.fsn_tc5_weight_stream_bytes(I, H)
    NCH, KBH = H // 32, H // 64
    assert nbytes == (NCH * (1 + KBH) + NCH * 2 * KBH) * 16384
    buf = np.zeros(nbytes // 2, np.uint16)
    vp = lambda a: C.c_void_p(a.ctypes.data)
    assert built_lib.fsn_tc5_pack_weights(I, H, vp(w[0]), vp(w[1]), vp(w[2]), vp(w[3]), vp(buf)) == 0
    st = buf.view(np.float16).reshape(-1, 8192)
    off = np.array([[built_lib.fsn_sw128_offset(n, k) // 2 for k in range(64)] for n in range(128)])
    s = 0
    for layer in range(2):
        for j in range(NCH):
            rows = np.array([built_lib.fsn_tc5_gate_row(H, j, n) for n in range(128)])
            assert list(rows[:3]) == [32 * j, 32 * j + 1, 32 * j + 2] and rows[8] == H + 32 * j and rows[32] == 32 * j + 8
            blocks = []
            if layer == 0:
                x = np.zeros((128, 64), np.float32); x[:, :I] = w[0][rows]
                blocks.append(x)
                blocks += [w[1][rows][:, kb * 64:(kb + 1) * 64] for kb in range(KBH)]
            else:
                blocks += [w[2][rows][:, kb * 64:(kb + 1) * 64] for kb in range(KBH)]
                blocks += [w[3][rows][:, kb * 64:(kb + 1) * 64] for kb in range(KBH)]
            for blk in blocks:
                assert np.array_equal(st[s][off], blk.astype(np.float16)), (layer, j, s)
                s += 1
    assert s == st.shape[0]
    assert built_lib.fsn_tc5_weight_stream_bytes(34, 100) == -1           # unsupported geometry


def test_tc5r_layer_packing(built_lib):
    """Layer-wise wgmma path (k_lstm_tc5r.cu): recurrent stream tiles, permuted input-projection matrix and pre-scaled biases
    of one layer follow the chunk column order n -> fsn_tc5_gate_row (gate q = (n % 32) // 8 of unit 32 j + 8 (n // 32) + n % 8)."""
    H, Kin, Kpad = 128, 34, 64
    rng = np.random.default_rng(1)
    w_ih, w_hh = rng.standard_normal((4 * H, Kin)).astype(np.float32), rng.standard_normal((4 * H, H)).astype(np.float32)
    b_ih, b_hh = rng.standard_normal(4 * H).astype(np.float32), rng.standard_normal(4 * H).astype(np.float32)
    NCH, KBH = H // 32, H // 64
    assert built_lib.fsn_tc5r_weight_stream_bytes(H) == NCH * KBH * 16384
    assert built_lib.fsn_tc5r_weight_stream_bytes(100) == -1 and built_lib.fsn_tc5r_weight_stream_bytes(576) == -1
    vp = lambda a: C.c_void_p(a.ctypes.data)
    off = np.array([[built_lib.fsn_sw128_offset(n, k) // 2 for k in range(64)] for n in range(128)])
    L2E = 1.4426950408889634
    for gru in (0, 1):
        stream, wih, bias = np.zeros(NCH * KBH * 8192, np.uint16), np.zeros(4 * H * Kpad, np.uint16), np.zeros(4 * H, np.float32)
        assert built_lib.fsn_tc5r_pack_layer(H, Kin, Kpad, vp(w_ih), vp(w_hh), vp(b_ih), vp(b_hh), gru, vp(stream), vp(wih), vp(bias)) == 0
        st, wp = stream.view(np.float16).reshape(NCH, KBH, 8192), wih.view(np.float16).reshape(4 * H, Kpad)
        for j in range(NCH):
            rows = np.array([built_lib.fsn_tc5_gate_row(H, j, n) for n in range(128)])
            for kb in range(KBH):
                assert np.array_equal(st[j, kb][off], w_hh[rows][:, kb * 64:(kb + 1) * 64].astype(np.float16))
            assert np.array_equal(wp[j * 128:(j + 1) * 128, :Kin], w_ih[rows].astype(np.float16))
            assert not wp[j * 128:(j + 1) * 128, Kin:].any()
            q = (np.arange(128) % 32) // 8
            scale = np.where((q == 2) | ((q == 3) & (gru == 1)), -2 * L2E, -L2E).astype(np.float32)
            assert np.allclose(bias[j * 128:(j + 1) * 128], scale * (b_ih[rows] + b_hh[rows]), rtol=1e-6)
    assert built_lib.fsn_tc5r_pack_layer(100, Kin, Kpad, vp(w_ih), vp(w_hh), vp(b_ih), vp(b_hh), 0, vp(stream), vp(wih), vp(bias)) != 0


def test_oracle_is_test_infrastructure_only():
    """Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import oracle/ (the product path has no CPU route)."""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    allowed = {os.path.join(root, "bench.py"), os.path.join(root, "__graft_entry__.py")}
    offenders = []
    for d, dirs, files in os.walk(root):
        dirs[:] = [x for x in dirs if x not in (".git", "gpurun_out", "tests", "oracle", "__pycache__", "baseline")]
        for f in files:
            p = os.path.join(d, f)
            if f.endswith((".py", ".cu", ".cuh", ".h", ".sh")) and p not in allowed:
                if re.search(r"^\s*(from|import)\s+oracle\b|oracle/[a-z_]+\.py|oracle\.", open(p, errors="ignore").read(), re.M):
                    offenders.append(os.path.relpath(p, root))
    assert not offenders, offenders
