"""CPU: the element-wise rule of tests/test_gpu_sb_recurrence.py pinned from both sides, and the host side of the sub-band stage hook.

* The rule accepts an independent float32 implementation of the kernels' rounding (fp16 weights, h and Gin, fp32 c) against fp64,
  with the bound built from the float64 emulation.
* It rejects every planted fault of sb_rnn_ref.emulate, and keeps rejecting it with the fast-math bound multiplied by 10: the bound
  stays at least 10x below the smallest fault error.
* The GPU file's case lists reach every ring plan of the layer-wise kernel and every row count of the generic one.
* fsn_model_sb_forward refuses what it must without a device.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import sb_rnn_ref as R
import test_gpu_sb_recurrence as G
from oracle import fsn_oracle as O

MARGIN = 10.0


def _setup(kind, H, L, N=64, Tp=190, seed=0, Ns=15):
    cfg = dict(O.default_plus_config(), num_freqs=64, sb_model_hidden_size=H, sequence_model=kind, sb_num_neighbors=Ns)
    sd = O.make_params_plus(cfg, seed=seed, num_layers=L)
    I = 2 * Ns + 1 + 3
    x = torch.from_numpy(np.random.default_rng(seed + 1).standard_normal((N, I, Tp))).half().double()
    return sd, x, cfg["look_ahead"]


@pytest.fixture(scope="module")
def lstm_case():
    sd, x, la = _setup("LSTM", 384, 2)
    return sd, x, la, R.truth(sd, "LSTM", x, la, None), R.emulate(sd, "LSTM", x, la, None)


@pytest.fixture(scope="module")
def gru_case():
    sd, x, la = _setup("GRU", 384, 2, seed=2)
    return sd, x, la, R.truth(sd, "GRU", x, la, None), R.emulate(sd, "GRU", x, la, None)


@pytest.mark.parametrize("kind", ["LSTM", "GRU"])
def test_checker_accepts_kernel_rounding(kind, lstm_case, gru_case):
    sd, x, la, want, emu = lstm_case if kind == "LSTM" else gru_case
    emu32 = R.emulate(sd, kind, x, la, None, dtype=torch.float32)
    r = R.compare(emu32, want, emu, 1.0)
    print(f"\n[{kind} H=384 L=2 T'=190] fp16 emulation vs fp64: max err/RMS {r['emu']:.2e}; float32 arithmetic: {r['err']:.2e} "
          f"(bound {r['bound']:.2e}) rel-L2 {r['rel']:.2e}")
    assert r["ok"], r
    assert r["emu"] < 5e-3, "the fp16 rounding alone should stay far below the fault errors"


@pytest.mark.parametrize("fault", R.FAULTS)
def test_checker_rejects_planted_faults(fault, lstm_case, gru_case):
    kind = "GRU" if fault == "gru_bias_fold" else "LSTM"
    sd, x, la, want, emu = lstm_case if kind == "LSTM" else gru_case
    bad = R.emulate(sd, kind, x, la, None, fault=fault, fault_t=32, fault_row=5)
    acc, fast = R.compare(bad, want, emu, 1.0), R.compare(bad, want, emu, R.FAST_FACTOR)
    print(f"\n[{fault}] max err/RMS {acc['err']:.2e} rel-L2 {acc['rel']:.2e}; bound {acc['bound']:.2e} (fast {fast['bound']:.2e}): "
          f"{acc['err'] / fast['bound']:.1f}x the fast-math bound")
    assert not acc["ok"] and not fast["ok"], fault
    assert acc["err"] > MARGIN * fast["bound"], (fault, acc["err"], fast["bound"])


def test_cases_reach_every_ring_plan_and_row_count(built_lib):
    """Every (H, first layer, last layer) of the layer-wise kernel, for both cells, is a GPU case, and the distinct ring plans are
    printed; the generic kernel's cases reach R = 64, 32 and 16."""
    roles = set()
    for H, L, kind in G.INSTANCES:
        roles.update((H, l == 0, l == L - 1, kind) for l in range(L))
    want = {(H, f, la, k) for H in range(64, 513, 64) for f in (True, False) for la in (True, False) for k in ("LSTM", "GRU")}
    assert roles == want, want - roles
    plans = {(H, f, la): built_lib.fsn_tc5r_ring_stages(H, int(f), int(la)) for H, f, la, _ in want}
    assert all(2 <= n <= 8 for n in plans.values()), plans
    print("\nring slots per (H, first, last):", plans)
    assert built_lib.fsn_tc5r_ring_stages(96, 1, 1) == -1
    rows = {built_lib.fsn_lstm_mma_rows(L, H, 64, 2) for H, L, _, _ in G.MMA}
    assert rows == {64, 32, 16}, rows
    assert built_lib.fsn_lstm_mma_rows(2, 40, 64, 2) == -1


def test_sb_forward_without_device(built_lib):
    """fsn_model_sb_forward: FSN_EINVAL for a null model; without a device no model can be created (FSN_ECUDA)."""
    from fsnplus_b200.model import FullSubNet_Plus
    x = torch.zeros(64)
    rc = built_lib.fsn_model_sb_forward(None, C.c_void_p(x.data_ptr()), 1, 8, 0, None, C.c_void_p(x.data_ptr()), None, None, None, None)
    assert rc == -1 and b"null" in built_lib.fsn_last_error()
    rc = built_lib.fsn_model_sb_forward(None, None, 1, 8, 0, None, None, None, None, None, None)
    assert rc == -1
    if not torch.cuda.is_available():
        m = FullSubNet_Plus(**O.default_plus_config())
        h = C.c_void_p()
        assert built_lib.fsn_model_create(C.byref(m._cfg), C.byref(h)) == -2
