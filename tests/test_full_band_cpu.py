"""CPU: the element-wise rule of tests/test_gpu_full_band.py pinned from both sides.

* tcn_ref.truth restates the oracle's TCN (O.seq_tcn, per clip for ragged groups) to 1e-12, and sb_rnn_ref's full-band head restates
  O.seq_lstm of fullsubnet.Model's full band.
* The rule accepts an independent float32 implementation of the kernels' rounding against fp64, with the bound built from the float64
  emulation.
* It rejects every planted fault of tcn_ref.emulate by at least 10x; the whole-tensor rel-L2 each fault produces is printed next to
  it.  tile_stats needs groups whose statistics differ: here the neighbour of the 3-frame clip (with three full-length clips of one
  distribution the swapped statistics are too alike for any whole-tensor or element-wise rule).
* The GPU file's case lists reach every edge they claim, computed from the host's own formulas.
"""
import numpy as np
import pytest
import torch

import sb_rnn_ref as R
import tcn_ref as TR
import test_gpu_full_band as G
from oracle import fsn_oracle as O

MARGIN = 10.0
C_, T_, TLEN = 33, 270, [270, 3, 270]        # group 1 is 3 frames long and starts inside a 128-row tile; groups 0 and 2 cross frame 256


def _groups(seed):
    """three groups of different structure: noise, a per-channel constant, noise again (x3: max |x| > 1, store scale < 1)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((3, C_, T_)) * 3
    x[1] = x[1] * 0.05 + 12 * rng.standard_normal((C_, 1))
    return x.astype(np.float32)


def _case(causal):
    cfg = dict(O.default_plus_config(), num_freqs=C_)
    sd = TR.distinct_slopes(O.make_params_plus(cfg, seed=3), G.FB_PREFIXES)
    x = _groups(4)
    args = (sd, "fb_model_real", x, TLEN, causal, "fb", "ReLU")
    mask = (torch.arange(T_)[None, None, :] < torch.tensor(TLEN)[:, None, None]).expand(3, C_, T_)
    return args, TR.truth(*args), TR.emulate(*args), mask


@pytest.fixture(scope="module")
def sym():
    return _case(False)


@pytest.fixture(scope="module")
def causal():
    return _case(True)


@pytest.mark.parametrize("kind", ["symmetric", "causal"])
def test_truth_restates_the_oracle(kind, sym, causal):
    (sd, pre, x, tl, cz, head, act), want, _, _ = sym if kind == "symmetric" else causal
    for n, L in enumerate(tl):
        ref = O.seq_tcn(x[n:n + 1, :, :L].astype(np.float64), sd, pre, act, cz)[0]
        assert np.abs(want[n, :, :L].numpy() - ref).max() <= 1e-12 * np.abs(ref).max(), (kind, n)


def test_sub_band_head_restates_the_oracle():
    cfg = dict(O.default_plus_config(), num_freqs=16, sequence_model="TCN", sb_num_neighbors=1)
    import sbtcn_oracle as S
    sd = S.make_params(cfg, seed=5)
    x = np.random.default_rng(6).standard_normal((4, S.isb(cfg), 30))
    for act in (None, "Tanh"):
        ref = O.seq_tcn(x, sd, "sb_model", act)[:, :, 2:]
        got = TR.truth(sd, "sb_model", x, None, False, "sb", act, 2).numpy()
        assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("kind", ["LSTM", "GRU"])
def test_full_band_lstm_head_restates_the_oracle(kind):
    cfg = dict(O.default_fsn_config(), num_freqs=33, fb_model_hidden_size=48, sequence_model=kind)
    sd = O.make_params_fsn(cfg, seed=7, num_layers=2)
    x = np.random.default_rng(8).standard_normal((3, 33, 25))
    ref = O.seq_lstm(x, sd, "fb_model", 2, "ReLU", kind)
    got = R.truth(sd, kind, x, 2, "ReLU", prefix="fb_model", head="fb").numpy()
    assert got.shape == ref.shape and np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
    emu32 = R.emulate(sd, kind, x, 2, "ReLU", dtype=torch.float32, prefix="fb_model", head="fb")
    r = R.compare(emu32, torch.from_numpy(ref), R.emulate(sd, kind, x, 2, "ReLU", prefix="fb_model", head="fb"), 1.0)
    print(f"\n[full-band {kind}] fp16 emulation vs fp64 {r['emu']:.2e}; float32 arithmetic {r['err']:.2e} (bound {r['bound']:.2e})")
    assert r["ok"], r


@pytest.mark.parametrize("kind", ["symmetric", "causal"])
def test_checker_accepts_kernel_rounding(kind, sym, causal):
    args, want, emu, mask = sym if kind == "symmetric" else causal
    emu32 = TR.emulate(*args, dtype=torch.float32)
    r = R.compare(emu32, want, emu, TR.TCN_FACTOR, mask)
    print(f"\n[TCN {kind} C={C_} T'={T_} tlen {TLEN}] emulation vs fp64: max err/RMS {r['emu']:.2e}; float32 arithmetic: {r['err']:.2e} "
          f"(bound {r['bound']:.2e}) rel-L2 {r['rel']:.2e}")
    assert r["ok"], r
    assert r["emu"] < 1e-2, "the tf32 / fp16 rounding alone should stay far below the fault errors"


@pytest.mark.parametrize("fault", TR.FAULTS)
def test_checker_rejects_planted_faults(fault, sym, causal):
    args, want, emu, mask = causal if fault == "causal_taps" else sym
    bad = TR.emulate(*args, fault=fault)
    r = R.compare(bad, want, emu, TR.TCN_FACTOR, mask)
    print(f"\n[{fault}] max err/RMS {r['err']:.2e} whole-tensor rel-L2 {r['rel']:.2e}; bound {r['bound']:.2e}: "
          f"{r['err'] / r['bound']:.1f}x the bound")
    assert not r["ok"], fault
    assert r["err"] > MARGIN * r["bound"], (fault, r["err"], r["bound"])


def test_cases_reach_every_edge():
    tiles = {F: G.tcn_tiles(F) for F in G.FB_WIDTHS}
    assert {nt for _, nt, _ in tiles.values()} == {64, 128}
    assert any(Cp % nt for Cp, nt, _ in tiles.values()), "no partial last N tile"
    assert any(n >= 3 for _, _, n in tiles.values()) and max(G.FB_WIDTHS) == 2048
    assert any(Cp == 32 for Cp, _, _ in tiles.values()) and any(Cp == 64 for Cp, _, _ in tiles.values())
    rows = {B * Tp for _, B, Tp in G.FB_ROWS}
    assert {127, 128, 129} <= rows
    assert any(B > 1 and any((b * Tp) % 128 and (b * Tp) // 128 != ((b + 1) * Tp - 1) // 128 for b in range(B)) for _, B, Tp in G.FB_ROWS), \
        "no gLN group straddles two 128-row tiles"
    F, B, Tp = G.FB_WAVES
    assert 3 * 4 * ((B * Tp + 127) // 128) > 2 * 132, "GEMM1 of the waves case fits in two waves"
    tps = {Tp for Tp, _, _ in G.FB_TPRIME}
    for edge in (255, 256, 257, 256 + 18, 256 + 19):                # the depth-wise chunk and its 2 x 9-frame halo
        assert edge in tps and edge in {Tp for Tp, _ in G.SB_TPRIME}
    for d in set(O.TCN_DILATIONS) - {1}:
        assert any(Tp < d for Tp in tps) and any(d <= Tp < 2 * d for Tp in tps), d
    assert {la for _, la, _ in G.FB_TPRIME} == {0, 2} and {c for _, _, c in G.FB_TPRIME} == {False, True}
    assert min(G.RAGGED) == 1 and {3, 9, 10, 19} <= set(G.RAGGED)
    assert {2 * Ns + 1 + 3 * (2 * Nf + 1) for Ns, Nf in G.SB_ISB} == {6, 34, 64}
    assert G.SB_GROUPS[0] * G.SB_GROUPS[1] > 65535
    sms = 132
    assert all(G.ws_eligible(L, H, F, B, sms) for B, H, L, _, _, F in G.WS)
    assert {B for B, *_ in G.WS} == {1, 2, 63, 64} and {H for _, H, *_ in G.WS} == {16, 48, 64, 256, 512, 528}
    assert {L for _, _, L, *_ in G.WS} == {1, 2, 3, 4} and {F for *_, F in G.WS} == {4, 33, 257, 513}
    assert {(k, f) for _, _, _, k, f, _ in G.WS} == {(k, f) for k in ("LSTM", "GRU") for f in (True, False)}
    assert 528 // 4 == sms
    assert not any(G.ws_eligible(L, H, F, B, sms) for B, H, L, _, _, F in G.MMA) and {B for B, *_ in G.MMA} == {65, 130}
    fit, over = G.ws_limit_widths(*G.WS_LIMIT_LH)
    L, H = G.WS_LIMIT_LH
    assert G.ws_eligible(L, H, fit, 2, sms) and not G.ws_eligible(L, H, over, 2, sms)
    assert G.ws_eligible(1, 4 * sms, 33, 2, sms) and not G.ws_eligible(1, 4 * sms + 16, 33, 2, sms)
    assert {Tp for Tp, _ in G.FSN_TPRIME} == {1, 2, 190, 2000}
    print(f"\nws shared-memory limit at (L, H) = {G.WS_LIMIT_LH}: F = {fit} fits ({G.ws_smem(L, H, (fit + 15) // 16 * 16)} B), "
          f"F = {over} does not ({G.ws_smem(L, H, (over + 15) // 16 * 16)} B)")
