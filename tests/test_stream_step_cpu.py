"""CPU: the pieces of tests/test_gpu_stream_step.py that need no device.

* The payload decoder (stream_ref.decode) agrees with the layout formula of test_stream_state_cpu.py and the library's stride.
* The GPU file's case lists reach the edges they claim: every generic-kernel row count R, both wide widths, B F straddling 128-row
  tiles, a cap that cuts a 37-frame call into windows with k0 > 0, both full-band kernels, and the late calls of the 30 s session.
* The per-frame STFT truth of the audio calls is the oracle's offline STFT.
* Every planted fault of a streaming stage leaves at least MARGIN x the rule's fast-math bound on its case; its whole-tensor rel-L2 is
  printed beside it, to show what a whole-tensor bar would have seen.
"""
import numpy as np
import pytest
import torch

import sb_rnn_ref as R
import stream_ref as S
import test_gpu_full_band as GF
import test_gpu_stream_step as G
import test_stream_state_cpu as SC
from oracle import fsn_oracle as O

MARGIN = 10.0
H100_SMS = 132


# ---- payload --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,L,fb,sb", [(33, 1, 96, 64), (257, 2, 512, 384), (513, 3, 96, 128)])
def test_decoder_matches_layout(built_lib, F, L, fb, sb):
    from fsnplus_b200 import _lib
    off, end = S.offsets(F, L, fb, sb)
    want, stride, _ = SC._formula(F, L, 2, fb, sb, 1)
    assert off == want[:6] and end <= stride == _lib.state_layout(SC._cfg(F, L, "LSTM", 2, fb, sb), 1)[0]
    assert SC._formula(F, L, 2, fb, sb, 2)[0][:6] == off                        # the audio payload starts with the same segments
    rng = np.random.default_rng(F)
    raw = np.zeros(stride, np.uint8)
    vals = {}
    for o, (name, shape, dt) in zip(off, S.segments(F, L, fb, sb)):
        v = rng.standard_normal(shape).astype(dt)
        raw[o:o + v.nbytes] = np.frombuffer(v.tobytes(), np.uint8)
        vals[name] = v
    got = S.decode(raw, F, L, fb, sb)
    assert all(np.array_equal(got[k], vals[k].astype(np.float64)) for k in vals)


# ---- case-list reach ------------------------------------------------------------------------------------------------------------------
def test_cases_reach_their_edges(built_lib):
    assert {F for F, _ in G.GEOMETRY} == {33, 65, 129, 257, 513}
    straddle = [(F, B) for F, B in G.GEOMETRY if B > 1 and any((b * F) // 128 != (b * F + F - 1) // 128 and (b * F) % 128 for b in range(B))]
    assert (257, 3) in straddle and (257, 80) in straddle and any(B > 64 for _, B in G.GEOMETRY)
    rows = {built_lib.fsn_lstm_mma_rows(L, H, 16, 2) for H, L in G.MMA_H}                 # Ns = 7: Isb = 16, Ipad 16
    assert rows == {64, 32, 16}, rows
    assert sorted(2 * Ns + 1 + 2 * Nf + 1 for Ns, Nf in G.WIDE) == [66, 128]
    assert 1 in G.KS and 37 in G.KS
    cap, Tw = G._window_cap(built_lib, SC._cfg(), 3, 37)
    assert 0 < Tw < 37 and Tw % 4 == 0, Tw                                                 # windows k0 = Tw, 2 Tw, ... > 0
    print(f"\ncap {cap / 1e6:.1f} MB: one session at a time in windows of {Tw} frames")
    assert GF.ws_eligible(2, 512, 257, 4, H100_SMS) and not GF.ws_eligible(2, 512, 257, 80, H100_SMS)
    n = -(-(G.LONG_T + 2) // G.LONG_K)
    assert G.LONG_T == 1876 and (n - 3) * G.LONG_K > 0.9 * G.LONG_T                       # the checked calls are the last tenth


# ---- planted faults -------------------------------------------------------------------------------------------------------------------
F_, T_, K_ = 65, 24, 8


def _setup(kind):
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=F_, fb_model_hidden_size=96, sb_model_hidden_size=64, sequence_model=kind, sb_num_neighbors=7,
               norm_type="cumulative_laplace_norm")
    return O.make_params_fsn(cfg, seed=3, num_layers=2), cfg


def _clip(seed, T=T_):
    return G._clip(F_, T, seed).astype(np.float64)


def _report(name, got, want, emu):
    r = R.compare(got, want, emu, R.FAST_FACTOR)
    if not r["finite"]:                                                                     # NaN (a negative variance): caught as well
        r["err"] = np.inf
    print(f"\n[{name}] max err/RMS {r['err']:.2e}, {r['err'] / r['bound']:.0f}x the fast-math bound {r['bound']:.2e}; whole-tensor "
          f"rel-L2 {r['rel']:.2e}")
    assert r["err"] > MARGIN * r["bound"], (name, r)


@pytest.mark.parametrize("fault", S.NORM_FAULTS)
def test_norm_faults(fault):
    x = _clip(1)
    for kind in ("cumulative_laplace_norm", "cumulative_layer_norm"):
        want, emu = S.norm_truth(x, kind), S.norm_emulate(x, kind)
        bad = S.norm_emulate(x, kind, fault, fault_at=5, carry=S.norm_sums(30 * _clip(2))[-1])
        _report(f"{fault} {kind}", bad, want, emu)


@pytest.mark.parametrize("fault", S.PACK_FAULTS)
def test_pack_faults(fault):
    mag, fb = _clip(3), _clip(4)
    for kind in ("cumulative_laplace_norm", "cumulative_layer_norm"):
        want, emu = S.sb_truth(mag, fb, 7, 0, kind), S.sb_emulate(mag, fb, 7, 0, kind)
        _report(f"{fault} {kind}", S.sb_emulate(mag, fb, 7, 0, kind, fault, fault_at=12), want, emu)


def _carried(params, kind, prefix, head, x):
    """the state after x's first T_ - K_ frames (emulation), h(t - 2) of the next frame, and the call's input (the last K_ frames)"""
    act = "ReLU" if head == "fb" else None
    xt = torch.as_tensor(x)
    _, st = R.emulate(params, kind, xt[..., :T_ - K_], 0, act, prefix=prefix, head=head, return_state=True)
    _, prev = R.emulate(params, kind, xt[..., :T_ - K_ - 1], 0, act, prefix=prefix, head=head, return_state=True)
    return st, prev[0], xt[..., T_ - K_:], act


def _state_fault(name, params, kind, prefix, head, x, edit, fault=None):
    st, hprev, xc, act = _carried(params, kind, prefix, head, x)
    want = R.truth(params, kind, xc, 0, act, prefix=prefix, head=head, state=st)
    emu = R.emulate(params, kind, xc, 0, act, prefix=prefix, head=head, state=st)
    bad_state = edit(st, hprev)
    bad = R.emulate(params, kind, xc, 0, act, prefix=prefix, head=head, state=bad_state, fault=fault, fault_t=0)
    _report(name, bad, want, emu)


def test_fault_held_row_fb_h_zeroed():
    params, _ = _setup("LSTM")
    _state_fault("held row's full-band h zeroed", params, "LSTM", "fb_model", "fb", _clip(5)[None],
                 lambda st, hp: (torch.zeros_like(st[0]), st[1]))


def test_fault_exchange_parity():
    params, _ = _setup("LSTM")
    x = _clip(6)
    x[:, T_ - K_ - 1] *= 20                                 # the last frame before the call is loud: h(t - 1) and h(t - 2) differ
    _state_fault("h(t - 2) at a call's first frame", params, "LSTM", "fb_model", "fb", x[None],
                 lambda st, hp: (st[0], st[1], hp), fault="h_lag")


def _sb_input(seed):
    mag, fb = _clip(seed), _clip(seed + 1)
    return S.sb_emulate(mag, fb, 7, 0, "cumulative_laplace_norm")                          # [F, I, T]


def test_fault_sb_c_reset_at_call():
    params, _ = _setup("LSTM")
    _state_fault("sub-band c reset at a call boundary", params, "LSTM", "sb_model", "sb", _sb_input(7),
                 lambda st, hp: (st[0], torch.zeros_like(st[1])))


def test_fault_carry_in_units_swapped():
    params, _ = _setup("LSTM")

    def swap(st, hp):
        c = st[1].clone()
        c[..., [3, 5]] = c[..., [5, 3]]
        return st[0], c
    _state_fault("two units swapped in the carry-in of c", params, "LSTM", "sb_model", "sb", _sb_input(9), swap)


def test_fault_mask_columns_shifted():
    params, _ = _setup("LSTM")
    st, _, xc, act = _carried(params, "LSTM", "sb_model", "sb", _sb_input(11))
    want = R.truth(params, "LSTM", xc, 0, act, state=st)
    emu = R.emulate(params, "LSTM", xc, 0, act, state=st)
    bad = torch.cat([torch.zeros_like(emu[..., :1]), emu[..., :-1]], dim=-1)              # column k holds frame k - 1
    _report("mask columns shifted one frame", bad, want, emu)


def test_fault_gru_carried_h_fp16():
    """The GRU's carried h rounded to fp16 moves the outputs by less than the rule's bound (the fp16 weights dominate the emulation's
    error): the GPU file catches it structurally instead -- the saved fp32 h of a GRU must not be fp16 values (gru_c_is_fp32)."""
    params, _ = _setup("GRU")
    st, _, xc, act = _carried(params, "GRU", "fb_model", "fb", _clip(13)[None])
    bad = (st[0], st[1].to(torch.float16).to(torch.float64))
    assert not G.gru_c_is_fp32(bad[1].numpy()) and G.gru_c_is_fp32(st[1].numpy())


def test_fault_right_reflect():
    """frame K's right reflect off by one sample (2 L - 1 - p instead of 2 (L - 1) - p), on the frames a FLUSH makes reach past L"""
    hop, Kh = 64, 10
    x = (np.random.default_rng(17).standard_normal(Kh * hop) * 0.1).astype(np.float32)
    L = Kh * hop
    want, emu = S.stft_mag_truth(x, Kh - 3, 5, hop, L), S.stft_mag_emulate(x, Kh - 3, 5, hop, L)
    assert not np.any(want[:, 4:]), "frames past the last hop are zero"
    _report("frame K's right reflect off by one sample", S.stft_mag_emulate(x, Kh - 3, 5, hop, L, "right_reflect"), want, emu)


def test_stft_truth_matches_offline_stft():
    """the per-frame truth of a flushed session is the oracle's torch.stft(center=True) magnitude"""
    hop, Kh = 64, 12
    x = np.random.default_rng(19).standard_normal(Kh * hop)
    want = np.abs(O.stft(x[None], 2 * hop, hop, 2 * hop))[0]
    assert np.allclose(S.stft_mag_truth(x, 0, Kh + 1, hop, Kh * hop), want, rtol=0, atol=1e-12 * np.abs(want).max())
