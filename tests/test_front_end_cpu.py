"""CPU checks of tests/front_ref.py and of the case lists of tests/test_gpu_front_end.py (no GPU needed).

* the fp64 truth restates oracle/fsn_oracle.py to 1e-12 (fb_in of every norm and attention, the subband_num grouping, fullsubnet.Model,
  the sub-band input from the oracle's own stages, and a ragged clip against the oracle run on that clip alone);
* the rule accepts an independent float32 implementation (the oracle evaluated in float32);
* every planted fault of front_ref leaves at least 10x the rule's bound; its whole-tensor rel-L2 is printed beside it, to show how
  little a whole-tensor check would have seen;
* the GPU case lists reach the edges they claim, computed from restatements of the launchers' formulas.
"""
import numpy as np
import pytest
import torch

import front_ref as FR
import sb_rnn_ref as R
import test_gpu_front_end as G
from oracle import fsn_oracle as O

H100_SMEM_OPTIN = 232448                      # bytes of dynamic shared memory one CTA may opt in to on sm_90


def _plus_cfg(F=33, attn="TSSE", norm="offline_laplace_norm", sub=1, Ns=3, Nf=0, la=2, kersize=(3, 5, 10)):
    c = O.default_plus_config()
    c.update(num_freqs=F, channel_attention_model=attn, norm_type=norm, subband_num=sub, sb_num_neighbors=Ns, fb_num_neighbors=Nf,
             look_ahead=la, kersize=list(kersize))
    return c


def _rule(got, want, emu, mask=None):
    m = None if mask is None else torch.from_numpy(np.ascontiguousarray(mask))
    return R.compare(torch.from_numpy(np.asarray(got, np.float64)), torch.from_numpy(np.asarray(want, np.float64)),
                     torch.from_numpy(np.asarray(emu, np.float64)), 1.0, m)


# ---- the truth restates the oracle ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("attn", ["TSSE", "SE", "CBAM", "ECA"])
@pytest.mark.parametrize("norm", FR.NORMS)
def test_truth_restates_oracle_plus(attn, norm):
    cfg = _plus_cfg(attn=attn, norm=norm)
    p = O.make_params_plus(cfg, seed=1)
    planes = G._spectra(2, 33, 30, 2, "zero_mean")
    st = {}
    O.fullsubnet_plus_forward(p, cfg, *planes, stages=st)
    want = FR.fb_in_truth(p, cfg, planes)
    assert np.abs(want - st["fb_in"]).max() <= 1e-12 * np.abs(st["fb_in"]).max()
    fb_out = st["fb_out"]
    sb, mu = FR.sb_in_truth(cfg, st["fb_in"][0], list(fb_out))
    assert np.abs(sb - st["sb_in"]).max() <= 1e-12 * np.abs(st["sb_in"]).max()


@pytest.mark.parametrize("sub,F", [(2, 32), (3, 33), (2, 33), (16, 33)])
def test_truth_restates_oracle_eca_subband_num(sub, F):
    cfg = _plus_cfg(F=F, attn="ECA", sub=sub)
    p = O.make_params_plus(cfg, seed=3)
    planes = G._spectra(1, F, 20, 4)
    st = {}
    O.fullsubnet_plus_forward(p, cfg, *planes, stages=st)
    assert np.abs(FR.fb_in_truth(p, cfg, planes) - st["fb_in"]).max() <= 1e-12 * np.abs(st["fb_in"]).max()


@pytest.mark.parametrize("norm", FR.NORMS)
def test_truth_restates_oracle_fsn(norm):
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, fb_model_hidden_size=32, sb_model_hidden_size=32, norm_type=norm)
    p = O.make_params_fsn(cfg, seed=5)
    mag = G._spectra(2, 33, 25, 6)[0]
    st = {}
    O.fullsubnet_forward(p, cfg, mag, stages=st)
    assert np.abs(FR.fb_in_truth(p, cfg, (mag,))[0] - st["fb_in"]).max() <= 1e-12 * np.abs(st["fb_in"]).max()
    win = np.pad(mag[:, 0].astype(np.float64), ((0, 0), (0, 0), (0, 2)))
    sb, _ = FR.sb_in_truth(cfg, win, [st["fb_out"]])
    assert np.abs(sb - st["sb_in"]).max() <= 1e-12 * np.abs(st["sb_in"]).max()


def test_truth_ragged_clip_is_the_clip_alone():
    cfg = _plus_cfg(attn="SE", norm="cumulative_layer_norm")
    p = O.make_params_plus(cfg, seed=7)
    planes = G._spectra(2, 33, 30, 8)
    frames = [12, 30]
    want = FR.fb_in_truth(p, cfg, planes, frames)
    st = {}
    O.fullsubnet_plus_forward(p, cfg, *(x[:1, :, :, :12] for x in planes), stages=st)
    assert np.abs(want[:, 0, :, :14] - st["fb_in"][:, 0]).max() <= 1e-12 * np.abs(st["fb_in"]).max()
    assert (want[:, 0, :, 14:] == 0).all()
    fbs = [np.pad(st["fb_out"][k], ((0, 1), (0, 0), (0, 18))) for k in range(3)]     # clip 0's own outputs, then nothing
    sb, _ = FR.sb_in_truth(cfg, want[0], fbs, frames)
    assert np.abs(sb[0, :, :, :14] - st["sb_in"][0]).max() <= 1e-12 * np.abs(st["sb_in"]).max()


# ---- the rule accepts an independent float32 implementation -------------------------------------------------------------------
@pytest.mark.parametrize("attn", ["TSSE", "SE", "CBAM", "ECA"])
@pytest.mark.parametrize("norm", FR.NORMS)
def test_rule_accepts_float32_oracle(attn, norm):
    cfg = _plus_cfg(attn=attn, norm=norm)
    p = O.make_params_plus(cfg, seed=9)
    planes = G._spectra(2, 33, 30, 10, "zero_mean")
    want = FR.fb_in_truth(p, cfg, planes)
    emu = FR.fb_in_emulate(p, cfg, planes)
    st = {}
    O.fullsubnet_plus_forward(p, cfg, *planes, dtype=np.float32, stages=st)
    r = _rule(st["fb_in"], want, emu)
    print(f"\n[fp32 oracle {attn} {norm}] fb_in err {r['err']:.2e} bound {r['bound']:.2e}")
    assert r["ok"], r
    win, fbs = st["fb_in"][0].astype(np.float32), [o.astype(np.float32) for o in st["fb_out"]]
    sw, _ = FR.sb_in_truth(cfg, win, fbs)
    se, _ = FR.sb_in_emulate(cfg, win, fbs)
    sf = O.NORMS[norm](np.concatenate([O.unfold(win[:, None], 3).reshape(2, 33, 7, 32)]
                                      + [O.unfold(o[:, None], 0).reshape(2, 33, 1, 32) for o in fbs], axis=2))
    r = _rule(sf, sw, se)
    print(f"[fp32 oracle {attn} {norm}] sb_in err {r['err']:.2e} bound {r['bound']:.2e}")
    assert r["ok"], r


# ---- planted faults -------------------------------------------------------------------------------------------------------------
FB_FAULT_CASES = {
    "tsse_suffix": dict(cfg=dict(attn="TSSE"), T=30),
    "mean_over_T": dict(cfg=dict(attn="SE"), T=30),
    "ragged_batch_T": dict(cfg=dict(attn="SE"), T=30, frames=[12, 30]),
    "eca_edge_self": dict(cfg=dict(attn="ECA"), T=30),
    "fc1_drop_last": dict(cfg=dict(attn="SE", F=37), T=30),
    "cbam_pad_ignored": dict(cfg=dict(attn="CBAM"), T=30, spectra="zero_mean"),
    "subband_reflect": dict(cfg=dict(attn="ECA", sub=3, F=34), T=30),
    "cum_count": dict(cfg=dict(attn="SE", norm="cumulative_layer_norm"), T=30),
    "biased_std": dict(cfg=dict(attn="SE", norm="offline_gaussian_norm"), T=30),
}
SB_FAULT_CASES = {
    "sb_edge_replicate": "offline_laplace_norm",
    "sb_fb_swap": "cumulative_laplace_norm",
    "sb_biased_std": "offline_gaussian_norm",
    "sb_mean_over_T": "offline_laplace_norm",
}


def test_fault_lists_complete():
    assert set(FB_FAULT_CASES) == set(FR.FB_FAULTS) and set(SB_FAULT_CASES) == set(FR.SB_FAULTS)


@pytest.mark.parametrize("fault", FR.FB_FAULTS)
def test_fb_in_faults_fail_the_rule(fault):
    c = FB_FAULT_CASES[fault]
    cfg = _plus_cfg(**c["cfg"])
    p = O.make_params_plus(cfg, seed=11)
    frames = c.get("frames")
    planes = G._spectra(len(frames) if frames else 2, cfg["num_freqs"], c["T"], 12, c.get("spectra", "plain"))
    want = FR.fb_in_truth(p, cfg, planes, frames)
    emu = FR.fb_in_emulate(p, cfg, planes, frames)
    bad = FR.fb_in_emulate(p, cfg, planes, frames, fault=fault)
    ok = _rule(emu, want, emu)
    assert ok["ok"]
    r = _rule(bad, want, emu)
    print(f"\n[{fault}] max err/RMS {r['err']:.2e} = {r['err'] / r['bound']:.0f} x the bound; whole-tensor rel-L2 {r['rel']:.2e}")
    assert not np.isfinite(r["err"]) or r["err"] >= 10 * r["bound"], r


@pytest.mark.parametrize("fault", FR.SB_FAULTS)
def test_sb_in_faults_fail_the_rule(fault):
    cfg = _plus_cfg(norm=SB_FAULT_CASES[fault], Ns=3, Nf=1)
    rng = np.random.default_rng(13)
    win = np.abs(rng.standard_normal((2, 33, 32))).astype(np.float32) + 0.1
    fbs = [rng.standard_normal((2, 33, 32)).astype(np.float32) * s + o for s, o in ((0.3, 0.2), (1.0, -0.1), (2.0, 0.3))]
    want, _ = FR.sb_in_truth(cfg, win, fbs)
    emu, _ = FR.sb_in_emulate(cfg, win, fbs)
    bad, _ = FR.sb_in_emulate(cfg, win, fbs, fault=fault)
    assert _rule(emu, want, emu)["ok"]
    r = _rule(bad, want, emu)
    print(f"\n[{fault}] max err/RMS {r['err']:.2e} = {r['err'] / r['bound']:.0f} x the bound; whole-tensor rel-L2 {r['rel']:.2e}")
    assert r["err"] >= 10 * r["bound"], r


def test_swizzle_fault_fails_and_decoder_round_trips():
    """A [2 tiles, T' = 3] image encoded with SWIZZLE_128B decodes back exactly; decoded with chunk (k / 8) ^ ((r >> 3) & 7) it does not."""
    rng = np.random.default_rng(14)
    rows, I, Tp = 200, 50, 3
    x = np.zeros((256, 64, Tp), np.float16)
    x[:rows, :I] = rng.standard_normal((rows, I, Tp)).astype(np.float16)
    raw = FR.encode_sw128(x)
    vals, rest = FR.decode_sb_img(raw, rows, Tp, I, "sw128")
    assert np.array_equal(vals, x[:rows, :I]) and (rest == 0).all()
    bad, _ = FR.decode_sb_img(raw, rows, Tp, I, "sw128", fault="swizzle_hi")
    w = x[:rows, :I].astype(np.float64)
    err = np.abs(bad.astype(np.float64) - w).max() / np.sqrt((w ** 2).mean())
    rel = np.linalg.norm(bad.astype(np.float64) - w) / np.linalg.norm(w)
    print(f"\n[swizzle_hi] max err/RMS {err:.2e}; whole-tensor rel-L2 {rel:.2e}")
    assert err > 1.0


def test_wide_layouts_decode():
    rows, I, Tp = 130, 100, 4
    rng = np.random.default_rng(15)
    x = rng.standard_normal((rows, I, Tp)).astype(np.float16)
    npair = FR.img_tiles(rows)
    lw = np.zeros((npair, Tp, 128, 128), np.float16)
    tm = np.zeros(npair * Tp * 128 * 128, np.float16)
    nt = (rows + 127) // 128
    for row in range(rows):
        for t in range(Tp):
            lw[row >> 7, t, row & 127, :I] = x[row, :, t]
            tm[(t * nt * 128 + row) * 128:(t * nt * 128 + row) * 128 + I] = x[row, :, t]
    for layout, buf in (("wide_layerwise", lw), ("wide_tm", tm)):
        vals, rest = FR.decode_sb_img(buf.view(np.uint8).ravel(), rows, Tp, I, layout)
        assert np.array_equal(vals, x) and (rest == 0).all(), layout


# ---- the GPU case lists reach their edges ---------------------------------------------------------------------------------------
TSSE_NORM_STATIC_SMEM = 144                   # tsse_norm_kernel's own __shared__ arrays (s_inv, s_amax[32]), as ptxas reports them


def tsse_norm_smem_before(F):
    """launch_tsse_norm's request before the prefix / suffix sums left shared memory: S, Pfx[F][16], Sfx[F][16], sq, gate, Mx, Mn, f1.
    The opt-in limit covers it plus the kernel's static shared memory."""
    return 4 * (F * (5 + 2 * 16) + F // 2 + 8)


def tsse_norm_smem(F):
    """tsse_norm_smem (k_front.cu): 5 F + F / 2 + 8 floats"""
    return 4 * (5 * F + F // 2 + 8)


def input_norm_smem_before(Tp):
    """launch_input_norm's request before its four per-frame arrays moved to the workspace: 4 float[T']"""
    return 16 * Tp


def test_case_lists_reach_the_edges():
    fit = max(F for F in range(1, 4097) if tsse_norm_smem_before(F) + TSSE_NORM_STATIC_SMEM <= H100_SMEM_OPTIN)
    assert fit == 1548 and tsse_norm_smem_before(2048) == 307232
    assert {fit, fit + 1, 2048} <= set(G.FB_WIDTHS)
    assert tsse_norm_smem(2048) <= 48 * 1024                           # every num_freqs the API accepts, without an opt-in
    lim = max(t for t in range(1, 40000) if input_norm_smem_before(t) <= H100_SMEM_OPTIN)
    assert lim == 14528 and {lim, lim + 1} <= set(G.LONG_T) and max(G.LONG_T) > lim
    assert G.HOUR_FRAMES + 2 > 14 * lim
    assert {255, 256, 257} <= set(G.TPRIME)                             # the rowstats loop's 256-frame chunk
    assert min(G.TPRIME) == max(O.default_plus_config()["kersize"])    # the shortest clip TSSE accepts
    assert any(ks == (16, 16, 16) and Tp == 16 for ks, Tp in G.KERSIZES)
    assert {(3 * B * 33) % 8 for B in G.ROWS_B} == set(range(8))        # 8 rows per rowstats CTA
    assert any(F % 32 for F, _, _ in G.SB_TCN_SHAPES) and any(Tp % 32 for _, _, Tp in G.SB_TCN_SHAPES)   # 32-bin / 32-frame tiles
    assert (4, 3) in [(F, Ns) for F, Ns, _ in G.SB_TCN_SHAPES]
    assert {B * F for F, B in G.SB_IMG_ROWS} == {127, 128, 129, 257}    # 128-row image tiles
    wide = [2 * Ns + 1 + 2 * Nf + 1 for _, Ns, Nf in G.SB_IMG_WIDE]
    assert 66 in wide and 128 in wide and any(Ns == F - 1 for F, Ns, _ in G.SB_IMG_WIDE)
    subs = [(F // 2 if s == "half" else s, F) for s, F in G.ECA_SUB]
    assert any(F % s == 0 for s, F in subs) and any(F % s for s, F in subs)
    assert min(G.RAGGED_TSSE) + 2 >= max(O.default_plus_config()["kersize"])
