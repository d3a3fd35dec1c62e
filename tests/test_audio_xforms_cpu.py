"""CPU: the pieces of tests/test_gpu_audio_xforms.py that need no device.

* The fp64 truths of audio_ref are the oracle's O.stft / O.istft / O.enhance, end samples included.
* The single-precision emulation passes the rule on the weighted arrays.
* Every planted fault fails the rule by at least MARGIN x its bound; beside each, what the whole-clip bars of the older files
  (STFT_TOL per clip and plane, XFORM_TOL and WAVE_TOL per waveform, the cIRM tests' absolute tolerance) see of it.  The faults those
  bars pass are the gap the element-wise check closes.
* The GPU file's case lists reach the edges they claim: every run boundary from both sides in frames and in output hops, every
  L mod hop class, the shortest clips, a clip of more than three runs, at every n_fft.
"""
import numpy as np
import pytest

import audio_ref as A
import sb_rnn_ref as R
from oracle import fsn_oracle as O

MARGIN = 10.0
STFT_TOL, XFORM_TOL, WAVE_TOL = 2e-6, 1e-5, 2e-3          # the whole-clip bars of test_gpu_audio_offline.py
CIRM_ATOL = 2e-5                                          # the cIRM product's bar: atol 2e-5 max |enh| (test_gpu_full_band.py)


def _row(Lb, extra, seed):
    return A.speech(Lb + extra, seed)


def _mask(shape, seed, lo=-1.5, hi=1.5):
    return np.random.default_rng(seed).uniform(lo, hi, shape).astype(np.float32)


# ---- truths -----------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", A.N_FFTS)
def test_truths_match_oracle(n_fft):
    hop = n_fft // 2
    for i, Lb in enumerate(A.short_lengths(n_fft) + [9 * hop + r for r in A.residues(hop)]):
        row = _row(Lb, 50, i)
        X, _ = A.stft_truth(row, Lb, hop)
        ref = O.stft(row[None, :Lb].astype(np.float64), n_fft, hop, n_fft)[0]
        assert np.abs(X - ref).max() <= 1e-12 * np.abs(ref).max(), (n_fft, Lb)
        mask = _mask((1, 2) + X.shape, Lb)
        E, _ = A.cirm_truth(mask, X[None])
        want = O.enhance(X[None], mask.astype(np.float64))
        assert np.abs(E - want).max() <= 1e-12 * np.abs(want).max(), (n_fft, Lb)
        y = A.istft_truth(E[0], Lb, hop)
        yref = O.istft(E, n_fft, hop, n_fft, length=Lb)[0]
        assert np.abs(y - yref).max() <= 1e-12 * np.abs(yref).max(), (n_fft, Lb)
        r = Lb % hop                                                   # the one-frame end on its own
        if r:
            assert np.abs(y[-r:] - yref[-r:]).max() <= 1e-12 * np.abs(yref[-r:]).max(), (n_fft, Lb)


def test_limit_truth():
    """The floor: |M'| = max(|M|, lam) with M's phase, (lam, 0) for M = 0, per clip"""
    mask = np.zeros((2, 2, 3, 4), np.float32)
    mask[:, :, 1] = 0.01
    mask[:, :, 2] = 5.0
    X = np.ones((2, 3, 4), np.complex128)
    lam = np.array([0.5, 0.0], np.float32)
    E, _ = A.cirm_truth(mask, X, lam)
    M = O.decompress_cIRM(mask.astype(np.float64))
    assert np.allclose(E[0, 0], 0.5) and np.allclose(np.abs(E[0, 1]), 0.5)
    assert np.allclose(np.angle(E[0, 1]), np.angle(M[0, 0, 1] + 1j * M[0, 1, 1]))
    assert np.allclose(E[0, 2], M[0, 0, 2] + 1j * M[0, 1, 2])
    assert np.allclose(E[1], M[1, 0] + 1j * M[1, 1])


# ---- the emulation passes ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", A.N_FFTS)
def test_emulation_passes(n_fft):
    hop = n_fft // 2
    for i, Lb in enumerate([hop + 1, A.long_length(n_fft)] + A.run_lengths(n_fft, runs=(1,))[::3]):
        row = A.with_silence(Lb, i) if i == 1 else _row(Lb, 0, i)
        X, nrm = A.stft_truth(row, Lb, hop)
        emu = A.stft_emulate(row, Lb, hop)
        g, w, e, silent = A.stft_arrays(emu.real, emu.imag, X, emu, nrm)
        assert R.compare(g, w, e, 1.0)["ok"] and silent == 0
        mask = _mask((1, 2) + X.shape, Lb, -12, 12)
        lam = np.array([0.3], np.float32)
        Xk = emu.astype(np.complex64)[None]
        E, sc = A.cirm_truth(mask, Xk, lam)
        Ee = A.cirm_emulate(mask, Xk, lam)
        assert R.compare(*A.cirm_arrays(Ee, E, Ee, sc)[:3], 1.0)["ok"]
        Ek = Ee[0].astype(np.complex64)
        y, ye = A.istft_truth(Ek, Lb, hop), A.istft_emulate(Ek, Lb, hop)
        assert R.compare(*A.istft_arrays(ye, y, ye, Lb, hop), 1.0)["ok"]


# ---- planted faults ---------------------------------------------------------------------------------------------------------------------
N_FFT, HOP = 512, 256
RUN = A.run_frames(HOP)


def _stft_case(fault):
    """One clip of RUN + 3 hops + 1 sample (its last frame reflects hop - 1 samples), a near-silent stretch (-120 dB, a gated input)
    around the first run boundary, and more speech past its end in the row"""
    Lb = (RUN + 3) * HOP + 1
    row = _row(Lb, 3 * HOP, 7)
    row[(RUN - 2) * HOP:(RUN + 2) * HOP] *= 1e-6
    return row, Lb


def _gap(line, passes, bars):
    print(f"{line}  passes the whole-clip bars: {', '.join(b for b, p in zip(bars, passes) if p) or 'none'}")
    return any(passes)


@pytest.mark.parametrize("fault", A.STFT_FAULTS)
def test_stft_faults_fail(fault):
    row, Lb = _stft_case(fault)
    X, nrm = A.stft_truth(row, Lb, HOP)
    emu = A.stft_emulate(row, Lb, HOP)
    bad = A.stft_emulate(row, Lb, HOP, fault)
    g, w, e, _ = A.stft_arrays(bad.real, bad.imag, X, emu, nrm)
    r = R.compare(g, w, e, 1.0)
    rel = max(O.rel_l2(f(bad), f(X)) for f in (np.abs, np.real, np.imag))
    _gap(f"\n[stft {fault:16s}] err/bound {r['err'] / r['bound']:9.1f}  clip rel-L2 {rel:.2e}", [rel <= STFT_TOL], ["STFT_TOL"])
    assert r["err"] >= MARGIN * r["bound"], (fault, r)


def _istft_input(Lb, seed):
    """The enhanced spectrum of a clip: the fp32 product of a random cIRM and its analysis, as the kernels would hand it on"""
    X, _ = A.stft_truth(_row(Lb, 0, seed), Lb, HOP)
    mask = _mask((1, 2) + X.shape, seed)
    return A.cirm_emulate(mask, X.astype(np.complex64)[None])[0].astype(np.complex64)


@pytest.mark.parametrize("fault", A.ISTFT_FAULTS)
def test_istft_faults_fail(fault):
    """At L mod hop = 1 and hop - 1, over more than one synthesis run (env_at_end only at hop - 1: at L mod hop = 1 the end is the one
    sample k = 0, where both envelopes are w^2(hop) = 1)"""
    for r_ in ((HOP - 1,) if fault == "env_at_end" else (1, HOP - 1)):
        Lb = (RUN + 3) * HOP + r_
        E = _istft_input(Lb, r_)
        y, ye = A.istft_truth(E, Lb, HOP), A.istft_emulate(E, Lb, HOP)
        bad = A.istft_emulate(E, Lb, HOP, fault)
        r = R.compare(*A.istft_arrays(bad, y, ye, Lb, HOP), 1.0)
        rel = O.rel_l2(bad, y)
        _gap(f"\n[istft {fault:18s} L mod hop {r_:3d}] err/bound {r['err'] / r['bound']:9.1f}  waveform rel-L2 {rel:.2e}",
             [rel <= XFORM_TOL, rel <= WAVE_TOL], ["XFORM_TOL", "WAVE_TOL"])
        assert r["err"] >= MARGIN * r["bound"], (fault, r_, r)


def test_end_dominates_the_waveform_norm():
    """Why the synthesis is weighted: at L mod hop = hop - 1 the one-frame end holds nearly all of an enhanced clip's energy"""
    Lb = 20 * HOP + HOP - 1
    y = A.istft_truth(_istft_input(Lb, 3), Lb, HOP)
    share = float((y[-(HOP - 1):] ** 2).sum() / (y ** 2).sum())
    print(f"\nend share of the waveform energy at n_fft {N_FFT}, L mod hop = hop - 1: {share:.4%}")
    assert share > 0.9


@pytest.mark.parametrize("fault", A.CIRM_FAULTS)
def test_cirm_faults_fail(fault):
    rng = np.random.default_rng(5)
    B, F, T = 2, HOP + 1, 37
    mask = rng.uniform(-12, 12, (B, 2, F, T)).astype(np.float32)
    X = ((rng.standard_normal((B, F, T)) + 1j * rng.standard_normal((B, F, T))) * 10.0 ** rng.uniform(-3, 3, (B, F, T))).astype(np.complex64)
    lam = np.array([0.5, 0.0], np.float32) if fault == "limit_first" else None
    E, sc = A.cirm_truth(mask, X, lam)
    emu = A.cirm_emulate(mask, X, lam)
    bad = A.cirm_emulate(mask, X, lam, fault)
    r = R.compare(*A.cirm_arrays(bad, E, emu, sc)[:3], 1.0)
    passes = np.abs(bad - E).max() <= CIRM_ATOL * np.abs(E).max()
    _gap(f"\n[cirm {fault:14s}] err/bound {r['err'] / r['bound']:9.1f}", [passes], ["atol 2e-5 max |enh|"])
    assert r["err"] >= MARGIN * r["bound"], (fault, r)


def test_the_gap():
    """Faults the whole-clip bars pass and the element-wise rule fails: at least the two the issue of this check names"""
    row, Lb = _stft_case("run_early")
    X, _ = A.stft_truth(row, Lb, HOP)
    bad = A.stft_emulate(row, Lb, HOP, "run_early")
    assert max(O.rel_l2(f(bad), f(X)) for f in (np.real, np.imag)) <= STFT_TOL      # a staging fault in a quiet stretch
    Lb = (RUN + 3) * HOP + 1
    E = _istft_input(Lb, 1)
    y = A.istft_truth(E, Lb, HOP)
    rel = O.rel_l2(A.istft_emulate(E, Lb, HOP, "inv_last_shift"), y)
    print(f"\ninv_last shifted at L mod hop = 1: waveform rel-L2 {rel:.1e}")
    assert rel <= XFORM_TOL


# ---- case-list reach --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", A.N_FFTS)
def test_cases_reach_their_edges(n_fft):
    hop = n_fft // 2
    R_ = A.run_frames(hop)
    assert R_ == {64: 64, 128: 32, 256: 16, 512: 8, 1024: 4}[n_fft]
    lengths = A.offline_lengths(n_fft)
    hit = A.boundaries_hit(lengths, hop)
    for kind in ("stft", "istft"):
        for k in (1, 2):
            assert {(kind, k, -1), (kind, k, 0), (kind, k, 1)} <= hit, (n_fft, kind, k)
    assert {L % hop for L in lengths} >= set(A.residues(hop))
    for k in (1, 2):                                                  # every residue on both sides of both boundaries
        for r in A.residues(hop):
            qs = {L // hop for L in lengths if L % hop == r}
            assert {k * R_ - 1, k * R_} <= qs, (n_fft, k, r)
    assert set(A.short_lengths(n_fft)) <= set(lengths)
    assert min(lengths) == hop + 1 and max(A.frames_of(L, hop) for L in lengths) > 3 * R_


# ---- the batch grid limit ---------------------------------------------------------------------------------------------------------------
def test_plan_keeps_the_launch_grid(built_lib):
    """A sub-batch never holds more clips than gridDim.y / z (65 535): 3 B for FullSubNet+'s TSSE planes, B elsewhere; batches within
    it plan as before"""
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus, Model
    fsn = O.default_fsn_config()
    fsn.update(num_freqs=33, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=96)
    plus = O.default_plus_config()
    plus.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    for c, lim in ((Model(**fsn)._cfg, 65535), (FullSubNet_Plus(**plus)._cfg, 21845)):
        assert _lib.plan_audio(c, lim, 3000, cap_bytes=1e18)[0] == lim
        assert _lib.plan_audio(c, lim + 1, 3000, cap_bytes=1e18)[0] == (lim + 2) // 2
        assert _lib.plan_audio(c, 3 * lim, 3000, cap_bytes=1e18)[0] == lim
        assert _lib.plan_forward(c, lim + 1, 93, cap_bytes=1e18)[0] == (lim + 2) // 2
