"""CPU: the offline audio call (fsn_model_enhance_audio, DESIGN.md §3.12).

* An fp64 restatement of its two kernels with their indexing -- runs of R = 2048 / hop frames or hops per CTA, the reflected sample
  positions each analysis run stages, the frames each synthesis run reads and the end-of-clip envelope -- reproduces O.stft / O.istft
  and torch.stft / torch.istft in float64 per clip, for edge lengths and ragged sets of them.
* The host checks of the call (through fsn_plan_audio, which runs them without a GPU) reject what the call rejects, naming the clip.
* Its plan counts its own workspace and stays within the cap; the plain plans are unchanged.
"""
import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

RUN_POINTS = 2048                                    # k_audio.cu: AUDIO_RUN_POINTS


def analysis(x, Lb, n_fft, T):
    """audio_stft_kernel for one clip: [F, T] complex, zero at frames >= T_b.  x: the clip's row (read only below Lb)."""
    H = n_fft // 2
    F, R, Tb = H + 1, RUN_POINTS // H, Lb // H + 1
    w = O.hann_periodic(n_fft)
    X = np.zeros((F, T), complex)
    for t0 in range(0, T, R):
        nv = min(R, Tb - t0)
        if nv <= 0:
            continue
        p = H * (t0 - 1) + np.arange((nv + 1) * H)
        p = np.where(p < 0, -p, p)
        p = np.where(p >= Lb, 2 * (Lb - 1) - p, p)
        assert p.min() >= 0 and p.max() < Lb
        xs = x[p]
        for r in range(nv):
            X[:, t0 + r] = np.fft.rfft(xs[r * H: r * H + n_fft] * w)
    return X


def synthesis(E, Lb, L, n_fft):
    """audio_istft_kernel for one clip: E [F, >= T_b] -> [L], zero from Lb."""
    H = n_fft // 2
    R, Tb = RUN_POINTS // H, Lb // H + 1
    w = O.hann_periodic(n_fft)
    inv_env, inv_last = 1.0 / (w[:H] ** 2 + w[H:] ** 2), 1.0 / w[H:] ** 2
    out = np.zeros(L)
    for q0 in range(0, -(-L // H), R):
        nf = min(R + 1, Tb - q0)
        y = [np.fft.irfft(E[:, q0 + r], n=n_fft) * w for r in range(max(nf, 0))]
        for r in range(R):
            n = (q0 + r) * H + np.arange(H)
            keep = n < min(Lb, L)
            if not keep.any():
                continue
            if q0 + r + 1 < Tb:
                v = (y[r][H:] + y[r + 1][:H]) * inv_env
            else:
                v = y[r][H:] * inv_last
            out[n[keep]] = v[keep]
    return out


def edge_lengths(n_fft, k=5):
    hop = n_fft // 2
    return [hop + 1, k * hop - 1, k * hop, k * hop + 1, k * hop + hop // 2]


@pytest.mark.parametrize("n_fft", [64, 512, 1024])
def test_restatement_matches_stft_istft(n_fft):
    rng = np.random.default_rng(n_fft)
    hop, F = n_fft // 2, n_fft // 2 + 1
    lengths = edge_lengths(n_fft) + edge_lengths(n_fft, 37)        # 37 hops: several runs per clip at every n_fft
    L, T = max(lengths), max(lengths) // hop + 1
    for Lb in lengths:
        x = np.full(L, np.nan)
        x[:Lb] = rng.standard_normal(Lb)
        X = analysis(x, Lb, n_fft, T)
        Tb = Lb // hop + 1
        ref = O.stft(x[None, :Lb], n_fft, hop, n_fft)[0]
        assert ref.shape == (F, Tb)
        assert np.abs(X[:, :Tb] - ref).max() <= 1e-12 * np.abs(ref).max(), Lb
        assert not X[:, Tb:].any()
        tref = torch.stft(torch.from_numpy(x[:Lb]), n_fft, hop, n_fft, window=torch.hann_window(n_fft, dtype=torch.float64),
                          center=True, pad_mode="reflect", return_complex=True).numpy()
        assert np.abs(X[:, :Tb] - tref).max() <= 1e-12 * np.abs(tref).max(), Lb
        E = X * (rng.uniform(0.2, 2.0, X.shape) * np.exp(1j * rng.uniform(-3, 3, X.shape)))   # any enhanced spectrum
        y = synthesis(E, Lb, L, n_fft)
        yref = O.istft(E[None, :, :Tb], n_fft, hop, n_fft, length=Lb)[0]
        assert np.abs(y[:Lb] - yref).max() <= 1e-12 * np.abs(yref).max(), Lb
        assert not y[Lb:].any()
        tyref = torch.istft(torch.from_numpy(E[:, :Tb]), n_fft, hop, n_fft, window=torch.hann_window(n_fft, dtype=torch.float64),
                            length=Lb).numpy()
        assert np.abs(y[:Lb] - tyref).max() <= 1e-12 * np.abs(tyref).max(), Lb


@pytest.mark.parametrize("n_fft", [64, 512, 1024])
def test_ragged_batch_is_per_clip(n_fft):
    """A ragged batch (rows of L samples, T = the longest clip's frames): every clip's planes and waveform are its own."""
    rng = np.random.default_rng(n_fft + 1)
    hop = n_fft // 2
    lengths = list(rng.permutation(edge_lengths(n_fft) + edge_lengths(n_fft, 11)))
    L = max(lengths) + 3
    T = max(lengths) // hop + 1
    rows = np.full((len(lengths), L), np.nan)
    for b, Lb in enumerate(lengths):
        rows[b, :Lb] = rng.standard_normal(Lb)
    for b, Lb in enumerate(lengths):
        X = analysis(rows[b], Lb, n_fft, T)
        ref = O.stft(rows[b:b + 1, :Lb], n_fft, hop, n_fft)[0]
        assert np.abs(X[:, :ref.shape[1]] - ref).max() <= 1e-12 * np.abs(ref).max()
        y = synthesis(X, Lb, L, n_fft)
        yref = O.istft(X[None, :, :ref.shape[1]], n_fft, hop, n_fft, length=Lb)[0]
        assert np.abs(y[:Lb] - yref).max() <= 1e-12 * np.abs(yref).max() and not y[Lb:].any()
        # the identity enhancement gives the clip back; the last samples are divided by a small w^2, hence the looser bar
        assert np.abs(y[:Lb] - rows[b, :Lb]).max() <= 1e-10


def _cfg(**kw):
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus
    base = dict(O.default_plus_config())
    base.update(kw)
    return FullSubNet_Plus(**base)._cfg


@pytest.mark.parametrize("lengths,L,msg", [
    ([256, 4000], 4000, r"clip 0: h_lengths\[0\] = 256: a clip needs more than n_fft / 2 = 256 samples"),
    ([4000, 4001], 4000, r"clip 1: h_lengths\[1\] = 4001 exceeds the row length L = 4000"),
    ([4000, 1000], 4000, r"clip 1: h_lengths\[1\] = 1000 samples give 4 frames: frames \+ look_ahead = 6 is shorter than the TSSE "
                         r"kernel size 10 \(a clip needs at least 1792 samples\)"),
    (None, 200, r"L = 200: a clip needs more than n_fft / 2 = 256 samples"),
    (None, 1791, r"L = 1791 samples give 7 frames"),
    (None, 0, r"L = 0: the row length must be 1 \.\. 2\^31 - 1"),
    (None, 2 ** 31, r"L = 2147483648: the row length"),
    (None, 65535 * 256 * 256, r"the row length"),
])
def test_host_checks(built_lib, lengths, L, msg):
    from fsnplus_b200 import _lib
    cfg = _cfg()
    B = len(lengths) if lengths else 2
    with pytest.raises(_lib.FsnError, match=msg):
        _lib.plan_audio(cfg, B, L, lengths)


def test_host_checks_geometry(built_lib):
    from fsnplus_b200 import _lib
    with pytest.raises(_lib.FsnError, match=r"num_freqs 100: the audio call needs n_fft = 2 \(num_freqs - 1\) to be a power of two"):
        _lib.plan_audio(_cfg(num_freqs=100), 1, 16000)
    with pytest.raises(_lib.FsnError, match=r"num_freqs 1025"):
        _lib.plan_audio(_cfg(num_freqs=1025, sb_num_neighbors=3), 1, 16000)
    with pytest.raises(_lib.FsnError, match=r"B = 0: the batch needs at least one clip"):
        _lib.plan_audio(_cfg(), 0, 16000)
    with pytest.raises(_lib.FsnError, match=r"T \+ look_ahead = .* exceeds the limit"):
        _lib.plan_audio(_cfg(num_freqs=33, sb_num_neighbors=3), 1, 2 ** 31 - 1)
    # the smallest clips that pass: n_fft / 2 + 1 samples without TSSE, (kmax - look_ahead - 1) hops with it
    assert _lib.plan_audio(_cfg(channel_attention_model="SE"), 1, 257)[0] == 1
    assert _lib.plan_audio(_cfg(), 1, 1792)[0] == 1


def test_plan_counts_the_audio_workspace(built_lib):
    from fsnplus_b200 import _lib
    cfg = _cfg()
    F = cfg.num_freqs
    for B, secs, cap in [(64, 3, 24e9), (8, 10, 24e9), (64, 3, 2e9), (1, 240, 1e9), (256, 10, 6e9)]:
        L = secs * 16000
        T = L // 256 + 1
        bs, tw, fc, nb = _lib.plan_audio(cfg, B, L, cap_bytes=cap)
        pbs, ptw, pfc, pnb = _lib.plan_forward_bins(cfg, B, T, cap_bytes=cap)
        audio = 20 * bs * F * T + 4 * bs
        if pnb + 20 * pbs * F * T + 4 * pbs <= cap:              # the audio bytes are small: the plain plan, plus them
            assert (bs, tw, fc) == (pbs, ptw, pfc), (B, secs, cap)
            assert nb == pnb + audio
        if nb - audio <= cap and pnb <= cap:                     # a plan fits: the audio plan does too
            assert nb <= cap or (bs, tw) == (1, 256), (B, secs, cap, nb)
    # long clips: windows under a low cap, and the audio bytes inside it
    for cap in (1.2e9, 2e9):
        bs, tw, fc, nb = _lib.plan_audio(cfg, 1, 240 * 16000, cap_bytes=cap)
        assert bs == 1 and tw > 0 and nb <= cap


# fsn_plan_forward_bins of the default configurations before the audio call existed: its workspace entries are sized 0 outside it
PLAIN_PLANS = [
    ('plus', 64, 188, 24e9, (64, 0, 0, 12922048768)),
    ('plus', 1, 15001, 24e9, (1, 7520, 0, 15672356324)),
    ('plus', 1, 900000, 24e9, (1, 224, 0, 23980026020)),
    ('plus', 256, 626, 6e9, (20, 224, 0, 5133804240)),
    ('plus', 8, 3751, 1e9, (2, 256, 0, 980133576)),
    ('plus', 3, 60000, 2e9, (1, 192, 0, 1960774308)),
    ('tcn', 64, 188, 24e9, (64, 0, 0, 9131432448)),
    ('tcn', 1, 15001, 24e9, (1, 0, 0, 11250170888)),
    ('tcn', 1, 900000, 24e9, (1, 0, 1, 26056990664)),
    ('tcn', 256, 626, 6e9, (12, 0, 0, 5653196640)),
    ('tcn', 8, 3751, 1e9, (2, 0, 37, 978540848)),
    ('tcn', 3, 60000, 2e9, (1, 0, 2, 1906276588)),
    ('fsn', 64, 188, 24e9, (64, 0, 0, 12668592448)),
    ('fsn', 1, 15001, 24e9, (1, 7520, 0, 15879764052)),
    ('fsn', 1, 900000, 24e9, (1, 256, 0, 36476050612)),
    ('fsn', 256, 626, 6e9, (20, 224, 0, 4890623056)),
    ('fsn', 8, 3751, 1e9, (2, 256, 0, 953248232)),
    ('fsn', 3, 60000, 2e9, (1, 256, 0, 2919730612)),
]


def test_plain_plans_unchanged(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import Model
    cfgs = {"plus": _cfg(), "tcn": _cfg(sequence_model="TCN"), "fsn": Model(**O.default_fsn_config())._cfg}
    for name, B, T, cap, want in PLAIN_PLANS:
        assert _lib.plan_forward_bins(cfgs[name], B, T, cap_bytes=cap) == want, (name, B, T, cap)
        assert _lib.plan_forward(cfgs[name], B, T, cap_bytes=cap) == (want[0], want[1], want[3])
    # the audio plan of the same clips: the plain plan's bytes plus 20 bytes per bin and frame and the sample counts, when it fits
    cfg = cfgs["plus"]
    c = _lib.plan_audio(cfg, 64, 187 * 256, cap_bytes=24e9)
    assert c[:3] == (64, 0, 0) and c[3] == 12922048768 + 20 * 64 * 257 * 188 + 4 * 64
