"""SI-SDR and STOI on the device (fsnplus_b200.metrics, DESIGN.md §3.20), clip by clip against the float64 restatement in
metrics_ref.py: noisy speech at -5 .. 20 dB SNR, an enhancement model's output, est = ref, a silent estimate; 8, 16, 44.1 and 48 kHz;
clips shorter than one frame, around 30 envelope frames, at every length mod 128 around a tile edge, half silent, and ten minutes
long; and a ragged batch of 64 in which every clip's scores are bit-identical to the same clip scored alone.

Every fixture asserts that no frame energy of its reference lies within 1e-3 dB of its clip's keep threshold, so the comparison checks
arithmetic, not a keep / drop decision that fp32 resampling could flip."""
import numpy as np
import pytest
import torch

import audio_ref as A
import metrics_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STOI_TOL = 1e-5
SI_SDR_TOL = 1e-4          # dB
MARGIN_DB = 1e-3
F32 = np.float32


def noisy(x, snr_db, seed):
    rng = np.random.default_rng(seed)
    n = rng.standard_normal(x.size)
    rms = np.sqrt(np.mean(np.asarray(x, np.float64) ** 2)) or 1.0
    return (x + n * rms * 10 ** (-snr_db / 20)).astype(F32)


def speech_cases(sr, seconds=2.0, seed=0):
    """(ref, est) pairs: speech-like clips with noise from -5 to 20 dB SNR, one of them half silence."""
    n = int(seconds * sr)
    cases = []
    for k, snr in enumerate((-5, 0, 5, 10, 20)):
        x = A.speech(n + 37 * k, seed + k)
        cases.append((x, noisy(x, snr, seed + 100 + k)))
    x = A.with_silence(n, seed + 7)
    cases.append((x, noisy(x, 5, seed + 107)))
    return cases


def frame_cases():
    """At 10 kHz, white-noise references keep every frame: F frames give F - 1 envelope frames.  F = 30, 31, 32 put the clip just
    below, at and above 30 envelope frames; 2 and 200 samples have no frame at all."""
    rng = np.random.default_rng(3)
    out = []
    for n in (2, 200, 256, 257, 256 + 128 * 30, 256 + 128 * 31, 256 + 128 * 32, 256 + 128 * 32 + 1):
        x = rng.standard_normal(n).astype(F32)
        out.append((x, (x + 0.5 * rng.standard_normal(n)).astype(F32)))
    return out


def residue_cases():
    """Every length mod 128 around the energy kernel's 16-frame tile edge (and so the envelope kernel's 8-frame one), at 10 kHz."""
    rng = np.random.default_rng(4)
    out = []
    for r in range(128):
        n = 256 + 128 * 32 + r
        x = A.speech(n, 500 + r)
        out.append((x, (x + 0.1 * rng.standard_normal(n)).astype(F32)))
    return out


def ragged_cases(seed=9):
    rng = np.random.default_rng(seed)
    lengths = [int(v) for v in rng.integers(300, 60000, size=64)]
    lengths[:4] = [1, 300, 409, 410]                                   # below and at one 10 kHz frame at 16 kHz
    out = []
    for i, n in enumerate(lengths):
        x = A.speech(n, 700 + i)
        out.append((x, noisy(x, float(rng.uniform(-5, 20)), 800 + i)))
    return out


def assert_margin(cases, sr):
    for i, (x, _) in enumerate(cases):
        m = R.threshold_margin(x, sr)
        assert m > MARGIN_DB, f"fixture {i} at {sr} Hz: a frame energy lies {m:.2e} dB from its keep threshold"


def device_scores(cases, sr):
    from fsnplus_b200 import metrics
    ref = [torch.from_numpy(x).to(DEV) for x, _ in cases]
    est = [torch.from_numpy(y).to(DEV) for _, y in cases]
    return metrics.si_sdr(ref, est).cpu().numpy(), metrics.stoi(ref, est, sr=sr).cpu().numpy()


def check(cases, sr, sdr=True):
    assert_margin(cases, sr)
    got_sdr, got_stoi = device_scores(cases, sr)
    worst = [0.0, 0.0]
    for i, (x, y) in enumerate(cases):
        want = R.stoi(x, y, sr)
        d = abs(got_stoi[i] - want)
        worst[1] = max(worst[1], d)
        assert d <= STOI_TOL, f"clip {i} ({x.size} samples at {sr} Hz): STOI {got_stoi[i]!r} vs {want!r}"
        if sdr:
            want = R.si_sdr(x, y)
            d = 0.0 if got_sdr[i] == want else abs(got_sdr[i] - want)        # a one-sample clip is +inf on both sides
            worst[0] = max(worst[0], d)
            assert d <= SI_SDR_TOL, f"clip {i} ({x.size} samples): SI-SDR {got_sdr[i]!r} vs {want!r}"
    print(f"sr {sr}: {len(cases)} clips, worst |dSI-SDR| {worst[0]:.3e} dB, worst |dSTOI| {worst[1]:.3e}")
    return got_sdr, got_stoi


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    return built_lib


@pytest.mark.parametrize("sr", [8000, 16000, 44100, 48000])
def test_noisy_speech_every_rate(sr):
    check(speech_cases(sr), sr)


def test_frame_count_edges():
    cases = frame_cases()
    _, got = check(cases, 10000)
    envelope_frames = [R.band_envelopes(R.remove_silent_frames(x.astype(np.float64), y.astype(np.float64))[0]).shape[1]
                       if R.num_frames(x.size) else -1 for x, y in cases]
    assert envelope_frames == [-1, -1, -1, 0, 29, 30, 31, 32]
    assert list(got[:5]) == [1e-5] * 5 and got[5] != 1e-5


def test_every_length_residue():
    check(residue_cases(), 10000)


def test_identical_and_silent_estimates():
    x = A.speech(3 * 16000, 11)
    sdr, st = device_scores([(x, x.copy()), (x, np.zeros_like(x))], 16000)
    assert abs(st[0] - 1.0) <= 1e-6 and abs(st[0] - R.stoi(x, x, 16000)) <= STOI_TOL
    assert sdr[0] == np.inf
    assert st[1] == R.stoi(x, np.zeros_like(x), 16000) == 0.0
    assert np.isnan(sdr[1])


def test_enhanced_output_of_a_model():
    from oracle import fsn_oracle as O
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    cfg.update(sb_num_neighbors=3, sb_model_hidden_size=64)
    params = O.make_params_plus(cfg, seed=5)
    m = FullSubNet_Plus(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    m = m.to(DEV).eval()
    cases = speech_cases(16000, seconds=3.0, seed=40)
    lengths = [x.size for x, _ in cases]
    wave = torch.zeros((len(cases), max(lengths)), device=DEV)
    for i, (_, y) in enumerate(cases):
        wave[i, :lengths[i]] = torch.from_numpy(y)
    with torch.no_grad():
        enh = m.enhance_audio(wave, lengths).cpu().numpy()
    check([(x, enh[i, :lengths[i]].copy()) for i, (x, _) in enumerate(cases)], 16000)


def test_ten_minute_clip():
    x = A.speech(600 * 16000, 21)
    check([(x, noisy(x, 5, 22))], 16000)


def test_ragged_batch_is_clip_independent():
    cases = ragged_cases()
    sdr, st = check(cases, 16000)
    for i, c in enumerate(cases):
        s1, t1 = device_scores([c], 16000)
        assert s1[0].tobytes() == sdr[i].tobytes() and t1[0].tobytes() == st[i].tobytes(), f"clip {i}"


def test_tensor_form_matches_list_form():
    from fsnplus_b200 import metrics
    cases = ragged_cases(seed=12)[:8]
    lengths = [x.size for x, _ in cases]
    ref = torch.zeros((8, max(lengths)), device=DEV)
    est = torch.full((8, max(lengths)), float("nan"), device=DEV)      # samples past a clip's length are never read
    for i, (x, y) in enumerate(cases):
        ref[i, :lengths[i]] = torch.from_numpy(x)
        est[i, :lengths[i]] = torch.from_numpy(y)
    got = metrics.stoi(ref, est, sr=16000, lengths=lengths), metrics.si_sdr(ref, est, lengths=torch.tensor(lengths))
    want = device_scores(cases, 16000)
    assert got[0].dtype == torch.float64 and got[0].device == ref.device
    assert torch.equal(got[0].cpu(), torch.from_numpy(want[1])) and torch.equal(got[1].cpu(), torch.from_numpy(want[0]))
