"""SDR on the device (fsnplus_b200.metrics.sdr, DESIGN.md §3.21), clip by clip against the float64 restatement in sdr_ref.py:
noisy speech at -5 .. 20 dB SNR, an enhancement model's output, filtered references (64 and 512 taps, and a 2000-tap tail the filter
cannot absorb), ill-conditioned references, every length from 1 to 513 samples and the lengths around both kernels' tile edges, a
-100 dBFS clip and a ten-minute clip.  Also: NaN for silent inputs, > 100 dB for est = ref, a ragged batch of 64 in which every clip's
score is bit-identical to the same clip scored alone, and a workspace of 0xFF bytes scoring exactly as a zeroed one."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

import audio_ref as A
import sdr_ref as S

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SDR_TOL = 1e-4             # dB, wherever the truth is <= 100 dB
F32 = np.float32
CORR_TILE, PROJ_TILE = 3584, 4096
WORST = [0.0]


def noisy(x, snr_db, seed):
    rng = np.random.default_rng(seed)
    rms = np.sqrt(np.mean(np.asarray(x, np.float64) ** 2)) or 1.0
    return (x + rng.standard_normal(x.size) * rms * 10 ** (-snr_db / 20)).astype(F32)


def device_sdr(cases):
    from fsnplus_b200 import metrics
    ref = [torch.from_numpy(np.ascontiguousarray(x, F32)).to(DEV) for x, _ in cases]
    est = [torch.from_numpy(np.ascontiguousarray(y, F32)).to(DEV) for _, y in cases]
    return metrics.sdr(ref, est).cpu().numpy()


def check(cases, label):
    got = device_sdr(cases)
    worst = 0.0
    for i, (x, y) in enumerate(cases):
        want = S.sdr(x, y)
        if want <= S.HIGH_DB:
            d = abs(got[i] - want)
            worst = max(worst, d)
            assert d <= SDR_TOL, f"{label} clip {i} ({x.size} samples): SDR {got[i]!r} vs {want!r}"
        else:
            assert got[i] > S.HIGH_DB, f"{label} clip {i} ({x.size} samples): SDR {got[i]!r} vs {want!r} (both must exceed 100 dB)"
    WORST[0] = max(WORST[0], worst)
    print(f"{label}: {len(cases)} clips, worst |dSDR| {worst:.3e} dB (all SDR tests so far {WORST[0]:.3e} dB)")
    return got


def speech_cases(n=32000, seed=0):
    cases = []
    for k, snr in enumerate((-5, 0, 5, 10, 20)):
        x = A.speech(n + 37 * k, seed + k)
        cases.append((x, noisy(x, snr, seed + 100 + k)))
    x = A.with_silence(n, seed + 7)
    cases.append((x, noisy(x, 5, seed + 107)))
    return cases


def ragged_cases(seed=9):
    rng = np.random.default_rng(seed)
    lengths = [int(v) for v in rng.integers(1, 60001, size=64)]
    lengths[:4] = [1, 2, 511, 60000]
    out = []
    for i, n in enumerate(lengths):
        x = A.speech(n, 700 + i)
        out.append((x, noisy(x, float(rng.uniform(-5, 20)), 800 + i)))
    return out


@pytest.fixture(scope="module", autouse=True)
def _lib(built_lib):
    return built_lib


def test_noisy_speech():
    check(speech_cases(), "noisy speech")


def test_enhanced_output_of_the_default_model():
    from oracle import fsn_oracle as O
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=5)
    m = FullSubNet_Plus(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    m = m.to(DEV).eval()
    cases = speech_cases(48000, seed=40)
    lengths = [x.size for x, _ in cases]
    wave = torch.zeros((len(cases), max(lengths)), device=DEV)
    for i, (_, y) in enumerate(cases):
        wave[i, :lengths[i]] = torch.from_numpy(y)
    with torch.no_grad():
        enh = m.enhance_audio(wave, lengths).cpu().numpy()
    check([(x, enh[i, :lengths[i]].copy()) for i, (x, _) in enumerate(cases)], "model output")


def test_filtered_references():
    rng = np.random.default_rng(11)
    n = 40000
    cases = []
    for taps in (64, 512):
        x = A.speech(n, 30 + taps)
        h = rng.standard_normal(taps) * np.exp(-np.arange(taps) / (taps / 4))
        y = np.convolve(x, h)[:n]
        cases.append((x, (y + 0.01 * np.std(y) * rng.standard_normal(n)).astype(F32)))
    x = A.speech(n, 33)
    tail = np.exp(-np.arange(2000) / 600) * rng.standard_normal(2000)       # reverberation longer than the filter
    cases.append((x, np.convolve(x, tail)[:n].astype(F32)))
    got = check(cases, "filtered")
    assert got[2] < got[0] and got[2] < got[1]


def test_ill_conditioned_references():
    rng = np.random.default_rng(12)
    n = 32000
    t = np.arange(n) / 16000
    refs = [np.sin(2 * np.pi * 440 * t), sum(np.sin(2 * np.pi * 150 * k * t + k) / k for k in range(1, 6)),
            resample_poly(resample_poly(rng.standard_normal(n), 1, 2), 2, 1)]
    cases = []
    for r in refs:
        r = r.astype(F32)
        cases.append((r, (r + 0.1 * np.std(r) * rng.standard_normal(n)).astype(F32)))
    check(cases, "ill-conditioned")


def test_every_short_length():
    rng = np.random.default_rng(13)
    cases = []
    for n in range(1, 514):
        x = rng.standard_normal(n).astype(F32)
        cases.append((x, (x + 0.5 * rng.standard_normal(n)).astype(F32)))
    check(cases, "lengths 1 .. 513")


def test_tile_edges():
    lengths = sorted({v for k in (1, 2, 3) for c in (k * CORR_TILE, k * PROJ_TILE - 511) for v in (c - 1, c, c + 1)})
    cases = []
    for i, n in enumerate(lengths):
        x = A.speech(n, 60 + i)
        cases.append((x, noisy(x, 8, 90 + i)))
    check(cases, "tile edges")


def test_quiet_and_long_clips():
    x = A.speech(48000, 14)
    q = (x / np.abs(x).max() * 1e-5).astype(F32)                            # peak at -100 dBFS
    check([(q, noisy(q, 10, 15))], "-100 dBFS")
    x = A.speech(600 * 16000, 21)
    check([(x, noisy(x, 5, 22))], "ten minutes")


def test_silent_and_identical():
    x = A.speech(16000, 16)
    z = np.zeros_like(x)
    got = device_sdr([(z, x), (x, z), (z, z), (x, x.copy())])
    assert np.isnan(got[:3]).all()
    assert got[3] > S.HIGH_DB


def test_ragged_batch_is_clip_independent():
    cases = ragged_cases()
    got = check(cases, "ragged 64")
    for i, c in enumerate(cases):
        assert device_sdr([c])[0].tobytes() == got[i].tobytes(), f"clip {i}"


def test_tensor_form_matches_list_form_and_refusals():
    from fsnplus_b200 import metrics
    cases = ragged_cases(seed=12)[:8]
    lengths = [x.size for x, _ in cases]
    ref = torch.zeros((8, max(lengths)), device=DEV)
    est = torch.full((8, max(lengths)), float("nan"), device=DEV)      # samples past a clip's length are never read
    for i, (x, y) in enumerate(cases):
        ref[i, :lengths[i]] = torch.from_numpy(x)
        est[i, :lengths[i]] = torch.from_numpy(y)
    got = metrics.sdr(ref, est, lengths=lengths)
    assert got.dtype == torch.float64 and got.device == ref.device
    assert torch.equal(got.cpu(), torch.from_numpy(device_sdr(cases)))
    with pytest.raises(ValueError, match="float32"):
        metrics.sdr(ref.double(), est.double())
    with pytest.raises(ValueError, match="float32"):
        metrics.sdr(ref[0], est[0])
    with pytest.raises(ValueError, match="differ"):
        metrics.sdr(ref, est[:, :-1])


def test_workspace_contents_do_not_matter():
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    cases = ragged_cases(seed=14)[:6]
    lengths = [x.size for x, _ in cases]
    L = max(lengths)
    ref = torch.zeros((6, L), device=DEV)
    est = torch.zeros((6, L), device=DEV)
    for i, (x, y) in enumerate(cases):
        ref[i, :lengths[i]] = torch.from_numpy(x)
        est[i, :lengths[i]] = torch.from_numpy(y)
    hl = (C.c_int64 * 6)(*lengths)
    nb = C.c_int64()
    assert lib.fsn_metric_sdr_workspace(6, L, hl, C.byref(nb)) == 0
    outs = []
    for fill in (0x00, 0xFF):
        work = torch.full((nb.value,), fill, dtype=torch.uint8, device=DEV)
        out = torch.empty(6, dtype=torch.float64, device=DEV)
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        assert lib.fsn_metric_sdr(C.c_void_p(ref.data_ptr()), C.c_void_p(est.data_ptr()), 6, L, hl, C.c_void_p(work.data_ptr()),
                                  nb.value, C.c_void_p(out.data_ptr()), stream) == 0
        outs.append(out.cpu().numpy())
    assert outs[0].tobytes() == outs[1].tobytes()
    assert not np.isnan(outs[0]).any()                                 # clip 0 is one sample long: +inf
