"""CPU: the float64 SDR restatement (sdr_ref.py) against its direct-sum + Levinson variant on well- and ill-conditioned references
and at the lengths where the 512-tap filter outgrows the clip, its invariance to scale, its conventions (NaN for silent inputs,
rounding noise above 100 dB), the argument checks of fsn_metric_sdr / fsn_metric_sdr_workspace, which run before any device work,
and the refusals of fsnplus_b200.metrics.sdr that need no device."""
import ctypes as C

import numpy as np
import pytest
import torch
from scipy.linalg import solve_toeplitz
from scipy.signal import resample_poly

import sdr_ref as S

AGREE_DB = 1e-9


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def ill_conditioned(n=32000, seed=1):
    """(name, ref, est): a single fp32 sinusoid (cond(G) ~ 1e9), pure harmonics, 4 kHz band-limited noise, each plus white noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 16000
    refs = [("sinusoid", f32(np.sin(2 * np.pi * 440 * t))),
            ("harmonics", f32(sum(np.sin(2 * np.pi * 150 * k * t + k) / k for k in range(1, 6)))),
            ("band-limited", f32(resample_poly(resample_poly(rng.standard_normal(n), 1, 2), 2, 1)))]
    return [(name, r, f32(r + 0.1 * np.std(r) * rng.standard_normal(n))) for name, r in refs]


def short_clips(seed=2):
    rng = np.random.default_rng(seed)
    out = []
    for n in (1, 2, 100, 511, 512, 513):
        r = f32(rng.standard_normal(n))
        out.append((f"N={n}", r, f32(r + 0.3 * rng.standard_normal(n))))
    return out


def filtered(seed=3, n=20000):
    rng = np.random.default_rng(seed)
    r = f32(rng.standard_normal(n))
    h = rng.standard_normal(64) * np.exp(-np.arange(64) / 10)
    return [("filtered", r, f32(np.convolve(r, h)[:n] + 0.01 * rng.standard_normal(n)))]


def assert_agree(a, b, what):
    if a <= S.HIGH_DB or b <= S.HIGH_DB:
        assert abs(a - b) <= AGREE_DB, f"{what}: {a!r} vs {b!r}"
    else:
        assert a > S.HIGH_DB and b > S.HIGH_DB, f"{what}: {a!r} vs {b!r}"


@pytest.mark.parametrize("case", ill_conditioned() + short_clips() + filtered(), ids=lambda c: c[0])
def test_restatement_matches_direct_sums_and_levinson(case):
    name, r, e = case
    assert_agree(S.sdr(r, e), S.sdr_direct(r, e), name)


def test_levinson_solves_the_toeplitz_system():
    rng = np.random.default_rng(4)
    r = f32(rng.standard_normal(3000))
    R, D = S.correlations(r, f32(r + rng.standard_normal(3000)))
    want = solve_toeplitz(R, D)
    assert np.abs(S.levinson(R, D) - want).max() <= 1e-12 * np.abs(want).max()
    assert S.levinson(np.zeros(512), D) is None


def test_scale_invariance():
    _, r, e = ill_conditioned()[2]
    base = S.sdr(r, e)
    for sr, se in ((3.5, 1.0), (1.0, 0.25), (1e-5, 1e3)):
        assert abs(S.sdr(sr * r, se * e) - base) <= AGREE_DB


def test_conventions():
    rng = np.random.default_rng(5)
    r = f32(rng.standard_normal(4000))
    z = np.zeros_like(r)
    for f in (S.sdr, S.sdr_direct):
        assert np.isnan(f(z, r)) and np.isnan(f(r, z)) and np.isnan(f(z, z))
        assert f(r, r) > S.HIGH_DB
    assert S.sdr(r[:1], 2 * r[:1]) > S.HIGH_DB                         # one sample: est is a filtered ref exactly
    noisy = f32(r + rng.standard_normal(r.size))
    assert 0 < S.sdr(r, noisy) < 10


# ---- Python and C ABI argument checks (no device needed) ----------------------------------------------------------------------

def test_python_refusals_before_any_device_work():
    from fsnplus_b200 import metrics
    x = torch.zeros(2, 100)
    with pytest.raises(ValueError, match="CUDA"):
        metrics.sdr(x, x)
    with pytest.raises(ValueError, match="CUDA"):
        metrics.sdr([x[0]], [x[1]])
    with pytest.raises(ValueError, match="samples"):
        metrics.sdr([x[0]], [x[1, :50]])
    with pytest.raises(ValueError, match="1 reference clips and 2 estimates"):
        metrics.sdr([x[0]], [x[0], x[1]])
    with pytest.raises(TypeError, match="both"):
        metrics.sdr([x[0]], x)
    with pytest.raises(ValueError, match="lengths"):
        metrics.sdr([x[0]], [x[1]], lengths=[100])


def _err(lib):
    return lib.fsn_last_error().decode()


def test_c_abi_validation(built_lib):
    lib = built_lib
    nb = C.c_int64()
    L3 = (C.c_int64 * 3)(100, 0, 50)
    long3 = (C.c_int64 * 3)(100, 101, 50)
    ok = (C.c_int64 * 3)(100, 80, 50)
    fn = "fsn_metric_sdr_workspace"
    assert lib.fsn_metric_sdr_workspace(0, 100, None, C.byref(nb)) == -1 and f"{fn}: B = 0" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(65536, 100, None, C.byref(nb)) == -1 and "65535" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(3, 0, None, C.byref(nb)) == -1 and f"{fn}: L = 0" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(3, 1 << 31, None, C.byref(nb)) == -1 and f"L = {1 << 31}" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(3, 100, L3, C.byref(nb)) == -1 and "clip 1: h_lengths[1] = 0" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(3, 100, long3, C.byref(nb)) == -1 and "clip 1: h_lengths[1] = 101" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(3, 100, ok, None) == -1 and f"{fn}: null bytes" in _err(lib)
    assert lib.fsn_metric_sdr_workspace(3, 100, ok, C.byref(nb)) == 0
    need = nb.value
    # lengths 8 B, partials one correlation tile and one projection tile per clip, R and D, c; each segment rounded up to 256 bytes
    rnd = lambda v: (v + 255) // 256 * 256
    assert need == rnd(8 * 3) + rnd(3 * 8192) + rnd(3 * 8192) + rnd(3 * 4096) + rnd(3 * 16)
    big = C.c_int64()
    assert lib.fsn_metric_sdr_workspace(1, 16000 * 3600, None, C.byref(big)) == 0
    assert big.value == rnd(8) + rnd(8192 * -(-16000 * 3600 // 3584)) + 8192 + 4096 + rnd(16 * -(-(16000 * 3600 + 511) // 4096))
    p = C.c_void_p(4096)                                                  # never dereferenced: every check fails first
    out = C.c_void_p(8192)
    assert lib.fsn_metric_sdr(p, p, 3, 100, ok, p, need - 1, out, None) == -1 and f"fsn_metric_sdr: work_bytes = {need - 1}, " \
        f"the call needs {need}" in _err(lib)
    for args in ((None, p, p, out), (p, None, p, out), (p, p, None, out), (p, p, p, None)):
        r, e, w, o = args
        assert lib.fsn_metric_sdr(r, e, 3, 100, ok, w, need, o, None) == -1 and "fsn_metric_sdr: null device pointer" in _err(lib)
    assert lib.fsn_metric_sdr(p, p, 0, 100, ok, p, need, out, None) == -1 and "fsn_metric_sdr: B = 0" in _err(lib)
    assert lib.fsn_metric_sdr(p, p, 3, 0, ok, p, need, out, None) == -1 and "fsn_metric_sdr: L = 0" in _err(lib)
    assert lib.fsn_metric_sdr(p, p, 3, 100, L3, p, 1 << 20, out, None) == -1 and "fsn_metric_sdr: clip 1: h_lengths[1] = 0" in _err(lib)
    assert lib.fsn_metric_sdr(p, p, 3, 100, ok, p, -1, out, None) == -1 and "work_bytes = -1" in _err(lib)
