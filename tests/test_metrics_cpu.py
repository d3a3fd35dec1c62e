"""CPU: the float64 metric restatement (metrics_ref.py) against the algorithm's constants and known values, against pystoi where
it is installed (it is skipped where it is not), the calculate_metrics command line with the device scores replaced by the
restatement, and the argument checks of the metric C ABI, which run before any device work."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
from scipy.io import wavfile
from scipy.signal import resample_poly

import metrics_ref as R

RATES = {8000: (365, 5, 4), 16000: (581, 5, 8), 24000: (871, 5, 12), 48000: (1741, 5, 24), 22050: (31947, 200, 441),
         44100: (31947, 100, 441)}


def test_stoi_of_a_clip_with_itself_is_one():
    x = np.random.default_rng(0).standard_normal(16000 * 3)
    assert abs(R.stoi(x, x, 16000) - 1.0) <= 1e-12


def test_si_sdr_scale_invariance_and_closed_form():
    rng = np.random.default_rng(1)
    x, n = rng.standard_normal(20000), rng.standard_normal(20000)
    eps = 1e-3
    e = x + eps * n
    a = 1 + eps * np.dot(x, n) / np.dot(x, x)
    n_perp = n - np.dot(x, n) / np.dot(x, x) * x
    want = 10 * np.log10(a * a * np.dot(x, x) / (eps * eps * np.dot(n_perp, n_perp)))
    assert abs(R.si_sdr(x, e) - want) <= 1e-9
    assert abs(R.si_sdr(3.5 * x, e) - R.si_sdr(x, e)) <= 1e-9
    assert abs(R.si_sdr(x, 0.25 * e) - R.si_sdr(x, e)) <= 1e-9


def test_band_table():
    assert R.thirdoct_bins() == R.BANDS


@pytest.mark.parametrize("fs", sorted(RATES))
def test_resampler_filter_and_length(fs):
    taps, p, q = RATES[fs]
    assert R.resample_filter(fs).size == taps and R.rates(fs) == (p, q)
    x = np.random.default_rng(fs).standard_normal(4001)
    y = R.resample(x, fs)
    assert y.size == R.resampled_length(x.size, fs) == resample_poly(x, p, q).size
    m = np.arange(0, y.size, 7)
    assert np.abs(R.resample_direct(x, fs, m) - y[m]).max() <= 1e-12


def test_silent_frames_of_a_tone_then_silence():
    n = np.arange(128 * 40 + 256)
    x = np.where(n < 128 * 20, np.sin(2 * np.pi * 440 * n / 10000), 0.0)
    _, _, mask = R.kept_frames(x)
    assert mask.size == R.num_frames(x.size) == 40
    assert list(mask) == [True] * 20 + [False] * 20                      # frame 19 still holds half a window of tone
    xs, _ = R.remove_silent_frames(x, x)
    assert xs.size == 19 * 128 + 256


def test_matches_pystoi_where_installed():
    pystoi = pytest.importorskip("pystoi")
    rng = np.random.default_rng(5)
    for fs in (8000, 16000, 44100):
        x = rng.standard_normal(fs * 2)
        y = x + rng.standard_normal(x.size)
        assert abs(pystoi.stoi(x, y, fs, extended=False) - R.stoi(x, y, fs)) <= 1e-9


# ---- command line -------------------------------------------------------------------------------------------------------------

@pytest.fixture()
def cm(monkeypatch):
    from fsnplus_b200.tools import calculate_metrics as M

    def oracle(metric, refs, ests, sr, device):
        f = R.si_sdr if metric == "SI_SDR" else (lambda r, e: R.stoi(r, e, sr))
        return [f(r, e) for r, e in zip(refs, ests)]
    monkeypatch.setattr(M, "score_batch", oracle)
    return M


def _write(path, x, sr=16000):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    wavfile.write(path, sr, (np.clip(x, -1, 1) * 32767).astype(np.int16))


def _pairs(tmp_path, names_ref, names_est, n=16000, longer=()):
    rng = np.random.default_rng(7)
    for i, (a, b) in enumerate(zip(names_ref, names_est)):
        x = 0.3 * np.sin(2 * np.pi * (200 + 50 * i) * np.arange(n) / 16000) * (1 + 0.5 * np.sin(np.arange(n) / 900))
        _write(str(tmp_path / "clean" / f"{a}.wav"), x)
        m = n + 10 if b in longer else n - 5 * i
        _write(str(tmp_path / "enh" / f"{b}.wav"), x[:m] + 0.05 * (i + 1) * rng.standard_normal(min(m, n))[:m] if m <= n
               else np.concatenate([x, np.zeros(10)]))


def test_cli_pairs_by_basename_prints_and_exports(cm, tmp_path, capsys):
    names = ["a", "b", "c"]
    _pairs(tmp_path, names, names)
    out = str(tmp_path / "out") + "/"
    cm.main(["-R", str(tmp_path / "clean"), "-E", str(tmp_path / "enh"), "-M", "SI_SDR,STOI", "-D", out, "--limit", "3"])
    lines = capsys.readouterr().out.splitlines()
    assert lines[0] == f"=== {tmp_path / 'enh'} === {tmp_path / 'clean'} ==="
    res = {}
    for m in ("SI_SDR", "STOI"):
        row = [ln for ln in lines if ln.startswith(m + ": [")][0]
        res[m] = eval(row[len(m) + 2:])
        assert [n for n, _ in res[m]] == names
        mean = [ln for ln in lines if ln.startswith(m + ": ") and not ln.startswith(m + ": [")][0]
        assert float(mean.split(": ")[1]) == pytest.approx(np.mean([v for _, v in res[m]]))
        ranked = sorted(res[m], key=lambda nv: nv[1], reverse=True)
        assert open(out + m + ".txt").read() == "".join(f"{n}: {v}\n" for n, v in ranked)
    assert res["SI_SDR"][0][1] > res["SI_SDR"][2][1]                     # less noise scores higher
    assert any("not in the same length" in ln for ln in lines)           # estimates 1, 2 are shorter than their references


def test_cli_scp_and_dns_rules(cm, tmp_path):
    _pairs(tmp_path, ["clean_fileid_3", "clean_fileid_10"], ["x_snr5_fileid_10", "y_snr0_fileid_3"])
    enh = sorted(str(p) for p in (tmp_path / "enh").iterdir())
    cln = sorted(str(p) for p in (tmp_path / "clean").iterdir())
    (tmp_path / "est.scp").write_text("\n".join(enh) + "\n")
    (tmp_path / "ref.scp").write_text("\n".join(cln) + "\n")
    res = cm.run(str(tmp_path / "ref.scp"), str(tmp_path / "est.scp"), "SI_SDR", specific_dataset="dns_1", log=lambda s: None)
    refs, ests = cm.align(cln, enh, "DNS_1")
    assert [cm.basename(e) for e in ests] == ["x_snr5_fileid_10", "y_snr0_fileid_3"] and [n for n, _ in res["SI_SDR"]] == \
        ["clean_fileid_10", "clean_fileid_3"]
    r2, e2 = cm.align(["/c/synthetic_clean_fileid_47.wav"], ["/e/synthetic_french_x_snr14_tl-26_fileid_47.wav"], "DNS_2")
    assert cm.basename(e2[0]).endswith("fileid_47")
    with pytest.raises(ValueError, match="matches 0 estimates"):
        cm.align(["/c/clean_fileid_1.wav"], ["/e/noisy_fileid_2.wav"], "DNS_1")
    with pytest.raises(NotImplementedError, match="maxhub"):
        cm.align(cln, enh, "maxhub_noisy")


def test_cli_misaligned_lists(cm, tmp_path):
    _pairs(tmp_path, ["a", "b"], ["a", "c"])
    with pytest.raises(ValueError, match="row 2"):
        cm.run(str(tmp_path / "clean"), str(tmp_path / "enh"), "STOI", log=lambda s: None)


def test_cli_refuses_unsupported_metrics_before_reading(cm, monkeypatch):
    def no_read(*a, **k):
        raise AssertionError("a file was read")
    monkeypatch.setattr(cm, "load_list", no_read)
    monkeypatch.setattr(cm, "read_wav", no_read)
    for m in ("SI_SDR,STOI,WB_PESQ,NB_PESQ", "MOSNET", "SDR", "SI_SDR,BOGUS"):
        with pytest.raises(NotImplementedError, match="supported: SI_SDR, STOI"):
            cm.run("/nonexistent/R", "/nonexistent/E", m, log=lambda s: None)


def test_cli_estimate_longer_than_reference(cm, tmp_path):
    _pairs(tmp_path, ["a", "b"], ["a", "b"], longer=("b",))
    with pytest.raises(ValueError, match=r"enh/b\.wav has 16010 samples, more than its reference .*clean/b\.wav \(16000\)"):
        cm.run(str(tmp_path / "clean"), str(tmp_path / "enh"), "SI_SDR", log=lambda s: None)


# ---- Python and C ABI argument checks (no device needed) ----------------------------------------------------------------------

def test_python_refuses_cpu_tensors():
    from fsnplus_b200 import metrics
    x = torch.zeros(2, 100)
    with pytest.raises(ValueError, match="CUDA"):
        metrics.si_sdr(x, x)
    with pytest.raises(ValueError, match="CUDA"):
        metrics.stoi([x[0]], [x[1]])
    with pytest.raises(ValueError, match="samples"):
        metrics.stoi([x[0]], [x[1, :50]])


def _err(lib):
    return lib.fsn_last_error().decode()


def test_c_abi_validation(built_lib):
    lib = built_lib
    nb = C.c_int64()
    L3 = (C.c_int64 * 3)(100, 0, 50)
    ok = (C.c_int64 * 3)(100, 80, 50)
    assert lib.fsn_metric_si_sdr_workspace(0, 100, None, C.byref(nb)) == -1 and "B = 0" in _err(lib)
    assert lib.fsn_metric_si_sdr_workspace(70000, 100, None, C.byref(nb)) == -1 and "65535" in _err(lib)
    assert lib.fsn_metric_si_sdr_workspace(3, 0, None, C.byref(nb)) == -1 and "L = 0" in _err(lib)
    assert lib.fsn_metric_si_sdr_workspace(3, 100, L3, C.byref(nb)) == -1 and "clip 1: h_lengths[1] = 0" in _err(lib)
    assert lib.fsn_metric_stoi_workspace(3, 60, ok, 16000, C.byref(nb)) == -1 and "clip 0: h_lengths[0] = 100" in _err(lib)
    for sr in (7999, 48001):
        assert lib.fsn_metric_stoi_workspace(3, 100, ok, sr, C.byref(nb)) == -1 and f"sr = {sr}" in _err(lib)
    assert lib.fsn_metric_si_sdr_workspace(3, 100, ok, None) == -1
    assert lib.fsn_metric_si_sdr_workspace(3, 100, ok, C.byref(nb)) == 0 and nb.value > 0
    assert lib.fsn_metric_stoi_workspace(3, 100, ok, 16000, C.byref(nb)) == 0
    need = nb.value
    big = C.c_int64()
    assert lib.fsn_metric_stoi_workspace(3, 16000 * 60, None, 44100, C.byref(big)) == 0 and big.value > need
    p = C.c_void_p(4096)                                                  # never dereferenced: every check fails first
    out = C.c_void_p(8192)
    assert lib.fsn_metric_stoi(p, p, 3, 100, ok, 16000, p, need - 1, out, None) == -1 and f"the call needs {need}" in _err(lib)
    assert lib.fsn_metric_stoi(p, None, 3, 100, ok, 16000, p, need, out, None) == -1 and "null" in _err(lib)
    assert lib.fsn_metric_stoi(p, p, 3, 100, ok, 9, p, need, out, None) == -1 and "sr = 9" in _err(lib)
    assert lib.fsn_metric_si_sdr(p, p, 3, 100, L3, p, 1 << 20, out, None) == -1 and "h_lengths[1]" in _err(lib)
    assert lib.fsn_metric_si_sdr(p, p, 3, 100, ok, None, 1 << 20, out, None) == -1 and "null" in _err(lib)
