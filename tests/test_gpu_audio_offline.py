"""Waveforms in, waveforms out through the offline forward (fsn_model_enhance_audio, model.enhance_audio; DESIGN.md §3.12).

Each transform is checked on its own through the "stft" / "enh" stages, the forward between them against the spectral ragged entry
point, the whole chain against the fp64 pipeline and against enhance_batch / enhance_ragged (torch transforms around the same library
forward), ragged batches clip by clip, long clips under a low workspace cap, a C caller, and every error case."""
import ctypes as C
import os
import re
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

import sbtcn_oracle as S
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
XFORM_TOL = 1e-5          # a waveform vs the fp64 iSTFT of the enhanced spectrum it was synthesised from
WAVE_TOL = 2e-3           # a waveform vs the fp64 pipeline, and vs enhance_batch / enhance_ragged
CLIP_TOL = 1e-5           # a clip of a batch (or a capped call) vs the same clip alone (uncapped)
STFT_TOL = 2e-6           # the analysis planes vs fp64 O.stft, per clip and plane
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _model(cls, cfg, params, monkeypatch=None, cap_gb=None, **kw):
    if monkeypatch is not None:
        if cap_gb is None:
            monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
        else:
            monkeypatch.setenv("FSN_WS_CAP_GB", str(cap_gb))
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    if monkeypatch is not None:
        monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
    return m


def _plus(**over):
    c = O.default_plus_config()
    c.update(over)
    return c


def _edge(n_fft, k=9):
    hop = n_fft // 2
    return [k * hop - 1, k * hop, k * hop + 1, k * hop + hop // 2]


def _batch(lengths, seed, L=None):
    """Rows [B, L] of synthetic noisy speech, NaN past each clip's length."""
    L = L or max(lengths)
    x = O.synth_clips(len(lengths), num_samples=L, seed0=seed)
    rows = np.full((len(lengths), L), np.nan, np.float32)
    for b, n in enumerate(lengths):
        rows[b, :n] = x[b, :n]
    return rows


def _run(m, rows, lengths):
    with torch.no_grad():
        return m.enhance_audio(_t(rows), lengths).cpu().numpy()


def _stage(m, name, shape):
    return m.get_stage(name, shape, torch.device(DEV)).cpu().numpy()


def _oracle(kind, params, cfg, X):
    mag, real, imag = np.abs(X)[:, None], X.real[:, None], X.imag[:, None]
    if kind == "fsn":
        return O.fullsubnet_forward(params, cfg, mag)
    if kind == "tcn":
        return S.forward(params, cfg, mag, real, imag)
    return O.fullsubnet_plus_forward(params, cfg, mag, real, imag)


def _check_model(m, kind, params, cfg, lengths, seed, fp64=True):
    """The transforms on their own, the forward between them, and the chain end to end, for one ragged batch."""
    from fsnplus_b200 import inference as inf
    F = cfg["num_freqs"]
    n_fft, hop = 2 * (F - 1), F - 1
    rows = _batch(lengths, seed)
    B, L = rows.shape
    T = max(lengths) // hop + 1
    frames = [n // hop + 1 for n in lengths]
    got = _run(m, rows, lengths)
    assert m.last_plan_bins()[0] == B
    planes = _stage(m, "stft", (3, B, 1, F, T))
    enh = torch.view_as_complex(m.get_stage("enh", (B, F, T, 2), torch.device(DEV))).cpu().numpy()
    worst = {"stft": 0.0, "istft": 0.0, "fwd": 0.0, "fp64": 0.0, "torch": 0.0}
    for b, n in enumerate(lengths):
        X = O.stft(rows[b:b + 1, :n].astype(np.float64), n_fft, hop, n_fft)
        Tb = frames[b]
        for i, ref in enumerate((np.abs(X[0]), X[0].real, X[0].imag)):
            e = O.rel_l2(planes[i, b, 0, :, :Tb], ref)
            worst["stft"] = max(worst["stft"], e)
            assert e <= STFT_TOL, (b, i, e)
        assert not planes[:, b, :, :, Tb:].any()
        y = O.istft(enh[b:b + 1, :, :Tb].astype(np.complex128), n_fft, hop, n_fft, length=n)[0]
        e = O.rel_l2(got[b, :n], y)
        worst["istft"] = max(worst["istft"], e)
        assert e <= XFORM_TOL, (b, e)
        assert (got[b, n:] == 0).all()
        if fp64:
            ref = O.istft(O.enhance(X, _oracle(kind, params, cfg, X)), n_fft, hop, n_fft, length=n)[0]
            e = O.rel_l2(got[b, :n], ref)
            worst["fp64"] = max(worst["fp64"], e)
            assert e <= WAVE_TOL, (b, e)
    # the same forward: the spectral ragged entry point on the returned planes
    with torch.no_grad():
        p = _t(planes)
        again = m.enhance_spectrum(p[0], p[1], p[2], frames=frames).cpu().numpy()
    worst["fwd"] = float(np.abs(again - enh).max())
    assert worst["fwd"] <= 1e-6
    # torch transforms around the same library forward
    with torch.no_grad():
        clips = [_t(rows[b, :n]) for b, n in enumerate(lengths)]
        tr = inf.enhance_ragged(m, clips, n_fft, hop, n_fft, complex_inputs=kind != "fsn")
    for b, n in enumerate(lengths):
        e = O.rel_l2(got[b, :n], tr[b].cpu().numpy())
        worst["torch"] = max(worst["torch"], e)
        assert e <= WAVE_TOL, (b, e)
    print(f"\n[{kind} F={F}] worst: stft {worst['stft']:.2e}  waveform vs fp64 iSTFT of enh {worst['istft']:.2e}  forward re-run "
          f"max |diff| {worst['fwd']:.2e}  vs fp64 pipeline {worst['fp64']:.2e}  vs enhance_ragged {worst['torch']:.2e}")
    return got


def test_default_config(built_lib):
    cfg = _plus()
    params = O.make_params_plus(cfg, seed=3)
    from fsnplus_b200.model import FullSubNet_Plus
    m = _model(FullSubNet_Plus, cfg, params)
    _check_model(m, "plus", params, cfg, [16000, 257 + 1535, 9 * 256 + 100, 12033], seed=11)


def test_equal_lengths_match_enhance_batch(built_lib):
    """Equal lengths: the unmasked forward (2 launches more than the spectral forward) and enhance_batch's result."""
    from fsnplus_b200 import inference as inf
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _plus()
    params = O.make_params_plus(cfg, seed=4)
    m = _model(FullSubNet_Plus, cfg, params)
    rows = _batch([24000] * 4, seed=12)
    got = _run(m, rows, None)
    n_audio = m.last_launch_count()
    with torch.no_grad():
        want = inf.enhance_batch(m, _t(rows), 512, 256, 512).cpu().numpy()
    n_spec = m.last_launch_count()
    assert n_audio == n_spec + 2, (n_audio, n_spec)
    for b in range(4):
        assert O.rel_l2(got[b], want[b]) <= WAVE_TOL
    assert np.array_equal(_run(m, rows, [24000] * 4), got)        # every length given, all equal: the same call


@pytest.mark.parametrize("variant", ["fsn_cumulative", "GRU", "TCN", "F513", "F33", "F129"])
def test_variants(built_lib, variant):
    from fsnplus_b200.model import FullSubNet_Plus, Model
    if variant == "fsn_cumulative":
        cfg = O.default_fsn_config()
        cfg.update(norm_type="cumulative_laplace_norm", sb_model_hidden_size=128, fb_model_hidden_size=256)
        params = O.make_params_fsn(cfg, seed=5)
        m, kind = _model(Model, cfg, params), "fsn"
    elif variant == "TCN":
        cfg = _plus(sequence_model="TCN")
        params = S.make_params(cfg, seed=6)
        m, kind = _model(FullSubNet_Plus, cfg, params), "tcn"
    else:
        over = {"GRU": dict(sequence_model="GRU", sb_model_hidden_size=128),
                "F513": dict(num_freqs=513, sb_model_hidden_size=128),
                "F33": dict(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64),
                "F129": dict(num_freqs=129, sb_num_neighbors=7, sb_model_hidden_size=64)}[variant]
        cfg = _plus(**over)
        params = O.make_params_plus(cfg, seed=7)
        m, kind = _model(FullSubNet_Plus, cfg, params), "plus"
    n_fft = 2 * (cfg["num_freqs"] - 1)
    lengths = _edge(n_fft, 11) + [n_fft * 7 + 5]
    _check_model(m, kind, params, cfg, lengths, seed=13)


def test_ragged_clip_by_clip(built_lib):
    """Edge lengths and 1-10 s clips in one batch, NaN past each length: each clip equals the call with that clip alone."""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _plus()
    params = O.make_params_plus(cfg, seed=8)
    m = _model(FullSubNet_Plus, cfg, params)
    rng = np.random.default_rng(9)
    lengths = [1792, 256 * 12 - 1, 256 * 12, 256 * 12 + 1, 256 * 12 + 128] + [int(v) for v in rng.integers(16000, 160001, 7)]
    L = max(lengths) + 77
    rows = _batch(lengths, seed=14, L=L)
    got = _run(m, rows, lengths)
    identical = 0
    for b, n in enumerate(lengths):
        alone = _run(m, rows[b:b + 1, :n], None)[0]
        e = O.rel_l2(got[b, :n], alone)
        assert e <= CLIP_TOL, (b, n, e)
        identical += bool(np.array_equal(got[b, :n], alone))
        assert (got[b, n:] == 0).all()
    print(f"\n[ragged] {identical} of {len(lengths)} clips bit-identical to their lone call")


@pytest.mark.parametrize("sb", ["LSTM", "TCN"])
def test_long_clip_capped(built_lib, monkeypatch, sb):
    """A 4-minute clip under a low cap: windowed (LSTM) or in bin chunks (TCN), within CLIP_TOL of the uncapped call, and the model
    holds at most the reported plan's bytes afterwards."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _plus(sequence_model=sb)
    params = S.make_params(cfg, seed=15) if sb == "TCN" else O.make_params_plus(cfg, seed=15)
    L = 240 * 16000
    rows = _batch([L], seed=16)
    ref = _run(_model(FullSubNet_Plus, cfg, params, monkeypatch), rows, None)
    torch.cuda.empty_cache()
    m = _model(FullSubNet_Plus, cfg, params, monkeypatch, cap_gb=1.2 if sb == "LSTM" else 0.6)
    got = _run(m, rows, None)
    bs, tw, fc = m.last_plan_bins()
    assert (tw > 0) if sb == "LSTM" else (fc > 0), (bs, tw, fc)
    plan = _lib.plan_audio(m._cfg, 1, L, cap_bytes=(1.2 if sb == "LSTM" else 0.6) * 1e9)
    assert plan[:3] == (bs, tw, fc)
    assert m.workspace_bytes() <= plan[3], (m.workspace_bytes(), plan)
    e = O.rel_l2(got[0], ref[0])
    print(f"\n[long {sb}] plan {bs, tw, fc}: rel-L2 vs uncapped {e:.2e}, bit-identical {np.array_equal(got, ref)}")
    assert e <= CLIP_TOL
    _stage(m, "stft", (3, 1, 1, 257, L // 256 + 1))                           # kept: one sub-batch ran


def test_c_caller(built_lib, tmp_path):
    """tests/c_enhance_audio.c, compiled with the system C compiler against the header and the built library: bit-identical to
    model.enhance_audio."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "no system C compiler"
    cfg = _plus(num_freqs=129, sb_num_neighbors=7, sb_model_hidden_size=64)
    params = O.make_params_plus(cfg, seed=17)
    m = _model(FullSubNet_Plus, cfg, params)
    libdir = os.path.dirname(_lib.lib_path())
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = tmp_path / "c_enhance_audio"
    subprocess.run([cc, os.path.join(ROOT, "tests", "c_enhance_audio.c"), "-o", str(exe), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(cuda, "include"), "-L", libdir, "-l:libfsnplus_b200.so", "-L", os.path.join(cuda, "lib64"),
                    "-lcudart", f"-Wl,-rpath,{libdir}:{os.path.join(cuda, 'lib64')}"], check=True)
    lib = _lib.load_library()
    keys = []
    for i in range(lib.fsn_model_num_params(m._handle)):                      # the keys the configuration expects
        key, numel = C.c_char_p(), C.c_int64()
        _lib.check(lib.fsn_model_param_info(m._handle, i, C.byref(key), C.byref(numel)))
        keys.append(key.value.decode())
    with open(tmp_path / "model.bin", "wb") as f:
        f.write(bytes(m._cfg))
        f.write(struct.pack("<i", len(keys)))
        for k in keys:
            v = np.ascontiguousarray(params[k], np.float32).ravel()
            f.write(struct.pack("<i", len(k)) + k.encode() + struct.pack("<q", v.size) + v.tobytes())
    lengths = [1000, 9000, 8001, 4321]
    rows = _batch(lengths, seed=18)
    with open(tmp_path / "wave.bin", "wb") as f:
        f.write(struct.pack("<iq", *rows.shape) + np.asarray(lengths, np.int64).tobytes() + rows.tobytes())
    r = subprocess.run([str(exe), str(tmp_path / "model.bin"), str(tmp_path / "wave.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(tmp_path / "out.bin", np.float32).reshape(rows.shape)
    want = _run(m, rows, lengths)
    assert np.array_equal(got, want)


def test_errors(built_lib):
    """Every rejected call names its cause, and the model's next forward is unaffected."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = _plus(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    params = O.make_params_plus(cfg, seed=19)
    m = _model(FullSubNet_Plus, cfg, params)
    lib = _lib.load_library()
    rows = _batch([3000, 2000], seed=20)
    x, out = _t(rows), torch.empty((2, 3000), device=DEV)
    before = _run(m, rows, [3000, 2000])
    ptr = lambda t: C.c_void_p(t.data_ptr())

    def call(wave=x, B=2, L=3000, lengths=(3000, 2000), o=out):
        hl = _lib.lengths_arg(lengths, len(lengths)) if lengths is not None else None
        return lib.fsn_model_enhance_audio(m._handle, wave if wave is None else ptr(wave), B, L, hl, o if o is None else ptr(o), None)

    cases = [(dict(wave=None), "d_wave is null"), (dict(o=None), "d_out is null"), (dict(B=0, lengths=None), "B = 0"),
             (dict(lengths=(3000, 16)), r"clip 1: h_lengths\[1\] = 16: a clip needs more than n_fft / 2 = 32 samples"),
             (dict(lengths=(3001, 2000)), r"clip 0: h_lengths\[0\] = 3001 exceeds the row length L = 3000"),
             (dict(lengths=(3000, 200)), r"clip 1: h_lengths\[1\] = 200 samples give 7 frames: frames \+ look_ahead = 9 is shorter"),
             (dict(L=0, lengths=None), "L = 0")]
    for kw, msg in cases:
        assert call(**kw) == -1, kw
        err = lib.fsn_last_error().decode()
        assert re.search(msg, err), (kw, err)
    assert lib.fsn_model_enhance_audio(None, ptr(x), 2, 3000, None, ptr(out), None) == -1
    bad = _model(FullSubNet_Plus, _plus(num_freqs=100, sb_num_neighbors=3, sb_model_hidden_size=64),
                 O.make_params_plus(_plus(num_freqs=100, sb_num_neighbors=3, sb_model_hidden_size=64), seed=1))
    with pytest.raises(_lib.FsnError, match="num_freqs 100"):
        bad.enhance_audio(torch.zeros((1, 4000), device=DEV))
    with pytest.raises(ValueError):
        m.enhance_audio(x, [3000])
    # the stages are kept only after an audio call that ran as one sub-batch
    with torch.no_grad():
        mag = torch.rand((1, 1, 33, 50), device=DEV)
        m(mag, mag, mag)
    with pytest.raises(_lib.FsnError, match="kept only by an audio call"):
        m.get_stage("enh", (1, 33, 50, 2), torch.device(DEV))
    assert np.array_equal(_run(m, rows, [3000, 2000]), before)
