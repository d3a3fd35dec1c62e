"""Model files on the GPU (fsn_model_load, DESIGN.md §3.15): a handle loaded from a file saved by the Python module has the module's
weights_id, and its forward, enhanced spectrum and enhanced audio are bit-identical to the module's, for the six configurations of the
CPU tests; the default configuration stays under the cIRM bar against the reference golden; a C program loads an exported file and
enhances audio bit-identically; streaming sessions move from a Python-built handle to a file-loaded one; a corrupted file or other
weights are refused."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O
from test_model_file_cpu import CASES, ROOT, build, parse, small

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASK_TOL = 1e-3


class Loaded:
    """A handle from fsn_model_load, with what StreamingFullSubNet reads of a model (_handle, _cfg, look_ahead, _ensure_handle)."""

    def __init__(self, path):
        from fsnplus_b200 import _lib
        self.lib = _lib.load_library()
        h = C.c_void_p(1)                                                  # fsn_model_load sets it to NULL first
        rc = self.lib.fsn_model_load(os.fsencode(path), C.byref(h))
        assert rc == 0, self.lib.fsn_last_error()
        self._handle, self._cfg = h, _lib.model_file_config(path)
        self.look_ahead = self._cfg.look_ahead

    def _ensure_handle(self, device):
        return self.lib

    def keys(self):
        out = []
        for i in range(self.lib.fsn_model_num_params(self._handle)):
            key, numel = C.c_char_p(), C.c_int64()
            assert self.lib.fsn_model_param_info(self._handle, i, C.byref(key), C.byref(numel)) == 0
            out.append(key.value.decode())
        return out

    def close(self):
        self.lib.fsn_model_destroy(self._handle)


def _stream():
    return C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr() if t is not None else None)


def _inputs(F, B, T, seed):
    rng = np.random.default_rng(seed)
    real = torch.from_numpy((rng.standard_normal((B, 1, F, T)) * 0.05 + 0.004).astype(np.float32)).to(DEV)
    imag = torch.from_numpy((rng.standard_normal((B, 1, F, T)) * 0.05 - 0.003).astype(np.float32)).to(DEV)
    return torch.sqrt(real ** 2 + imag ** 2), real, imag


def _waves(lengths, seed, L=None):
    rng = np.random.default_rng(seed)
    L = L or max(lengths)
    rows = np.zeros((len(lengths), L), np.float32)
    for b, n in enumerate(lengths):
        rows[b, :n] = (rng.standard_normal(n) * 0.1).astype(np.float32)
    return rows


@pytest.mark.parametrize("name", list(CASES))
def test_loaded_handle_is_the_module(built_lib, tmp_path, name):
    """weights_id, the key list, the forward, the enhanced spectrum and the enhanced audio of the loaded handle equal the module's."""
    lib = built_lib
    m = build(name, seed=11).to(DEV)
    path = tmp_path / "m.fsn"
    m.save_model_file(path)
    h = Loaded(path)
    try:
        plus = m._kind == 0
        F, B, T = m._cfg.num_freqs, 2, 40
        mag, real, imag = _inputs(F, B, T, seed=12)
        with torch.no_grad():
            want = m(mag, real, imag) if plus else m(mag)
            want_enh = m.enhance_spectrum(mag, real, imag)
        assert lib.fsn_model_weights_id(h._handle) == m.weights_id() != 0
        assert h.keys() == [k for k, _ in parse(path.read_bytes(), verify_hash=False)["params"]]
        got = torch.empty_like(want)
        assert lib.fsn_model_forward(h._handle, _ptr(mag), _ptr(real if plus else None), _ptr(imag if plus else None), B, T, _ptr(got),
                                     _stream()) == 0, lib.fsn_last_error()
        got_enh = torch.empty_like(want_enh)
        assert lib.fsn_model_forward_enhance(h._handle, _ptr(mag), _ptr(real), _ptr(imag), B, T, _ptr(got_enh), _stream()) == 0
        lengths = [9000, 6001]
        wave = torch.from_numpy(_waves(lengths, seed=13)).to(DEV)
        want_audio = m.enhance_audio(wave, lengths)
        got_audio = torch.empty_like(wave)
        hl = (C.c_int64 * B)(*lengths)
        assert lib.fsn_model_enhance_audio(h._handle, _ptr(wave), B, wave.shape[1], hl, _ptr(got_audio), _stream()) == 0
        torch.cuda.synchronize()
        assert torch.equal(got, want) and torch.equal(got_enh, want_enh) and torch.equal(got_audio, want_audio)
    finally:
        h.close()


def test_default_config_meets_the_cirm_bar(built_lib, tmp_path, golden):
    """The default FullSubNet+ loaded from a file, on the reference golden's clip: cIRM rel-L2 <= 1e-3 against the reference output."""
    from fsnplus_b200.model import FullSubNet_Plus
    g = golden("plus_default")
    cfg = O.default_plus_config()
    params = O.make_params_plus(cfg, seed=int(g["seed"]), lstm_scale=float(g["lstm_scale"]))
    m = FullSubNet_Plus(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m.save_model_file(tmp_path / "m.fsn")
    h = Loaded(tmp_path / "m.fsn")
    try:
        x = [torch.from_numpy(np.ascontiguousarray(g[k])).to(DEV) for k in ("mag", "real", "imag")]
        out = torch.empty((1, 2) + tuple(x[0].shape[2:]), dtype=torch.float32, device=DEV)
        assert built_lib.fsn_model_forward(h._handle, *[_ptr(t) for t in x], 1, x[0].shape[3], _ptr(out), _stream()) == 0
        err = O.rel_l2(out.cpu().numpy(), g["out"])
        print(f"\n[default from file] cIRM rel-L2 vs reference {err:.3e}")
        assert err < MASK_TOL
    finally:
        h.close()


def test_c_program(built_lib, tmp_path):
    """tests/c_model_file.c on a file written by the exporter from a checkpoint: bit-identical to model.enhance_audio of the module the
    inference tool builds from the same checkpoint, and the same weights_id."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.tools import export, inference as T
    cc = shutil.which("cc") or shutil.which("gcc")
    assert cc, "no system C compiler"
    toml = tmp_path / "inference.toml"
    toml.write_text(open(os.path.join(ROOT, "tests", "golden", "inference_reference.toml")).read())
    conf = T.load_toml(toml)
    params = O.make_params_plus(O.default_plus_config(), seed=14)
    torch.save({"model": {k: torch.from_numpy(v) for k, v in params.items()}, "epoch": 1}, tmp_path / "ckpt.tar")
    export.main(["-C", str(toml), "-M", str(tmp_path / "ckpt.tar"), "-O", str(tmp_path / "model.fsn")])
    m, _ = T.build_model(conf["model"], tmp_path / "ckpt.tar", DEV)
    libdir = os.path.dirname(_lib.lib_path())
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    exe = tmp_path / "c_model_file"
    subprocess.run([cc, os.path.join(ROOT, "tests", "c_model_file.c"), "-o", str(exe), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(cuda, "include"), "-L", libdir, "-l:libfsnplus_b200.so", "-L", os.path.join(cuda, "lib64"),
                    "-lcudart", f"-Wl,-rpath,{libdir}:{os.path.join(cuda, 'lib64')}"], check=True)
    lengths = [16000, 9000, 8001, 4321]
    rows = _waves(lengths, seed=15)
    with open(tmp_path / "wave.bin", "wb") as f:
        f.write(struct.pack("<iq", *rows.shape) + np.asarray(lengths, np.int64).tobytes() + rows.tobytes())
    r = subprocess.run([str(exe), str(tmp_path / "model.fsn"), str(tmp_path / "wave.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(tmp_path / "out.bin", np.float32).reshape(rows.shape)
    want = m.enhance_audio(torch.from_numpy(rows).to(DEV), lengths).cpu().numpy()
    assert np.array_equal(got, want)
    assert f"weights_id {m.weights_id():016x}" in r.stdout, r.stdout


def test_sessions_move_to_a_file_loaded_handle(built_lib, tmp_path):
    """fullsubnet.Model with a cumulative norm: sessions saved from a handle built in Python load into a handle of the file-loaded model
    and continue bit-identically to the sessions left on the Python handle; a file of other weights is refused at load_slots."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import START, STEP, StreamingFullSubNet
    m = small().to(DEV)
    m.save_model_file(tmp_path / "m.fsn")
    small_other = build("fsn_gru_cumulative", seed=4, num_freqs=33, sb_num_neighbors=3, fb_model_hidden_size=32, sb_model_hidden_size=32)
    small_other.save_model_file(tmp_path / "other.fsn")
    h, other = Loaded(tmp_path / "m.fsn"), Loaded(tmp_path / "other.fsn")
    a = StreamingFullSubNet(m, batch_size=3)
    b = StreamingFullSubNet(h, batch_size=2)
    c = StreamingFullSubNet(other, batch_size=2)
    try:
        F, K, cut = m._cfg.num_freqs, 40, 17
        x = torch.from_numpy(np.abs(np.random.default_rng(16).standard_normal((3, F, K))).astype(np.float32)).to(DEV)
        for k in range(cut):
            a.step_slots(x[:, :, k], [START if k == 0 else STEP] * 3)
        state = a.save_slots([0, 2])
        b.load_slots([1, 0], state)                                      # session 0 -> slot 1, session 2 -> slot 0
        for k in range(cut, K):
            ma, va = a.step_slots(x[:, :, k], [STEP] * 3)
            mb, vb = b.step_slots(torch.stack([x[2, :, k], x[0, :, k]]), [STEP] * 2)
            assert torch.equal(mb[1], ma[0]) and torch.equal(mb[0], ma[2]), k
            assert bool(vb[1]) == bool(va[0]) and bool(vb[0]) == bool(va[2])
        with pytest.raises(_lib.FsnError, match="weights_id"):
            c.load_slots([0, 1], state)
    finally:
        for s in (a, b, c):
            s.close()
        h.close()
        other.close()


def test_corrupted_file(built_lib, tmp_path):
    """One flipped data byte: FSN_EINVAL naming the checksum, and *out is NULL."""
    m = small()
    m.save_model_file(tmp_path / "m.fsn")
    b = bytearray((tmp_path / "m.fsn").read_bytes())
    b[len(b) // 2] ^= 0x01
    (tmp_path / "bad.fsn").write_bytes(bytes(b))
    h = C.c_void_p(1)
    rc = built_lib.fsn_model_load(os.fsencode(tmp_path / "bad.fsn"), C.byref(h))
    assert rc == -1 and b"checksum mismatch" in built_lib.fsn_last_error()
    assert h.value is None
