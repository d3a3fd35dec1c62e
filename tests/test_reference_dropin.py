"""The drop-in claim of INTEGRATION.md, executed: the reference's OWN loader and inferencer code (unmodified, imported from the
checkout named by FSN_REFERENCE_SRC or from the verbatim copy oracle/_ref/) driving ``fsnplus_b200.model.FullSubNet_Plus`` after
changing ONE string of config/inference.toml (``[model] path``).

  reference code on this path: audio_zen/utils.py:63-99 (initialize_module), audio_zen/inferencer/base_inferencer.py:22-60,97-110
  (_load_model: initialize_module + torch.load + load_state_dict + .to(device) + .eval()), :133-160 (__call__: int16 scaling,
  sf.write) and fullsubnet_plus/inferencer/inferencer.py:140-165 (mag_complex_full_band_crm_mask).

CPU test: everything up to the forward (construction from the shipped TOML's [model.args], strict checkpoint load, eval) and the
documented error on CPU tensors.  GPU test: the whole reference inferencer loop with the model on the GPU, its written int16
waveform compared with the golden waveform of the all-reference pipeline.
"""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O
from oracle import ref_loader

HERE = os.path.dirname(os.path.abspath(__file__))
needs_ref = pytest.mark.skipif(not ref_loader.available(), reason="reference not available (neither its checkout nor oracle/_ref)")


def _config(tmp_path, clips):
    import toml
    root = ref_loader.setup()
    cfg = toml.load(os.path.join(root, "config", "inference.toml"))
    assert cfg["model"]["path"] == "fullsubnet_plus.model.fullsubnet_plus.FullSubNet_Plus"
    cfg["model"]["path"] = "fsnplus_b200.model.FullSubNet_Plus"          # <- the one-string swap of INTEGRATION.md
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    np.save(tmp_path / "clips.npy", clips)
    cfg["dataset"] = {"path": "dropin_dataset.Dataset", "args": {"npy_path": str(tmp_path / "clips.npy"), "sr": 16000}}
    ckpt = tmp_path / "ckpt.tar"
    params = O.make_params_plus(O.default_plus_config(), seed=0)
    torch.save({"model": {k: torch.from_numpy(v) for k, v in params.items()}, "epoch": 7}, ckpt)
    return cfg, ckpt


@needs_ref
def test_reference_loader_builds_and_loads_the_dropin_class(tmp_path, built_lib):
    cfg, ckpt = _config(tmp_path, O.synth_clips(1).astype(np.float32))
    from audio_zen.utils import initialize_module
    from audio_zen.inferencer.base_inferencer import BaseInferencer
    from fsnplus_b200.model import FullSubNet_Plus
    m = initialize_module(cfg["model"]["path"], args=cfg["model"]["args"])
    assert isinstance(m, FullSubNet_Plus)
    model, epoch = BaseInferencer._load_model(cfg["model"], ckpt, torch.device("cpu"))      # strict load_state_dict inside
    assert isinstance(model, FullSubNet_Plus) and epoch == 7 and not model.training
    assert sum(p.numel() for p in model.parameters()) == 8675102                           # SURVEY.md 8a
    # same keys and shapes as the reference class built from the same TOML section
    Plus, _ = ref_loader.model_classes()
    ref_sd = Plus(**cfg["model"]["args"]).state_dict()
    sd = model.state_dict()
    assert list(sd.keys()) == list(ref_sd.keys())
    assert all(sd[k].shape == ref_sd[k].shape for k in sd)
    x = torch.zeros(1, 1, 257, 10)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model(x, x, x)


@needs_ref
@pytest.mark.gpu
def test_reference_inferencer_runs_the_dropin_model_on_gpu(tmp_path, built_lib, golden):
    """tools/inference.py:11-18 of the reference, verbatim: initialize_module(inferencer path) -> Inferencer(config, ckpt, out)()."""
    g = golden("plus_default")
    clips = O.synth_clips(2).astype(np.float32)                            # clip 0 is the golden clip
    cfg, ckpt = _config(tmp_path, clips)
    _, sf = ref_loader._stubs()
    sf.written.clear()
    from audio_zen.utils import initialize_module
    inferencer_class = initialize_module(cfg["inferencer"]["path"], initialize=False)
    inferencer = inferencer_class(cfg, ckpt, tmp_path / "out")
    from fsnplus_b200.model import FullSubNet_Plus
    assert isinstance(inferencer.model, FullSubNet_Plus) and inferencer.device.type == "cuda"
    inferencer()
    names = sorted(os.path.basename(k) for k in sf.written)
    assert names == ["clip0.wav", "clip1.wav"]
    key = [k for k in sf.written if k.endswith("clip0.wav")][0]
    assert os.path.basename(os.path.dirname(key)) == "enhanced_0007"
    pcm, rate = sf.written[key]
    want = np.int16(0.8 * np.iinfo(np.int16).max * g["enhanced"][0] / np.max(np.abs(g["enhanced"][0])))     # base_inferencer.py:151-152
    assert rate == 16000 and pcm.dtype == np.int16 and pcm.shape == want.shape
    err = O.rel_l2(pcm.astype(np.float64), want.astype(np.float64))
    print(f"\n[reference inferencer + drop-in model] int16 waveform vs all-reference pipeline: rel-L2 {err:.3e}, "
          f"max |diff| {np.abs(pcm.astype(int) - want.astype(int)).max()} LSB")
    assert err < 2e-3
