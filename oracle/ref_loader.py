"""Import the UNMODIFIED reference package (from its checkout, make_ref.SRC, else from the verbatim copy oracle/_ref/ made by
oracle/make_ref.py) with the two stubs it needs in this image.

TEST / BENCH INFRASTRUCTURE ONLY (see oracle/__init__.py).

The reference imports ``librosa`` (audio_zen/acoustics/feature.py:3, base_inferencer.py:5) and ``soundfile``
(base_inferencer.py:7) at module scope; neither is installed here and there is no network.  The model path never calls them
(SURVEY.md 8c), so empty stub modules are enough for the model classes; the inferencer needs ``librosa.stft/istft`` only as
attribute look-ups for two unused partials (base_inferencer.py:54-55) and ``soundfile.write`` as its output sink, which the
stub records in ``soundfile.written``.
"""
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))


def reference_root():
    from oracle.make_ref import SRC
    for root in (SRC, os.path.join(HERE, "_ref")):
        if os.path.isdir(os.path.join(root, "speech_enhance", "fullsubnet_plus")):
            return root
    return None


def available():
    return reference_root() is not None


def _stubs():
    if "librosa" not in sys.modules:
        lib = types.ModuleType("librosa")

        def _absent(*a, **k):
            raise RuntimeError("librosa is not installed in this image (stub): the model path never calls it")
        lib.stft = lib.istft = lib.load = _absent      # base_inferencer.py:54-55 wraps them in functools.partial (must be callable)
        lib.util = types.ModuleType("librosa.util")
        sys.modules["librosa"], sys.modules["librosa.util"] = lib, lib.util
    if "soundfile" not in sys.modules:
        sf = types.ModuleType("soundfile")
        sf.written = {}

        def write(path, data, samplerate=None, **kw):
            sf.written[str(path)] = (data, samplerate)
        sf.write = write
        sys.modules["soundfile"] = sf
    return sys.modules["librosa"], sys.modules["soundfile"]


def setup():
    """Put the reference on sys.path (both roots it imports from, SURVEY.md 8c) and install the stubs.  Returns the root."""
    root = reference_root()
    if root is None:
        raise RuntimeError("the reference is not available: neither its checkout (FSN_REFERENCE_SRC) nor oracle/_ref/ (run "
                           "oracle/make_ref.py where the checkout exists)")
    os.environ.setdefault("PYTHONDONTWRITEBYTECODE", "1")
    sys.dont_write_bytecode = True
    _stubs()
    for p in (os.path.join(root, "speech_enhance"), root):
        if p not in sys.path:
            sys.path.insert(0, p)
    return root


def model_classes():
    """(FullSubNet_Plus, fullsubnet.Model) of the unmodified reference."""
    setup()
    from fullsubnet_plus.model.fullsubnet_plus import FullSubNet_Plus
    from fullsubnet.model.fullsubnet import Model
    return FullSubNet_Plus, Model


class ReferenceCpu:
    """The reference's own CPU PyTorch path for the model forward: the unmodified class, ``load_state_dict`` of the given
    parameters, ``eval()``, one clip per call under ``no_grad`` -- exactly what its inferencer issues
    (fullsubnet_plus/inferencer/inferencer.py:149-151, base_inferencer.py:65-69)."""

    def __init__(self, params, cfg, kind="plus"):
        import numpy as np
        import torch
        Plus, Fsn = model_classes()
        self.torch = torch
        self.model = (Plus if kind == "plus" else Fsn)(**cfg)
        self.model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in params.items()}, strict=True)
        self.model.eval()
        self.kind = kind

    def forward(self, mag, real=None, imag=None):
        with self.torch.no_grad():
            return self.model(mag, real, imag) if self.kind == "plus" else self.model(mag)
