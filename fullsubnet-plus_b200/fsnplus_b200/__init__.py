"""fsnplus_b200 -- H100-native (sm_90a) FullSubNet+/FullSubNet inference forward (host-side mirror of the reference API).

Drop-in: point ``config[model].path`` of the reference's TOML at
``fsnplus_b200.model.FullSubNet_Plus`` (or ``fsnplus_b200.model.Model``) with this directory's parent
(``fullsubnet-plus_b200/``) on ``sys.path``; see INTEGRATION.md.
"""
from ._lib import load_library, lib_path, FsnError  # noqa: F401

__all__ = ["load_library", "lib_path", "FsnError"]
