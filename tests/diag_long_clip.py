#!/usr/bin/env python
"""Where does the error of the 30 s / x3-weights case (tests/test_gpu_round2.py::test_config4_30s_clip_parity, 9.7e-4 against a bar of
1e-3) come from?  Stage-wise: the full-band LSTM output (weight-stationary kernel) vs the CPU port, and the final mask when the sub-band
stage is fed (a) its own full-band output, (b) nothing else changed -- run on a GPU."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]
from oracle import fsn_oracle as O  # noqa: E402
from oracle.torch_port import TorchPort  # noqa: E402
from fsnplus_b200.model import Model  # noqa: E402

DEV = "cuda:0"
for scale in (1.0, 3.0):
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=21, lstm_scale=scale)
    mag = np.abs(O.stft(O.synth_clips(1, num_samples=480000, seed0=78)))[:, None].astype(np.float32)
    port = TorchPort(params, cfg, "fsn", dtype=torch.float32)
    x = F.pad(torch.from_numpy(mag), [0, 2])
    B, _, Fq, T = x.shape
    with torch.no_grad():
        fb_ref = port.seq_lstm(port.norm(x).reshape(B, Fq, T), "fb_model", cfg["fb_output_activate_function"]).numpy()
        ref = port.forward(torch.from_numpy(mag)).numpy()
    m = Model(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    for fast in (True, False):
        m2 = Model(**cfg, fast_math=fast)
        m2.load_state_dict(m.state_dict())
        m2 = m2.to(DEV).eval()
        with torch.no_grad():
            out = m2(torch.from_numpy(mag).to(DEV)).cpu().numpy()
        fb = m2.get_stage("fb_out", (1, 1, 257, T), DEV).cpu().numpy()[0]
        seg = lambda a, b, lo, hi: O.rel_l2(a[..., lo:hi], b[..., lo:hi])
        print(f"x{scale} fast_math={fast}: fb_out {O.rel_l2(fb, fb_ref):.3e} (first 3 s {seg(fb, fb_ref, 0, 188):.3e}, last 3 s {seg(fb, fb_ref, T - 188, T):.3e});  "
              f"mask {O.rel_l2(out, ref):.3e} (first 3 s {seg(out, ref, 0, 188):.3e}, last 3 s {seg(out, ref, T - 190, T - 2):.3e})")
