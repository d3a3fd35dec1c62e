#!/usr/bin/env python
"""BASELINE config #4: streaming/causal mode, look_ahead = 2 frames, one 30 s synthetic 16 kHz clip, per-frame latency
p50/p99 on one GPU.  Model: fullsubnet.Model (default hyper-parameters) + cumulative_laplace_norm, stepped frame by frame
through the stateful C-ABI step API; every frame is synchronised (a real-time caller needs the mask before the next hop)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]
from fsnplus_b200 import inference as inf  # noqa: E402
from fsnplus_b200.model import Model  # noqa: E402
from fsnplus_b200.streaming import StreamingFullSubNet  # noqa: E402
from fsnplus_b200.synth import synth_clips  # noqa: E402


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 1
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    cfg = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM",
               fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=512,
               sb_model_hidden_size=384, weight_init=False, norm_type="cumulative_laplace_norm", num_groups_in_drop_band=2)
    model = Model(**cfg).to(dev).eval()
    clip = synth_clips(B, 480000, 16000, seed=77).to(dev)
    mag = inf.stft(clip).abs().contiguous()                       # [B, 257, 1876]
    T = mag.shape[-1]
    st = StreamingFullSubNet(model, batch_size=B, device=dev)
    for t in range(20):                                           # warm-up
        st.step(mag[:, :, t].contiguous())
    torch.cuda.synchronize()
    st.close()
    st = StreamingFullSubNet(model, batch_size=B, device=dev)
    lat = []
    frames = [mag[:, :, t].contiguous() for t in range(T)]
    for t in range(T):
        t0 = time.perf_counter()
        st.step(frames[t])
        torch.cuda.synchronize()
        lat.append((time.perf_counter() - t0) * 1e3)
    lat = np.array(lat)
    print(json.dumps({"config": "BASELINE #4: streaming fullsubnet.Model + cumulative_laplace_norm, look_ahead=2, 30 s clip", "batch": B,
                      "frames": int(T), "hop_ms": 16.0, "algorithmic_latency_ms": 16.0 * 3,
                      "per_frame_ms": {"p50": float(np.percentile(lat, 50)), "p99": float(np.percentile(lat, 99)),
                                       "mean": float(lat.mean()), "max": float(lat.max())},
                      "rtf": float(lat.sum() / 1e3 / 30.0)}))


if __name__ == "__main__":
    main()
