"""Cost of attenuation limits (DESIGN.md §3.18).

  * offline: BASELINE config #2 (default FullSubNet+, B = 64 clips of 4 s) through enhance_audio with no limit, every clip at 12 dB and
    half the clips at 12 dB, the three arms alternated call by call;
  * live: 1280 audio sessions stepping K = 32 hops per call (bench_stream_audio_chunks' workload, every slot STEPping) with and without
    per-slot limits, alternated; real time means the p99 call stays under K x 16 ms.
Prints one JSON line per arm with the GPU name, power limit and max SM clock read in the same run.

    python scripts/bench_atten_lim.py [--iters 20] [--sessions 1280] [--K 32] [--out DIR]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200"), os.path.join(ROOT, "scripts")]
from bench_stream_audio_chunks import CFG, HOP, gpu_info, stats, timed  # noqa: E402
from fsnplus_b200.model import FullSubNet_Plus, Model  # noqa: E402
from fsnplus_b200.streaming import START, STEP, StreamingFullSubNet  # noqa: E402
from bench import plus_cfg  # noqa: E402

DEV = "cuda:0"


def offline(iters):
    torch.manual_seed(0)                                           # PyTorch default init, as bench.py
    m = FullSubNet_Plus(**plus_cfg()).to(DEV).eval()
    x = (0.05 * torch.randn(64, 64000, generator=torch.Generator().manual_seed(3))).to(DEV)
    arms = {"none": None, "all_12dB": 12.0, "half_12dB": [12.0 if b % 2 else float("inf") for b in range(64)]}
    t = {k: [] for k in arms}
    with torch.no_grad():
        for k, v in arms.items():                                  # warm-up of every arm
            m.enhance_audio(x, atten_lim_db=v)
        torch.cuda.synchronize()
        for _ in range(iters):
            for k, v in arms.items():
                t[k] += timed(lambda i: m.enhance_audio(x, atten_lim_db=v), 1)
    return {k: {"median_ms": round(float(np.median(v)), 3), "min_ms": round(float(np.min(v)), 3)} for k, v in t.items()}


def live(B, K, iters):
    torch.manual_seed(0)
    m = Model(**CFG).to(DEV).eval()
    x = (0.05 * torch.randn(B, K * HOP, generator=torch.Generator().manual_seed(5))).to(DEV)
    res = {}
    handles = {}
    for arm in ("none", "per_slot"):
        st = StreamingFullSubNet(m, batch_size=B, device=DEV)
        if arm == "per_slot":
            st.set_atten_lim(list(range(B)), [float(6 + (b % 4) * 6) for b in range(B)])
        st.step_audio_chunk(x, [START] * B, [K] * B)
        st.step_audio_chunk(x, [STEP] * B, [K] * B)                # warm-up
        handles[arm] = st
    t = {k: [] for k in handles}
    for _ in range(iters):
        for k, st in handles.items():
            t[k] += timed(lambda i: st.step_audio_chunk(x, [STEP] * B, [K] * B), 1)
    for k, st in handles.items():
        res[k] = stats(t[k], B, K)
        st.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--sessions", type=int, default=1280)
    ap.add_argument("--K", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_atten_lim.py needs a CUDA device")
    gpu = gpu_info()
    lines = [{"bench": "atten_lim_offline", "config": 2, "gpu": gpu, **offline(a.iters)},
             {"bench": "atten_lim_live", "sessions": a.sessions, "K": a.K, "gpu": gpu, **live(a.sessions, a.K, a.iters)}]
    for r in lines:
        print(json.dumps(r))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_atten_lim.json"), "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
