"""Sample-granular audio sessions (fsn_stream_step_audio_samples, DESIGN.md §3.19) on the config #4 model.

B sessions (1280 and 1024) are fed packets of P samples (160 = 10 ms and 320 = 20 ms at 16 kHz), staggered so that their hop
boundaries do not line up: slot b starts with b * 37 mod 256 samples already pending.  Each call delivers one packet to every slot.
Against it, in the same run and alternating with it call by call, the hop-aligned arms on the same audio: the per-hop call
(fsn_stream_step_audio_slots, one hop per slot) and the K-hop call at K = 2 (fsn_stream_step_audio_chunk).  Reported per case: device
time per call (CUDA events; median and p99), session-hops per second, and whether the p99 fits the packet period (P / 16 ms per hop).
Also the largest tested session count whose p99 fits.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200"), os.path.join(ROOT, "scripts")]
from bench_stream_audio_chunks import CFG, HOP, HOP_MS, Model, gpu_info  # noqa: E402
from fsnplus_b200.streaming import START, STEP, StreamingFullSubNet  # noqa: E402


def run(m, B, P, calls, warmup):
    dev = torch.device("cuda:0")
    smp, per, kh = (StreamingFullSubNet(m, batch_size=B, device=dev) for _ in range(3))
    x = torch.randn(B, max(P, 2 * HOP), device=dev) * 0.05
    start = torch.full((B,), START, dtype=torch.int32)
    step = torch.full((B,), STEP, dtype=torch.int32)
    # the staggered start: slot b holds b * 37 mod hop samples, then one hop each on the hop arms
    smp.step_audio_samples(x, torch.tensor([b * 37 % HOP for b in range(B)], dtype=torch.int32), start)
    per.step_audio(x[:, :HOP], start)
    kh.step_audio_chunk(x[:, :2 * HOP], start, torch.full((B,), 2, dtype=torch.int32))
    counts = torch.full((B,), P, dtype=torch.int32)
    twos = torch.full((B,), 2, dtype=torch.int32)
    arms = {"samples": lambda: smp.step_audio_samples(x[:, :P], counts, step),
            "per_hop": lambda: per.step_audio(x[:, :HOP], step),
            "k_hop_2": lambda: kh.step_audio_chunk(x[:, :2 * HOP], step, twos)}
    t = {k: [] for k in arms}
    ev = [torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)]
    for i in range(warmup + calls):
        for k, fn in arms.items():                          # alternate the arms call by call
            ev[0].record()
            fn()
            ev[1].record()
            ev[1].synchronize()
            if i >= warmup:
                t[k].append(ev[0].elapsed_time(ev[1]))
    for h in (smp, per, kh):
        h.close()
    hops = {"samples": B * P / HOP, "per_hop": B, "k_hop_2": 2 * B}
    period = {"samples": P / HOP * HOP_MS, "per_hop": HOP_MS, "k_hop_2": 2 * HOP_MS}
    res = {}
    for k, v in t.items():
        v = np.array(v)
        med, p99 = float(np.median(v)), float(np.percentile(v, 99))
        res[k] = {"median_ms": round(med, 3), "p99_ms": round(p99, 3), "session_hops_per_s": round(hops[k] / med * 1e3),
                  "period_ms": round(period[k], 2), "real_time": p99 < period[k]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", type=int, nargs="+", default=[1280, 1024])
    ap.add_argument("--packets", type=int, nargs="+", default=[160, 320])
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    a = ap.parse_args()
    torch.manual_seed(0)
    m = Model(**CFG).to("cuda:0").eval()
    info = gpu_info()
    best = {}
    for P in a.packets:
        for B in a.sessions:
            r = run(m, B, P, a.calls, a.warmup)
            print(json.dumps({"gpu": info, "B": B, "packet": P, **r}), flush=True)
            if r["samples"]["real_time"]:
                best[P] = max(best.get(P, 0), B)
    print(json.dumps({"gpu": info, "largest_real_time_sessions": best}), flush=True)


if __name__ == "__main__":
    main()
