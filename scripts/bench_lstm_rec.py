"""The sub-band LSTM recurrence (`lstm_tc5r_kernel`) inside a forward: its time per layer, per step and against its MMA bound.

    python scripts/bench_lstm_rec.py [--config 2 5] [--steps 5]

Runs bench.py's workload (config #2: 64 x 3 s clips, F = 257, hidden 384, 2 layers; config #5: 32 x 3 s, F = 513, hidden 512,
3 layers) through `enhance_spectrum`, a few forwards under torch.profiler, and prints one JSON line with the card's name, power
limit and maximum SM clock.  Per layer: ms per forward (median over the forwards), and us per step of one CTA, i.e. the layer's
time over (waves x T'), with waves = CTAs / (2 x 66 clusters on 132 SMs) rounded up.  The MMA bound of one CTA step is
64 x K x 4H x 2 FLOP (K = H, plus the 64-wide input k-block on the first layer) at 4096 dense fp16 FLOP per clock and SM; it is
given in clocks, and in us at the maximum SM clock (a loaded, power-capped card holds less, so the bound in us is then longer).
The kernels of one forward run in layer order, so the n-th recurrence launch of a forward is layer n.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]

SM_COUNT_CLUSTERS = 66          # CTA pairs resident at one CTA per SM on 132 SMs


def smi(fields):
    q = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip().split(", ") if q.returncode == 0 else []


def one_config(cid, steps, max_mhz):
    import bench
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200.synth import synth_clips
    from fsnplus_b200 import inference as inf
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda:0")
    w = bench.workload(cid, 0)
    c, B, L = w["cfg"], w["B"], w["L"]
    X = inf.stft(synth_clips(B, w["nsamp"], 16000, seed=1000).to(dev), w["n_fft"], w["hop"], w["n_fft"])
    mag, real, imag = X.abs().unsqueeze(1).contiguous(), X.real.unsqueeze(1).contiguous(), X.imag.unsqueeze(1).contiguous()
    torch.manual_seed(0)
    m = FullSubNet_Plus(**c, num_layers=L).to(dev).eval()
    F, H, Tp = c["num_freqs"], c["sb_model_hidden_size"], X.shape[-1] + c["look_ahead"]
    ctas = ((B * F + 127) // 128 + 1) // 2 * 2 * 2                  # two CTAs per 128-row tile, tiles padded to pairs
    waves = math.ceil(ctas / (2 * SM_COUNT_CLUSTERS))
    with torch.no_grad():
        for _ in range(3):
            m.enhance_spectrum(mag, real, imag)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                m.enhance_spectrum(mag, real, imag)
            torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "lstm_tc5r_kernel" in e.name),
                  key=lambda e: e.time_range.start)
    durs = [e.time_range.elapsed_us() for e in kern]
    if len(durs) != steps * L:
        raise SystemExit(f"config {cid}: {len(durs)} recurrence kernels in {steps} forwards, expected {steps * L}")
    layers = []
    for l in range(L):
        ms = statistics.median(durs[l::L]) / 1e3
        K = H + (64 if l == 0 else 0)
        bound_clk = 64 * K * 4 * H * 2 / 4096
        layers.append({"layer": l, "ms_per_forward": ms, "us_per_cta_step": ms * 1e3 / (waves * Tp), "mma_bound_clk_per_step": bound_clk,
                       "mma_bound_us_per_step_at_max_clock": bound_clk / max_mhz if max_mhz else None})
    return {"config": cid, "B": B, "F": F, "H": H, "layers": L, "Tp": Tp, "ctas": ctas, "waves": waves, "forwards": steps,
            "recurrence": layers, "launches_per_forward": m.last_launch_count()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, nargs="+", default=[2, 5], choices=[2, 5])
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    name, power, mhz = (smi("name,power.limit,clocks.max.sm") + ["", "", ""])[:3]
    max_mhz = float(mhz) if mhz else None
    out = {"card": {"name": name or torch.cuda.get_device_name(0), "power_limit_w": float(power) if power else None, "max_sm_clock_mhz": max_mhz}}
    out["runs"] = [one_config(c, args.steps, max_mhz) for c in args.config]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
