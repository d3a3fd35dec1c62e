"""FullSubNet+ with the TCN sub-band model against the LSTM one at BASELINE config #2's geometry (64 clips x 3 s, F = 257).

    python scripts/bench_sbtcn.py [--steps 10] [--rounds 3]

Prints one JSON line: the card's name and power limit (read in the same run), then per sub-band model, alternated round by round
on the same inputs: plain forward and fused-enhance ms per 64-clip step, the sub-band model's own ms (CUDA events around it),
frames/s and RTF; and for the sub-band TCN the FLOPs and HBM bytes it needs, counted from the shapes, with the achieved rates.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
TF32_FLOPS = 495e12                # H100 SXM data sheet, dense TF32 (the first 1x1 convolution); FP16 (the second): 989e12
FP16_FLOPS = 989e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().split(", ") + ["", "", ""])[:3] if q.returncode == 0 else ("", "", "")
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit_w": float(power) if power else None,
            "max_sm_clock_mhz": float(clk) if clk else None}


def sbtcn_counts(B, F, Tp, I, O, la):
    """Work and HBM traffic of the sub-band TCN per step, from the shapes.  Per row (sequence x frame) and block: the first 1x1
    convolution reads the fp32 stream (64 padded channels) and writes the fp16 hidden (512), the depth-wise convolution reads and
    writes 512 fp16 (halo reads ignored), the second 1x1 convolution reads the hidden and the old stream and writes the new stream
    (not in the last block, which writes the 2-float mask of frames >= look_ahead instead); plus the packer's input write."""
    rows = B * F * Tp
    flops = rows * (8 * (2 * 2 * I * 512 + 2 * 3 * 512) + 2 * I * O)
    per_block = 64 * 4 + 512 * 2 + 512 * 2 + 512 * 2 + 512 * 2 + 64 * 4 + 64 * 4
    hbm = rows * (8 * per_block - 64 * 4 + 64 * 4) + B * F * (Tp - la) * O * 4
    return rows, flops, hbm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200.synth import synth_clips
    from fsnplus_b200 import inference as inf

    dev = torch.device("cuda:0")
    B, nsamp, la = 64, 48000, 2
    cfg = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=la, fb_output_activate_function="ReLU",
               sb_output_activate_function=False, channel_attention_model="TSSE", fb_model_hidden_size=512, sb_model_hidden_size=384,
               norm_type="offline_laplace_norm", num_groups_in_drop_band=2, kersize=[3, 5, 10], subband_num=1)
    X = inf.stft(synth_clips(B, nsamp, 16000, seed=1000).to(dev), 512, 256, 512)
    mag, real, imag = X.abs().unsqueeze(1).contiguous(), X.real.unsqueeze(1).contiguous(), X.imag.unsqueeze(1).contiguous()
    T = mag.shape[-1]
    models = {}
    for kind in ("TCN", "LSTM"):
        torch.manual_seed(0)                                             # PyTorch default-style init through the reference's weight_init
        models[kind] = FullSubNet_Plus(**cfg, sequence_model=kind).to(dev).eval()

    def timed(fn, steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    res = {k: {"forward_ms": [], "enhance_ms": [], "subband_ms": []} for k in models}
    with torch.no_grad():
        for _ in range(args.rounds):
            for kind, m in models.items():
                res[kind]["forward_ms"].append(timed(lambda: m(mag, real, imag), args.steps))
                res[kind]["subband_ms"].append(statistics.median(x for x in m.lstm_ms_history(min(args.steps, 32)) if x > 0))
                res[kind]["enhance_ms"].append(timed(lambda: m.enhance_spectrum(mag, real, imag), args.steps))
                res[kind]["impl"] = m.last_lstm_impl()
    out = {"card": card(), "workload": f"config #2 geometry: B = {B} x 3 s clips, F = 257, T = {T}, default weights (seed 0)",
           "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "timing": "CUDA events; median over the alternated rounds"}
    for kind, r in res.items():
        fwd, enh, sub = (statistics.median(r[k]) for k in ("forward_ms", "enhance_ms", "subband_ms"))
        out[kind] = {"impl": r["impl"], "forward_ms": fwd, "enhance_ms": enh, "subband_ms": sub,
                     "frames_per_s": B * T / (enh / 1e3), "rtf": (enh / 1e3) / (B * nsamp / 16000),
                     "rounds": {k: r[k] for k in ("forward_ms", "enhance_ms", "subband_ms")}}
    rows, flops, hbm = sbtcn_counts(B, 257, T + la, 34, 2, la)
    sub = out["TCN"]["subband_ms"] / 1e3
    out["TCN"]["counts"] = {"rows": rows, "flop": flops, "hbm_bytes": hbm,
                            "achieved_tflop_s": flops / sub / 1e12, "achieved_gb_s": hbm / sub / 1e9,
                            "share_of_hbm_datasheet": hbm / sub / HBM_BYTES_PER_S,
                            "hbm_bound_ms": hbm / HBM_BYTES_PER_S * 1e3,
                            "tensor_bound_ms": (rows * 8 * 2 * 34 * 512 / TF32_FLOPS + rows * 8 * 2 * 512 * 34 / FP16_FLOPS) * 1e3}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
