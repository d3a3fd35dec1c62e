"""FullSubNet+ at BASELINE config #2's geometry (64 clips x 3 s, F = 257) with a narrow and a wide sub-band input: fb_num_neighbors 0
(Isb 34, layer 0's input projection fused into the recurrence) against fb_num_neighbors 15 (Isb 124, layer 0 projected by the
input-projection GEMM from rows of 128 halves, DESIGN.md §3.3).

    python scripts/bench_wide_subband.py [--steps 10] [--rounds 3] [--out DIR]

Prints one JSON line: the card's name and power limit (read in the same run); per model, alternated round by round on the same inputs,
the forward's ms per 64-clip step (CUDA events); then, in a separate torch.profiler run of one step of each model, the GPU time per
kernel name, so the cost of the wide layer-0 route is measured rather than estimated.  With --out the profiler tables go to
DIR/bench_wide_subband_profile.json.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().split(", ") + ["", "", ""])[:3] if q.returncode == 0 else ("", "", "")
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit_w": float(power) if power else None,
            "max_sm_clock_mhz": float(clk) if clk else None}


def build(fb):
    """The default FullSubNet+ (config/inference.toml) with fb_num_neighbors = fb, PyTorch default-style init; (model, Isb)"""
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = dict(sb_num_neighbors=15, fb_num_neighbors=fb, num_freqs=257, look_ahead=2, fb_output_activate_function="ReLU",
               sb_output_activate_function=False, channel_attention_model="TSSE", fb_model_hidden_size=512, sb_model_hidden_size=384,
               norm_type="offline_laplace_norm", num_groups_in_drop_band=2, kersize=[3, 5, 10], subband_num=1, sequence_model="LSTM")
    torch.manual_seed(0)
    m = FullSubNet_Plus(**cfg)
    return m.to("cuda:0").eval(), 2 * cfg["sb_num_neighbors"] + 1 + 3 * (2 * fb + 1)


def step_ms(m, x, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        s.record()
        for _ in range(steps):
            m(*x)
        e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=188, help="frames per clip (188: 3 s at 16 kHz, hop 256)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wide_subband.py measures on a CUDA GPU; none is visible")
    import __graft_entry__ as ge
    ge.build()
    from fsnplus_b200.synth import synth_clips
    from fsnplus_b200 import inference as inf
    X = inf.stft(synth_clips(a.batch, 256 * (a.frames - 1), 16000, seed=1000).to("cuda:0"), 512, 256, 512)
    x = (X.abs().unsqueeze(1).contiguous(), X.real.unsqueeze(1).contiguous(), X.imag.unsqueeze(1).contiguous())
    models = {fb: build(fb) for fb in (0, 15)}
    for m, _ in models.values():                                         # warm every shape
        step_ms(m, x, 2)
    times = {fb: [] for fb in models}
    for _ in range(a.rounds):
        for fb, (m, _) in models.items():
            times[fb].append(step_ms(m, x, a.steps))
    res = {"card": card(), "batch": a.batch, "frames": a.frames, "steps": a.steps, "rounds": a.rounds, "models": {}}
    for fb, (m, I) in models.items():
        res["models"][f"fb{fb}"] = {"isb": I, "lstm_impl": m.last_lstm_impl(), "ms_per_step": times[fb],
                                   "median_ms": statistics.median(times[fb]), "launches": m.last_launch_count()}
    prof = {}
    from torch.profiler import ProfilerActivity, profile
    for fb, (m, I) in models.items():
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            step_ms(m, x, 1)
        k = {}
        for ev in p.key_averages():
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            if t > 0:
                k[ev.key[:90]] = round(t / 1e3, 3)
        prof[f"fb{fb}"] = dict(sorted(k.items(), key=lambda kv: -kv[1]))
        res["models"][f"fb{fb}"]["kernel_ms_top"] = dict(list(prof[f"fb{fb}"].items())[:8])
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_wide_subband_profile.json"), "w") as f:
            json.dump(prof, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
