"""The offline audio call (model.enhance_audio, fsn_model_enhance_audio) against the torch transforms around the spectral call.

    python scripts/bench_audio_offline.py [--steps 10] [--rounds 3] [--clips 256] [--profile DIR]

Default FullSubNet+ config (config/inference.toml) with the reference's weight initialisation, seeded synthetic clips.  Arms are
alternated --rounds times in one process; every timed pass ends in a device synchronise.
  (a) config #2: 64 x 3 s clips per step.  enhance_batch (torch.stft, the fused spectral call, torch.istft) against enhance_audio:
      ms per step, the library's launches per step, rel-L2 between the arms.
  (b) the bench_ragged.py workload: --clips clips of distinct lengths uniform in [1 s, 10 s], length-sorted batches of 64.
      enhance_ragged against enhance_audio(lengths=...): seconds of audio per second.
  (c) --profile DIR, a separate run: torch.profiler device time of the two transform kernels at config #2 and every kernel's count per
      step of both arms; the transforms' bandwidth is the bytes counted from the shapes over their kernel time.
Prints one JSON line with the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "fullsubnet-plus_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_ragged import DEFAULT_CONFIG, HOP, N_FFT, SR  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def transform_bytes(B, L, F, T):
    """Bytes the two transform kernels move at least: analysis reads B L samples and writes three [B, F, T] fp32 planes, synthesis
    reads the [B, F, T] complex64 spectrum and writes B L samples."""
    return 4 * B * L + 12 * B * F * T, 8 * B * F * T + 4 * B * L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_audio_offline.py measures on a CUDA device; none is available")
    from fsnplus_b200 import inference as H
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200.synth import synth_clips

    dev = torch.device("cuda:0")
    torch.manual_seed(args.seed)
    model = FullSubNet_Plus(**DEFAULT_CONFIG, weight_init=True).to(dev).eval()
    F = DEFAULT_CONFIG["num_freqs"]
    line = {"card": card()}

    # (a) config #2
    B, L = 64, 3 * SR
    x = synth_clips(B, num_samples=L, seed=args.seed).to(dev)
    T = L // HOP + 1
    arms = {"enhance_batch": lambda: H.enhance_batch(model, x, N_FFT, HOP, N_FFT), "enhance_audio": lambda: model.enhance_audio(x)}
    launches = {}
    with torch.no_grad():
        for name, fn in arms.items():                                   # warm-up: module loads, workspaces, iSTFT envelopes
            fn(); fn()
            launches[name] = model.last_launch_count()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            os.makedirs(args.profile, exist_ok=True)
            counts, dev_us = {}, {}
            for name, fn in arms.items():
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        fn()
                    torch.cuda.synchronize()
                prof.export_chrome_trace(os.path.join(args.profile, f"{name}.pt.trace.json"))
                ev = prof.key_averages()
                counts[name] = round(sum(e.count for e in ev if e.device_time_total > 0) / args.steps, 1)
                dev_us[name] = {e.key: round(e.device_time_total / e.count, 1) for e in ev
                                if e.count and ("audio_stft_kernel" in e.key or "audio_istft_kernel" in e.key)}
            ba, bs = transform_bytes(B, L, F, T)
            an = next((v for k, v in dev_us["enhance_audio"].items() if "audio_stft" in k), None)
            sy = next((v for k, v in dev_us["enhance_audio"].items() if "audio_istft" in k), None)
            line["profile"] = {"kernels_per_step": counts, "analysis_us": an, "synthesis_us": sy,
                               "analysis_MB": round(ba / 1e6, 1), "synthesis_MB": round(bs / 1e6, 1),
                               "analysis_TB_s": round(ba / an / 1e6, 2) if an else None,
                               "synthesis_TB_s": round(bs / sy / 1e6, 2) if sy else None}
            print(json.dumps(line))
            return
        ms = {k: [] for k in arms}
        for _ in range(args.rounds):
            for name, fn in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    y = fn()
                torch.cuda.synchronize()
                ms[name].append(round((time.perf_counter() - t0) * 1e3 / args.steps, 3))
                if name == "enhance_batch":
                    ya = y
                else:
                    yb = y
        errs = ((yb - ya).norm(dim=1) / ya.norm(dim=1)).max().item()
        line["a_config2_B64_3s"] = {"ms_per_step": ms, "library_launches_per_step": launches, "rel_l2_max": errs}

        # (b) the ragged workload
        g = torch.Generator().manual_seed(args.seed)
        lengths = (torch.randperm(9 * SR + 1, generator=g)[: args.clips] + SR).tolist()
        clips = [synth_clips(1, num_samples=int(n), seed=args.seed * 1000 + i)[0].to(dev) for i, n in enumerate(lengths)]
        audio_s = sum(lengths) / SR
        order = sorted(range(len(clips)), key=lambda i: lengths[i])
        batches = [order[i:i + args.batch] for i in range(0, len(order), args.batch)]
        rows = []
        for b in batches:                                               # [B, L_max] rows of each batch, built once outside the timing
            Lm = max(lengths[i] for i in b)
            r = torch.zeros((len(b), Lm), device=dev)
            for j, i in enumerate(b):
                r[j, :lengths[i]] = clips[i]
            rows.append((r, [lengths[i] for i in b]))

        def ragged():
            for b in batches:
                H.enhance_ragged(model, [clips[i] for i in b], N_FFT, HOP, N_FFT)

        def audio():
            for r, n in rows:
                model.enhance_audio(r, n)

        ragged(); audio()
        rates = {"enhance_ragged": [], "enhance_audio": []}
        for _ in range(args.rounds):
            for name, fn in (("enhance_ragged", ragged), ("enhance_audio", audio)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                rates[name].append(round(audio_s / (time.perf_counter() - t0), 1))
        line["b_ragged_256"] = {"audio_s": round(audio_s, 1), "batch": args.batch, "audio_s_per_s": rates,
                                "audio_over_ragged": round(sum(rates["enhance_audio"]) / sum(rates["enhance_ragged"]), 3)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
