"""Ragged batches against today's exact-length strategy of the command line, on 256 synthetic clips of distinct lengths.

    python scripts/bench_ragged.py [--clips 256] [--batch 64] [--rounds 2]

Inputs: seeded synthetic clips (fsnplus_b200.synth) with distinct lengths uniform in [1 s, 10 s], the default FullSubNet+ config
with the reference's weight initialisation.  Two arms, alternated --rounds times in one process, no file I/O:
  A  the command line's default: exact-length buckets (here one clip each, the lengths are distinct), 4 CUDA streams with one
     model replica each (fsnplus_b200.tools.inference.run), enhance_batch per bucket;
  B  length-sorted ragged batches of --batch clips through enhance_ragged, one stream, one model.
Prints one JSON line: audio seconds enhanced per second of each arm (every pass ends in a device synchronise), the padded-frame
fraction of B, per-clip rel-L2 of B against A, and the card's name and power limit read in the same run.
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

SR, N_FFT, HOP = 16000, 512, 256
# the reference's config/inference.toml model arguments
DEFAULT_CONFIG = dict(num_freqs=257, look_ahead=2, sequence_model="LSTM", fb_num_neighbors=0, sb_num_neighbors=15,
                      fb_output_activate_function="ReLU", sb_output_activate_function=False, channel_attention_model="TSSE",
                      fb_model_hidden_size=512, sb_model_hidden_size=384, norm_type="offline_laplace_norm", num_groups_in_drop_band=2,
                      kersize=[3, 5, 10], subband_num=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ragged.py measures on a CUDA device; none is available")
    from fsnplus_b200 import inference as H
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200.synth import synth_clips

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(args.seed)
    lengths = torch.randperm(9 * SR + 1, generator=g)[: args.clips] + SR          # distinct, uniform in [1 s, 10 s]
    clips = [synth_clips(1, num_samples=int(n), seed=args.seed * 1000 + i)[0].to(dev) for i, n in enumerate(lengths.tolist())]
    audio_s = float(lengths.sum()) / SR

    cfg = dict(DEFAULT_CONFIG, weight_init=True)
    torch.manual_seed(args.seed)
    base = FullSubNet_Plus(**cfg)
    models = []
    for _ in range(args.streams):
        mk = FullSubNet_Plus(**cfg)
        mk.load_state_dict(base.state_dict())
        models.append(mk.to(dev).eval())
    streams = [torch.cuda.Stream(dev) for _ in range(args.streams)]

    order = sorted(range(len(clips)), key=lambda i: clips[i].numel())
    batches = [order[i:i + args.batch] for i in range(0, len(order), args.batch)]
    frames = [1 + c.numel() // HOP for c in clips]
    padded = sum(len(b) * max(frames[i] for i in b) for b in batches)
    pad_frac = 1.0 - sum(frames) / padded

    def arm_a():
        out = [None] * len(clips)
        main = torch.cuda.current_stream(dev)
        for s in streams:
            s.wait_stream(main)
        for i, c in enumerate(clips):
            k = i % args.streams
            with torch.cuda.stream(streams[k]):
                out[i] = H.enhance_batch(models[k], c[None], N_FFT, HOP, N_FFT)[0]
        torch.cuda.synchronize(dev)
        return out

    def arm_b():
        out = [None] * len(clips)
        for b in batches:
            for i, y in zip(b, H.enhance_ragged(models[0], [clips[i] for i in b], N_FFT, HOP, N_FFT)):
                out[i] = y
        torch.cuda.synchronize(dev)
        return out

    arm_a(); arm_b()                                                               # warm-up: module loads, workspaces, iSTFT envelopes
    rates = {"A": [], "B": []}
    for _ in range(args.rounds):
        for name, fn in (("A", arm_a), ("B", arm_b)):
            t0 = time.perf_counter()
            res = fn()
            rates[name].append(audio_s / (time.perf_counter() - t0))
            if name == "A":
                ya = res
            else:
                yb = res
    errs = sorted(float((b - a).norm() / a.norm()) for a, b in zip(ya, yb))
    line = {
        "card": card(),
        "clips": len(clips), "audio_s": round(audio_s, 1), "batch": args.batch, "streams_A": args.streams,
        "A_exact_length_streams_audio_s_per_s": [round(r, 1) for r in rates["A"]],
        "B_ragged_audio_s_per_s": [round(r, 1) for r in rates["B"]],
        "B_over_A": round(sum(rates["B"]) / sum(rates["A"]), 3),
        "B_padded_frame_fraction": round(pad_frac, 4),
        "rel_l2_B_vs_A": {"median": errs[len(errs) // 2], "max": errs[-1]},
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
