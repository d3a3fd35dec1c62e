#!/usr/bin/env python
"""Chunked streaming steps (fsn_stream_step_chunk, DESIGN.md §3.13) against per-frame slot steps on BASELINE config #4's model.

Per session count B and chunk size K, every slot steps every call (sessions in steady state, started before the timed window).  The
chunk arm makes one fsn_stream_step_chunk call of K frames; the per-frame arm makes K fsn_stream_step_slots calls; the arms alternate
(--reps rounds of --iters calls each) on two handles of the same model, and every call (or group of K ticks) ends in a synchronise.
Reported: device time per call (CUDA events, median and p99), session-frames per second, and per K the largest B whose p99 stays under
K x 16 ms (the real-time budget of K hops).  --profile instead traces the chunk arm at one (B, K) under torch.profiler and reports the
device time per call of every kernel.

    python scripts/bench_stream_chunks.py [--sessions 256,512,1024,1280,1536,2048] [--K 8,16,32,64] [--iters 20] [--reps 2] [--out DIR]
    python scripts/bench_stream_chunks.py --profile [--sessions 1280] [--K 32]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]
from fsnplus_b200.model import Model  # noqa: E402
from fsnplus_b200.streaming import START, STEP, StreamingFullSubNet  # noqa: E402

HOP_MS = 16.0
CFG = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM",
           fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=512,
           sb_model_hidden_size=384, weight_init=False, norm_type="cumulative_laplace_norm", num_groups_in_drop_band=2)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def arm_times(st, x, K, iters, chunk):
    """Device ms of `iters` calls: one chunk call of K frames, or K per-frame slot calls."""
    B = st.B
    flags = [STEP] * B
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        if chunk:
            st.step_chunk(x, flags)
        else:
            for k in range(K):
                st.step_slots(x[:, :, k], flags)
        b.record()
        b.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="256,512,1024,1280,1536,2048")
    ap.add_argument("--K", default="8,16,32,64")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA GPU"
    dev = "cuda:0"
    torch.manual_seed(0)
    model = Model(**CFG).to(dev).eval()
    Bs, Ks = [int(v) for v in args.sessions.split(",")], [int(v) for v in args.K.split(",")]
    info = gpu_info()
    rows = []
    rng = np.random.default_rng(1)
    for B in Bs:
        chunk_h, frame_h = StreamingFullSubNet(model, B, dev), StreamingFullSubNet(model, B, dev)
        x0 = torch.from_numpy(np.abs(rng.standard_normal((B, 257, 4))).astype(np.float32) * 0.1).to(dev)
        chunk_h.step_chunk(x0, [START] * B)
        for k in range(4):
            frame_h.step_slots(x0[:, :, k].contiguous(), [START if k == 0 else STEP] * B)
        for K in Ks:
            x = torch.from_numpy(np.abs(rng.standard_normal((B, 257, K))).astype(np.float32) * 0.1).to(dev)
            if args.profile:
                arm_times(chunk_h, x, K, 3, True)
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    arm_times(chunk_h, x, K, args.iters, True)
                per = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    if t:
                        per[e.key] = per.get(e.key, 0.0) + t / 1e3 / args.iters
                tot = sum(per.values())
                line = {"gpu": info, "B": B, "K": K, "ms_per_call_total": round(tot, 3),
                        "kernels_ms_per_call": {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}}
                print(json.dumps(line)); rows.append(line)
                continue
            arm_times(chunk_h, x, K, 2, True); arm_times(frame_h, x, K, 1, False)       # warm-up of this shape
            ch, fr = [], []
            for _ in range(args.reps):
                ch += arm_times(chunk_h, x, K, args.iters, True)
                fr += arm_times(frame_h, x, K, args.iters, False)
            line = {"gpu": info, "B": B, "K": K}
            for name, t in (("chunk", ch), ("per_frame", fr)):
                t = np.array(t)
                med, p99 = float(np.median(t)), float(np.percentile(t, 99))
                line[name] = {"median_ms": round(med, 3), "p99_ms": round(p99, 3), "session_frames_per_s": round(B * K / med * 1e3),
                              "real_time": p99 < K * HOP_MS}
            print(json.dumps(line)); rows.append(line)
        chunk_h.close(); frame_h.close()
    if not args.profile:
        for K in Ks:
            for name in ("chunk", "per_frame"):
                ok = [r["B"] for r in rows if "chunk" in r and r["K"] == K and r[name]["real_time"]]
                cap = {"gpu": info, "K": K, "arm": name, "capacity_sessions": max(ok) if ok else 0, "budget_ms": K * HOP_MS}
                print(json.dumps(cap)); rows.append(cap)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_stream_chunks%s.json" % ("_profile" if args.profile else "")), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
