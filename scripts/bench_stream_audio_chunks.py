#!/usr/bin/env python
"""Audio chunk calls (fsn_stream_step_audio_chunk, DESIGN.md §3.14) on BASELINE config #4's model, against the mask chunk call and
against per-hop audio calls.

Per session count B and chunk size K, three arms alternate (--reps rounds of --iters calls each) on handles of the same model: one
audio chunk call of K hops per slot, one mask chunk call of K frames (fsn_stream_step_chunk), and K per-hop audio calls
(fsn_stream_step_audio_slots).  Steady state: every slot steps every call, sessions started before the timed window.  With --churn,
sessions START and FLUSH inside the audio chunk calls with seeded partial hop counts (the other arms are not run); the line also
reports the launches per call and the number of layer-wise groups (distinct per-slot frame counts).  Reported: device time per call (CUDA
events, median and p99), session-hops per second, and per K and arm the largest B whose p99 stays under K x 16 ms.  --profile traces
the audio chunk arm at one (B, K) under torch.profiler and reports the device time per call of every kernel.

    python scripts/bench_stream_audio_chunks.py [--sessions 512,1024,1280,2048] [--K 8,16,32,64] [--iters 10] [--reps 2] [--out DIR]
    python scripts/bench_stream_audio_chunks.py --churn [--sessions 1280] [--K 32]
    python scripts/bench_stream_audio_chunks.py --profile [--sessions 1280] [--K 32]
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
from fsnplus_b200.streaming import FLUSH, START, STEP, StreamingFullSubNet  # noqa: E402

HOP_MS = 16.0
CFG = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM",
           fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=512,
           sb_model_hidden_size=384, weight_init=False, norm_type="cumulative_laplace_norm", num_groups_in_drop_band=2)
HOP = 256


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, iters):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for i, (a, b) in enumerate(ev):
        a.record()
        fn(i)
        b.record()
        b.synchronize()
    return [a.elapsed_time(b) for a, b in ev]


def stats(t, B, K):
    t = np.array(t)
    med, p99 = float(np.median(t)), float(np.percentile(t, 99))
    return {"median_ms": round(med, 3), "p99_ms": round(p99, 3), "session_hops_per_s": round(B * K / med * 1e3), "real_time": p99 < K * HOP_MS}


class Churn:
    """Seeded sessions on every slot of an audio handle: each lasts 20-200 hops, STARTs with a partial hop count, STEPs a random
    1..K hops (K most of the time), FLUSHes its last hops and then FLUSHes with 0 hops until its output is complete; the slot
    restarts in the next call."""

    def __init__(self, B, la, seed):
        self.B, self.la, self.rng = B, la, np.random.default_rng(seed)
        self.left = np.zeros(B, int)          # hops still to send
        self.tail = np.zeros(B, int)          # FLUSH ticks still to run after the input ended

    def plan(self, K):
        """(flags, hops, model frames per slot) of the next call."""
        flags, hops, kf = np.zeros(self.B, np.int32), np.zeros(self.B, np.int32), np.zeros(self.B, int)
        for b in range(self.B):
            r = self.rng
            if self.left[b] == 0 and self.tail[b] == 0:              # (re)start
                self.left[b] = int(r.integers(20, 200))
                n = int(r.integers(1, min(K, self.left[b] - 1) + 1))
                flags[b], hops[b], kf[b] = START, n, n - 1
                self.left[b] -= n
                continue
            if self.left[b] > 0:
                n = min(K, self.left[b]) if r.random() < 0.8 else int(r.integers(1, min(K, self.left[b]) + 1))
                if n == self.left[b] and n < K:
                    flags[b], hops[b], kf[b] = FLUSH, n, n + min(K - n, self.la + 2)
                    self.tail[b] = max(0, self.la + 2 - (K - n))
                else:                                                   # a STEP that sends the last hops leaves la + 2 FLUSH ticks
                    flags[b], hops[b], kf[b] = STEP, n, n
                    self.tail[b] = self.la + 2 if n == self.left[b] else 0
                self.left[b] -= n
                continue
            flags[b], hops[b], kf[b] = FLUSH, 0, min(K, self.tail[b])
            self.tail[b] = max(0, self.tail[b] - K)
        return flags, hops, kf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sessions", default="512,1024,1280,2048")
    ap.add_argument("--K", default="8,16,32,64")
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--churn", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a CUDA GPU"
    dev = "cuda:0"
    torch.manual_seed(0)
    model = Model(**CFG).to(dev).eval()
    la = model.look_ahead
    Bs, Ks = [int(v) for v in args.sessions.split(",")], [int(v) for v in args.K.split(",")]
    info = gpu_info()
    rows = []
    rng = np.random.default_rng(1)
    for B in Bs:
        for K in Ks:
            audio = StreamingFullSubNet(model, B, dev)
            x = torch.from_numpy(rng.standard_normal((B, K * HOP)).astype(np.float32) * 0.05).to(dev)
            if args.churn:
                ch = Churn(B, la, seed=B * 100 + K)
                plans = [ch.plan(K) for _ in range(5 + args.reps * args.iters)]       # warm-up, timed, profiled
                groups = [len(set(kf[kf > 0].tolist())) for _, _, kf in plans][4:-1]
                plans = [p[:2] for p in plans]
                for p in plans[:4]:
                    audio.step_audio_chunk(x, *p)
                torch.cuda.synchronize()
                t = timed(lambda i: audio.step_audio_chunk(x, *plans[4 + i]), args.reps * args.iters)
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    audio.step_audio_chunk(x, *plans[-1])
                    torch.cuda.synchronize()
                launches = sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA" and "Memcpy" not in e.key
                               and "Memset" not in e.key)
                line = {"gpu": info, "B": B, "K": K, "churn": True, "audio_chunk": stats(t, B, K), "launches_last_call": launches,
                        "layerwise_groups_per_call_mean": round(float(np.mean(groups)), 2), "layerwise_groups_per_call_max": max(groups)}
                print(json.dumps(line)); rows.append(line)
                audio.close()
                continue
            audio.step_audio_chunk(x, [START] * B, [K] * B)
            if args.profile:
                audio.step_audio_chunk(x, [STEP] * B, [K] * B)
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    timed(lambda i: audio.step_audio_chunk(x, [STEP] * B, [K] * B), args.iters)
                per = {}
                for e in prof.key_averages():
                    t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                    if t:
                        per[e.key] = per.get(e.key, 0.0) + t / 1e3 / args.iters
                line = {"gpu": info, "B": B, "K": K, "ms_per_call_total": round(sum(per.values()), 3),
                        "kernels_ms_per_call": {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}}
                print(json.dumps(line)); rows.append(line)
                audio.close()
                continue
            mask_h, hop_h = StreamingFullSubNet(model, B, dev), StreamingFullSubNet(model, B, dev)
            mag = torch.from_numpy(np.abs(rng.standard_normal((B, 257, K))).astype(np.float32) * 0.1).to(dev)
            mask_h.step_chunk(mag, [START] * B)
            xs = [x[:, k * HOP:(k + 1) * HOP].contiguous() for k in range(K)]
            for k in range(4):
                hop_h.step_audio(xs[k % K], [START if k == 0 else STEP] * B)
            flags, hops = [STEP] * B, [K] * B
            arms = {"audio_chunk": lambda i: audio.step_audio_chunk(x, flags, hops),
                    "mask_chunk": lambda i: mask_h.step_chunk(mag, flags),
                    "per_hop_audio": lambda i: [hop_h.step_audio(xs[k], flags) for k in range(K)]}
            for fn in arms.values():                                    # warm-up of this shape
                timed(fn, 1)
            t = {name: [] for name in arms}
            for _ in range(args.reps):
                for name, fn in arms.items():
                    t[name] += timed(fn, args.iters)
            line = {"gpu": info, "B": B, "K": K}
            for name in arms:
                line[name] = stats(t[name], B, K)
            line["audio_vs_mask_chunk"] = round(line["audio_chunk"]["median_ms"] / line["mask_chunk"]["median_ms"], 4)
            line["audio_chunk_vs_per_hop_rate"] = round(line["audio_chunk"]["session_hops_per_s"] /
                                                        line["per_hop_audio"]["session_hops_per_s"], 2)
            print(json.dumps(line)); rows.append(line)
            audio.close(); mask_h.close(); hop_h.close()
    if not (args.profile or args.churn):
        for K in Ks:
            for name in ("audio_chunk", "mask_chunk", "per_hop_audio"):
                ok = [r["B"] for r in rows if r.get("K") == K and name in r and r[name]["real_time"]]
                cap = {"gpu": info, "K": K, "arm": name, "capacity_sessions": max(ok) if ok else 0, "budget_ms": K * HOP_MS}
                print(json.dumps(cap)); rows.append(cap)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        tag = "_profile" if args.profile else "_churn" if args.churn else ""
        with open(os.path.join(args.out, f"bench_stream_audio_chunks{tag}.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
