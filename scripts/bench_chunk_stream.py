#!/usr/bin/env python
"""Overlapped-chunk sessions (fsn_chunk_stream_step, ChunkStream; DESIGN.md §3.16) on the default FullSubNet+ configuration.

Every slot serves one live session and pushes --push samples (default 320 = 20 ms at 16 kHz) per call.  Per chunk length C and session
count B, two start patterns: "staggered" (slot b's session is b H / B samples ahead of slot 0's, so about B / (H / push) chunks complete
in every call) and "aligned" (every session starts together, so every chunk of every session lands in one call every H / push calls:
the burst case).  After a warm-up of two chunk periods (H / push calls each) the timed window is --periods chunk periods.  Reported per
(C, B, pattern): device time per call (CUDA events, p50 and p99), chunks per call (mean and max), and the compute per second of audio
(the window's summed device time over the audio each session pushed in it).  Per C and pattern, the capacity: the largest B whose
compute per second of audio stays under one second.  --profile traces --profile-calls calls of one (C, B, pattern) under torch.profiler,
in a run of its own, and reports each kernel's device time per call.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_chunk_stream.py [--chunk-s 1,2] [--sessions 64,256,1024,2048] [--push 320] [--periods 2] [--out DIR]
    python scripts/bench_chunk_stream.py --profile [--chunk-s 1] [--sessions 1024] [--pattern staggered]
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
from fsnplus_b200.model import FullSubNet_Plus  # noqa: E402
from fsnplus_b200.streaming import START, STEP, ChunkStream  # noqa: E402

SR = 16000
CFG = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM",
           fb_output_activate_function="ReLU", sb_output_activate_function=False, channel_attention_model="TSSE",
           fb_model_hidden_size=512, sb_model_hidden_size=384, weight_init=False, norm_type="offline_laplace_norm",
           num_groups_in_drop_band=2, kersize=[3, 5, 10], subband_num=1)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else torch.cuda.get_device_name(0)


class Sessions:
    """B live sessions on one handle, fed from a seeded noise bank: a prefill call STARTs each with its offset (staggered: b H / B
    rounded down to whole pushes, aligned: 0), then every call STEPs push samples on every slot."""

    def __init__(self, model, B, C, push, pattern, seed=0):
        self.cs = ChunkStream(model, B, C, "cuda:0")
        self.B, self.C, self.push = B, C, push
        H = C // 2
        self.per = H // push                                # calls per chunk period
        g = torch.Generator(device="cuda:0").manual_seed(seed)
        self.bank = torch.randn((self.per, B, push), device="cuda:0", generator=g) * 0.05
        off = [(b * self.per // B) * push if pattern == "staggered" else 0 for b in range(B)]
        pre = torch.randn((B, max(max(off), 1)), device="cuda:0", generator=g) * 0.05
        self.cs.step(pre, off, [START] * B)
        self.i = 0
        self.counts, self.flags = [push] * B, [STEP] * B

    def call(self):
        _, nout = self.cs.step(self.bank[self.i % self.per], self.counts, self.flags)
        self.i += 1
        return nout


def measure(model, B, C, push, pattern, periods):
    s = Sessions(model, B, C, push, pattern)
    per = s.per
    for _ in range(2 * per):                                # every session has completed chunks, every batch shape has run
        s.call()
    torch.cuda.synchronize()
    n = per * periods
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
    chunks = []
    for a, b in ev:
        a.record()
        nout = s.call()
        b.record()
        chunks.append(int(nout.sum()) // (C // 2))
    torch.cuda.synchronize()
    t = np.array([a.elapsed_time(b) for a, b in ev])
    s.cs.close()
    audio_s = n * push / SR
    return {"C_s": C / SR, "sessions": B, "pattern": pattern, "calls": n, "p50_ms": round(float(np.median(t)), 3),
            "p99_ms": round(float(np.percentile(t, 99)), 3), "max_ms": round(float(t.max()), 3),
            "chunks_per_call_mean": round(float(np.mean(chunks)), 2), "chunks_per_call_max": int(max(chunks)),
            "compute_s_per_audio_s": round(float(t.sum()) / 1e3 / audio_s, 4)}


def profile(model, B, C, push, pattern, calls):
    from torch.profiler import ProfilerActivity, profile as tprofile
    s = Sessions(model, B, C, push, pattern)
    for _ in range(2 * s.per):
        s.call()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            s.call()
        torch.cuda.synchronize()
    s.cs.close()
    per = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per.setdefault(e.name, [0.0, 0])
            per[e.name][0] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            per[e.name][1] += 1
    total = sum(v[0] for v in per.values())
    rows = sorted(per.items(), key=lambda kv: -kv[1][0])
    return {"profile": {"C_s": C / SR, "sessions": B, "pattern": pattern, "calls": calls, "device_ms_per_call": round(total / 1e3 / calls, 3),
                        "kernels": [{"name": k[:90], "us_per_call": round(v[0] / calls, 1), "launches_per_call": round(v[1] / calls, 2),
                                     "share": round(v[0] / total, 4)} for k, v in rows[:25]]}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk-s", default="1,2")
    ap.add_argument("--sessions", default="64,256,1024,2048")
    ap.add_argument("--pattern", default="staggered,aligned")
    ap.add_argument("--push", type=int, default=320)
    ap.add_argument("--periods", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--profile-calls", type=int, default=25)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_chunk_stream.py needs a CUDA GPU (H100)")
    torch.manual_seed(0)
    model = FullSubNet_Plus(**CFG).to("cuda:0").eval()
    info = {"gpu": gpu_info(), "config": "default FullSubNet+ (F = 257, TSSE, sub-band LSTM 384)", "push_samples": a.push}
    print(json.dumps(info), flush=True)
    results = [info]
    Cs = [int(float(c) * SR) for c in a.chunk_s.split(",")]
    Bs = [int(b) for b in a.sessions.split(",")]
    pats = a.pattern.split(",")
    if a.profile:
        r = profile(model, Bs[0], Cs[0], a.push, pats[0], a.profile_calls)
        print(json.dumps(r), flush=True)
        results.append(r)
    else:
        cap = {}
        for C in Cs:
            for pat in pats:
                for B in Bs:
                    r = measure(model, B, C, a.push, pat, a.periods)
                    print(json.dumps(r), flush=True)
                    results.append(r)
                    if r["compute_s_per_audio_s"] < 1.0:
                        cap[f"C={C / SR:g}s {pat}"] = max(cap.get(f"C={C / SR:g}s {pat}", 0), B)
        r = {"capacity_sessions": cap, "note": "largest tested B whose compute per second of audio is under one second"}
        print(json.dumps(r), flush=True)
        results.append(r)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        name = "chunk_stream_profile.json" if a.profile else "chunk_stream.json"
        with open(os.path.join(a.out, name), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
