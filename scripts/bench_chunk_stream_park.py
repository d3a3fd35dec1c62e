#!/usr/bin/env python
"""Park and resume overlapped-chunk sessions (fsn_chunk_stream_save_slots / _load_slots, ChunkStream; DESIGN.md §3.17) on the default
FullSubNet+ configuration.

Copy: a handle of --slots sessions (default 2048) per chunk length C, every session live.  For n in --n sessions, the device time
(CUDA events) of one save and of one load of n slots (a random choice, loaded into a permutation of them), p50 / p99 over --reps calls
after a warm-up.  Each timed call is queued behind a short spin kernel, so the events time the device work and not the host's enqueue.
The bytes it moves per session, (C + P + H) 4 read plus as many written, give an effective rate.

Step: the staggered workload of bench_chunk_stream.py (--sessions live sessions, --push samples per call) with m in --park sessions
saved and loaded back into their slots in every call, before the step (a park and a resume per call); device time per call (the
copies and the step) p50 / p99 over --periods chunk periods.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_chunk_stream_park.py [--chunk-s 1,2] [--slots 2048] [--n 1,64,1024,2048] [--sessions 1024] [--park 0,8,64]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200"), os.path.join(ROOT, "scripts")]
from bench_chunk_stream import CFG, SR, Sessions, gpu_info  # noqa: E402
from fsnplus_b200.model import FullSubNet_Plus  # noqa: E402

P = 256
SPIN = 200000                                              # cycles of the spin kernel ahead of each timed copy


def copy_times(model, C, slots, ns, reps, warm):
    s = Sessions(model, slots, C, 320, "staggered")
    for _ in range(2 * s.per):                             # every session has completed chunks
        s.call()
    cs = s.cs
    rng = np.random.default_rng(C)
    out = []
    for n in ns:
        src = rng.choice(slots, n, replace=False).tolist()
        dst = rng.permutation(src).tolist()
        st = cs.save_slots(src)
        res = {"C_s": C / SR, "slots": slots, "n": n, "payload_bytes_per_session": int(st.payload.shape[1])}
        for what in ("save", "load"):
            fn = (lambda: cs.save_slots(src)) if what == "save" else (lambda: cs.load_slots(dst, st))
            for _ in range(warm):
                fn()
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
            for a, b in ev:
                torch.cuda._sleep(SPIN)
                a.record()
                fn()
                b.record()
            torch.cuda.synchronize()
            t = np.array([a.elapsed_time(b) for a, b in ev])
            moved = 2 * n * (C + P + C // 2) * 4
            res[f"{what}_p50_ms"] = round(float(np.median(t)), 4)
            res[f"{what}_p99_ms"] = round(float(np.percentile(t, 99)), 4)
            res[f"{what}_GB_per_s_at_p50"] = round(moved / (float(np.median(t)) * 1e-3) / 1e9, 1)
        out.append(res)
        print(json.dumps(res), flush=True)
    cs.close()
    return out


def step_times(model, C, B, push, parks, periods):
    out = []
    for m in parks:
        s = Sessions(model, B, C, push, "staggered")
        per = s.per
        for _ in range(2 * per):
            s.call()
        rng = np.random.default_rng(m)
        n = per * periods
        picks = [rng.choice(B, m, replace=False).tolist() for _ in range(n)] if m else [None] * n
        if m:                                              # warm the park path too
            s.cs.load_slots(picks[0], s.cs.save_slots(picks[0]))
        torch.cuda.synchronize()
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
        for (a, b), pk in zip(ev, picks):
            a.record()
            if pk:
                s.cs.load_slots(pk, s.cs.save_slots(pk))
            s.call()
            b.record()
        torch.cuda.synchronize()
        t = np.array([a.elapsed_time(b) for a, b in ev])
        s.cs.close()
        r = {"C_s": C / SR, "sessions": B, "parked_per_call": m, "calls": n, "p50_ms": round(float(np.median(t)), 3),
             "p99_ms": round(float(np.percentile(t, 99)), 3), "max_ms": round(float(t.max()), 3)}
        out.append(r)
        print(json.dumps(r), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk-s", default="1,2")
    ap.add_argument("--slots", type=int, default=2048)
    ap.add_argument("--n", default="1,64,1024,2048")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warm", type=int, default=20)
    ap.add_argument("--sessions", type=int, default=1024)
    ap.add_argument("--park", default="0,8,64")
    ap.add_argument("--push", type=int, default=320)
    ap.add_argument("--periods", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_chunk_stream_park.py needs a CUDA GPU (H100)")
    torch.manual_seed(0)
    model = FullSubNet_Plus(**CFG).to("cuda:0").eval()
    info = {"gpu": gpu_info(), "config": "default FullSubNet+ (F = 257, TSSE, sub-band LSTM 384)", "push_samples": a.push}
    print(json.dumps(info), flush=True)
    results = [info]
    Cs = [int(float(c) * SR) for c in a.chunk_s.split(",")]
    ns = [int(v) for v in a.n.split(",")]
    parks = [int(v) for v in a.park.split(",")]
    for C in Cs:
        results += copy_times(model, C, a.slots, ns, a.reps, a.warm)
    for C in Cs:
        results += step_times(model, C, a.sessions, a.push, parks, a.periods)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "chunk_stream_park.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
