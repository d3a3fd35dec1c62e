#!/usr/bin/env python
"""Cost of parking and restoring streaming sessions (fsn_stream_save_slots / fsn_stream_load_slots, DESIGN.md §3.11) on BASELINE
config #4's model.

1. Save and load cost: per mode (mask, audio) and session count n (1, 16, 128, 1024) the device time of one save call and one load call
   (CUDA events, median of --rounds rounds, save and load alternating) and the effective bandwidth 2 n payload_bytes / time (every
   byte is read once and written once), against the H100 SXM data-sheet 3.35 TB/s.
2. Tick cost with parking: 1280 sessions under the churn of bench_stream_sessions.py; every tick also saves k live sessions in one call
   and loads them back in one call (a park plus a restore of k sessions), k = 0 (the baseline), 8, 64.  The arms alternate, --reps
   times each.  Reported: host latency per tick (enqueue + synchronize) p50 / p99 and whether p99 stays under the 16 ms hop.

    python scripts/bench_stream_park.py [--rounds 20] [--ticks 200] [--warmup 30] [--reps 2] [--out DIR]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200"), os.path.join(ROOT, "scripts")]
from bench_stream_sessions import CFG, HOP_MS, Churn, gpu_info  # noqa: E402
from fsnplus_b200 import inference as inf  # noqa: E402
from fsnplus_b200.model import Model  # noqa: E402
from fsnplus_b200.streaming import HOLD, START, StreamingFullSubNet  # noqa: E402
from fsnplus_b200.synth import synth_clips  # noqa: E402

DATASHEET_TBS = 3.35


def copy_cost(model, mode, counts, rounds, dev):
    """Median device ms of one save and one load of n sessions, per n; the handle has max(counts) slots, all started."""
    B = max(counts)
    st = StreamingFullSubNet(model, batch_size=B, device=dev)
    if mode == "audio":
        st.step_audio(torch.zeros((B, st.hop), device=dev), [START] * B)
    else:
        st.step_slots(torch.zeros((B, st.F), device=dev), [START] * B)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    rows = []
    for n in counts:
        slots = list(range(n))
        state = st.save_slots(slots)
        stride = state.payload.shape[1]
        ms_save, ms_load = [], []
        for r in range(rounds + 2):
            e[0].record()
            state = st.save_slots(slots)
            e[1].record()
            st.load_slots(slots, state)
            e[2].record()
            torch.cuda.synchronize()
            if r >= 2:
                ms_save.append(e[0].elapsed_time(e[1]))
                ms_load.append(e[1].elapsed_time(e[2]))
        for op, ms in (("save", ms_save), ("load", ms_load)):
            t = float(np.median(ms))
            gbs = 2 * n * stride / (t * 1e-3) / 1e9
            rows.append({"part": "copy", "mode": mode, "op": op, "sessions": n, "payload_bytes": stride, "us_per_call": t * 1e3,
                         "effective_GBps": gbs, "fraction_of_datasheet": gbs / (DATASHEET_TBS * 1e3), "rounds": rounds})
    st.close()
    return rows


def park_ticks(model, pool, B, k, ticks, warmup, seed, la):
    """bench_stream_sessions' churn at B slots; each tick also saves k random live sessions and loads them back (k = 0: baseline)."""
    dev = pool.device
    nclips, T1, W = pool.shape
    churn = Churn(B, nclips, T1 - 1, la, seed)
    rng = np.random.default_rng(seed + 1)
    st = StreamingFullSubNet(model, batch_size=B, device=dev)
    lat = []
    for t in range(warmup + ticks):
        flags, frame = churn.tick()
        idx = torch.from_numpy(churn.clip * T1 + frame).to(dev)
        x = pool.view(-1, W).index_select(0, idx)
        live = np.nonzero((flags != HOLD) & (flags != START))[0]
        park = sorted(rng.choice(live, size=min(k, len(live)), replace=False).tolist()) if k and t > 0 else []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if park:
            st.load_slots(park, st.save_slots(park))
        st.step_slots(x, flags)
        torch.cuda.synchronize()
        if t >= warmup:
            lat.append((time.perf_counter() - t0) * 1e3)
    st.close()
    lat = np.array(lat)
    return {"part": "tick", "slots": B, "parked_per_tick": k, "ticks": ticks, "host_ms": {"p50": float(np.percentile(lat, 50)),
            "p99": float(np.percentile(lat, 99)), "mean": float(lat.mean()), "max": float(lat.max())},
            "meets_hop_p99": float(np.percentile(lat, 99)) < HOP_MS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--counts", default="1,16,128,1024")
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--slots", type=int, default=1280)
    ap.add_argument("--parks", default="0,8,64")
    ap.add_argument("--ticks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="also write the results as DIR/stream_park.json")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = Model(**CFG).to(dev).eval()
    info = gpu_info()
    rows = []
    counts = [int(c) for c in args.counts.split(",")]
    for mode in ("mask", "audio"):
        for r in copy_cost(model, mode, counts, args.rounds, dev):
            r["gpu"] = info
            print(json.dumps(r), flush=True)
            rows.append(r)
    clips = synth_clips(8, 480000, 16000, seed=77).to(dev)
    mag = inf.stft(clips).abs().transpose(1, 2)
    pool = torch.cat([mag, torch.zeros_like(mag[:, :1])], dim=1).contiguous()
    for rep in range(args.reps):
        for k in [int(p) for p in args.parks.split(",")]:
            r = park_ticks(model, pool, args.slots, k, args.ticks, args.warmup, args.seed + args.slots, CFG["look_ahead"])
            r["gpu"], r["rep"] = info, rep
            print(json.dumps(r), flush=True)
            rows.append(r)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stream_park.json"), "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
