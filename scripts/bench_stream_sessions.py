#!/usr/bin/env python
"""Session capacity of one streaming handle (fsn_stream_step_slots, DESIGN.md §3.9): BASELINE config #4's model serving B slots of
independent real-time sessions with churn.

Per slot count: sessions of 3 to 30 s (seeded), a new session STARTs in every free slot on the next tick, each live session holds
about 1 % of its ticks (a frame that has not arrived), and a session ends with look_ahead zero frames.  Every tick is synchronised,
as a real-time caller must.  Reported per slot count: host latency per tick (enqueue + synchronize) p50 / p99, device time per tick
(CUDA events around the call), launches per tick, the FLOP rate the stepping sessions need, and, over all slot counts, the largest one
whose p99 stays under the 16 ms hop.

    python scripts/bench_stream_sessions.py [--slots 1,16,64,65,256,1024] [--ticks 300] [--warmup 50] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]
from fsnplus_b200 import inference as inf  # noqa: E402
from fsnplus_b200.model import Model  # noqa: E402
from fsnplus_b200.streaming import HOLD, START, STEP, StreamingFullSubNet  # noqa: E402
from fsnplus_b200.synth import synth_clips  # noqa: E402

HOP_MS = 16.0
GFLOP_PER_SESSION_FRAME = 0.96          # BASELINE.md §2: config #4's model, one frame of one clip
CFG = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM",
           fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=512,
           sb_model_hidden_size=384, weight_init=False, norm_type="cumulative_laplace_norm", num_groups_in_drop_band=2)


class Churn:
    """The caller's slot bookkeeping: per slot the clip, position and remaining flush frames of its session."""

    def __init__(self, B, nclips, T, la, seed):
        self.B, self.T, self.la = B, T, la
        self.rng = np.random.default_rng(seed)
        self.clip = np.zeros(B, np.int64)
        self.pos = np.zeros(B, np.int64)
        self.left = np.zeros(B, np.int64)           # frames of the session still to feed, flush included; 0 = free slot
        self.nclips = nclips
        self.first = True

    def _length(self, n):
        return self.rng.integers(int(3 * 1000 / HOP_MS), int(30 * 1000 / HOP_MS) + 1, size=n)

    def tick(self):
        """flags [B] int32, clip / frame index of every slot (frame index T = a zero flush frame), live-frame mask."""
        flags = np.full(self.B, STEP, np.int32)
        free = np.nonzero(self.left == 0)[0]
        if len(free):
            flags[free] = START
            n = self._length(len(free))
            if self.first:                          # the first sessions joined at random earlier times: stagger their ends
                n = self.rng.integers(1, n + 1)
                self.first = False
            self.clip[free] = self.rng.integers(0, self.nclips, size=len(free))
            self.pos[free] = 0
            self.left[free] = n + self.la
        hold = (self.rng.random(self.B) < 0.01) & (flags == STEP)
        flags[hold] = HOLD
        step = flags != HOLD
        frame = np.where(self.left - self.la > 0, self.pos, self.T)      # past the clip: a flush zero frame
        self.pos[step] += 1
        self.left[step] -= 1
        return flags, frame


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:                                               # noqa: BLE001
        return f"unavailable ({e})"


def run(model, pool, B, ticks, warmup, seed, la):
    dev = pool.device
    nclips, T1, F = pool.shape                                           # pool [nclips, T + 1, F]: row T of every clip is zero
    churn = Churn(B, nclips, T1 - 1, la, seed)
    st = StreamingFullSubNet(model, batch_size=B, device=dev)
    lat, dev_ms, starts, stepping = [], [], 0, 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for t in range(warmup + ticks):
        flags, frame = churn.tick()
        idx = torch.from_numpy(churn.clip * T1 + frame).to(dev)
        x = pool.view(-1, F).index_select(0, idx)                        # [B, F]; held rows hold a real frame the step never reads
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        st.step_slots(x, flags)
        e1.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if t >= warmup:
            lat.append((t1 - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            starts += int((flags == START).any())
            stepping += int((flags != HOLD).sum())
    st.close()
    lat, dev_ms = np.array(lat), np.array(dev_ms)
    pct = lambda a, q: float(np.percentile(a, q))
    # launches per tick, counted from the host path of fsn_stream_step_slots: one H2D copy of the slot counts, the reset kernel on
    # ticks with a START, then the six kernels of a step (+ the grid-barrier memset of the weight-stationary full-band step, B <= 64)
    kernels = 6 + starts / ticks
    flop = GFLOP_PER_SESSION_FRAME * 1e9 * stepping / ticks
    return {"slots": B, "ticks": ticks, "host_ms": {"p50": pct(lat, 50), "p99": pct(lat, 99), "mean": float(lat.mean()), "max": float(lat.max())},
            "device_ms": {"p50": pct(dev_ms, 50), "p99": pct(dev_ms, 99), "mean": float(dev_ms.mean())},
            "kernels_per_tick": kernels, "h2d_copies_per_tick": 1, "memsets_per_tick": 1 if B <= 64 else 0,
            "start_tick_fraction": starts / ticks, "stepping_sessions_per_tick": stepping / ticks,
            "required_tflop_per_tick": flop / 1e12, "achieved_tflops": flop / (float(dev_ms.mean()) * 1e-3) / 1e12,
            "meets_hop_p99": pct(lat, 99) < HOP_MS}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", default="1,16,64,65,256,1024")
    ap.add_argument("--ticks", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="also write the results as DIR/stream_sessions.json")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = Model(**CFG).to(dev).eval()
    clips = synth_clips(8, 480000, 16000, seed=77).to(dev)              # 8 x 30 s: sessions read their frames from this pool
    mag = inf.stft(clips).abs().transpose(1, 2)                          # [8, T, F]
    pool = torch.cat([mag, torch.zeros_like(mag[:, :1])], dim=1).contiguous()
    info = gpu_info()
    rows = []
    for B in [int(s) for s in args.slots.split(",")]:
        r = run(model, pool, B, args.ticks, args.warmup, args.seed + B, CFG["look_ahead"])
        r["gpu"] = info
        print(json.dumps(r), flush=True)
        rows.append(r)
    ok = [r["slots"] for r in rows if r["meets_hop_p99"]]
    summary = {"gpu": info, "hop_ms": HOP_MS, "largest_slots_p99_under_hop": max(ok) if ok else 0,
               "slot_counts": [r["slots"] for r in rows]}
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stream_sessions.json"), "w") as f:
            json.dump({"rows": rows, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
