#!/usr/bin/env python
"""Session capacity of one streaming handle (fsn_stream_step_slots, DESIGN.md §3.9): BASELINE config #4's model serving B slots of
independent real-time sessions with churn.

Per slot count: sessions of 3 to 30 s (seeded), a new session STARTs in every free slot on the next tick, each live session holds
about 1 % of its ticks (a frame that has not arrived), and a session ends with look_ahead zero frames.  Every tick is synchronised,
as a real-time caller must.  Reported per slot count: host latency per tick (enqueue + synchronize) p50 / p99, device time per tick
(CUDA events around the call), launches per tick, the FLOP rate the stepping sessions need, and, over all slot counts, the largest one
whose p99 stays under the 16 ms hop.

--audio measures the audio call (fsn_stream_step_audio_slots, DESIGN.md §3.10) against the mask call on the same churn: a session of
at least 2 hops ends with look_ahead + 2 FLUSH ticks, and per slot count the mask arm and the audio arm alternate (--reps times each).
--profile instead runs the audio arm under torch.profiler and reports the device time per tick of every kernel.

    python scripts/bench_stream_sessions.py [--slots 1,16,64,65,256,1024] [--ticks 300] [--warmup 50] [--out DIR]
    python scripts/bench_stream_sessions.py --audio [--reps 2] [--profile] ...
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
from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP, StreamingFullSubNet  # noqa: E402
from fsnplus_b200.synth import synth_clips  # noqa: E402

HOP_MS = 16.0
HOP = 256                               # samples per hop at 16 kHz (n_fft 512)
GFLOP_PER_SESSION_FRAME = 0.96          # BASELINE.md §2: config #4's model, one frame of one clip
CFG = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM",
           fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=512,
           sb_model_hidden_size=384, weight_init=False, norm_type="cumulative_laplace_norm", num_groups_in_drop_band=2)


class Churn:
    """The caller's slot bookkeeping: per slot the clip, position and remaining flush frames of its session."""

    def __init__(self, B, nclips, T, la, seed, min_len=1):
        self.B, self.T, self.la, self.min_len = B, T, la, min_len      # la: flush ticks that end a session
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
                n = self.rng.integers(self.min_len, n + 1)
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


def run(model, pool, B, ticks, warmup, seed, la, audio=False, prof=None):
    """One arm at B slots.  pool [nclips, T + 1, W]: per clip T magnitude frames (W = F) or, with audio, T hops of samples (W = hop),
    row T zero.  The audio arm runs the same churn with look_ahead + 2 flush ticks (FLUSH) and sessions of at least 2 hops."""
    dev = pool.device
    nclips, T1, W = pool.shape
    churn = Churn(B, nclips, T1 - 1, la + 2 if audio else la, seed, min_len=2 if audio else 1)
    st = StreamingFullSubNet(model, batch_size=B, device=dev)
    lat, dev_ms, starts, stepping = [], [], 0, 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for t in range(warmup + ticks):
        pos = churn.pos.copy()
        flags, frame = churn.tick()
        idx = torch.from_numpy(churn.clip * T1 + frame).to(dev)
        x = pool.view(-1, W).index_select(0, idx)                        # [B, W]; held rows hold real data the step never reads
        if audio:
            flags[(flags == STEP) & (frame == T1 - 1)] = FLUSH
            model_step = (flags != HOLD) & (flags != START)              # a session's model row starts on its second tick
            model_start = bool((model_step & (pos == 1)).any())
        else:
            model_step, model_start = flags != HOLD, bool((flags == START).any())
        torch.cuda.synchronize()
        if prof is not None and t == warmup:
            prof.__enter__()
        t0 = time.perf_counter()
        e0.record()
        if audio:
            st.step_audio(x, flags)
        else:
            st.step_slots(x, flags)
        e1.record()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if t >= warmup:
            lat.append((t1 - t0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            starts += int(model_start)
            stepping += int(model_step.sum())
    if prof is not None:
        prof.__exit__(None, None, None)
    st.close()
    lat, dev_ms = np.array(lat), np.array(dev_ms)
    pct = lambda a, q: float(np.percentile(a, q))
    # launches per tick, counted from the host path of fsn_stream_step_slots: one H2D copy of the slot counts, the reset kernel on
    # ticks with a START, then the six kernels of a step (+ the grid-barrier memset of the weight-stationary full-band step, B <= 64).
    # The audio call adds its analysis and synthesis kernels; its reset runs on ticks where a session's model row starts
    kernels = (8 if audio else 6) + starts / ticks
    flop = GFLOP_PER_SESSION_FRAME * 1e9 * stepping / ticks
    return {"arm": "audio" if audio else "mask", "slots": B, "ticks": ticks, "host_ms": {"p50": pct(lat, 50), "p99": pct(lat, 99), "mean": float(lat.mean()), "max": float(lat.max())},
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
    ap.add_argument("--audio", action="store_true", help="alternate the mask arm and the audio arm per slot count")
    ap.add_argument("--reps", type=int, default=2, help="--audio: runs of each arm per slot count, alternating")
    ap.add_argument("--profile", action="store_true", help="device time per kernel of the audio arm (torch.profiler)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = Model(**CFG).to(dev).eval()
    clips = synth_clips(8, 480000, 16000, seed=77).to(dev)              # 8 x 30 s: sessions read their frames from this pool
    mag = inf.stft(clips).abs().transpose(1, 2)                          # [8, T, F]
    pool = torch.cat([mag, torch.zeros_like(mag[:, :1])], dim=1).contiguous()
    info = gpu_info()
    rows = []
    if args.audio or args.profile:                                       # the same clips as hops of samples: [8, T, hop] + a zero row
        T = clips.shape[1] // HOP
        hops = clips[:, :T * HOP].reshape(clips.shape[0], T, HOP)
        apool = torch.cat([hops, torch.zeros_like(hops[:, :1])], dim=1).contiguous()
    slots = [int(s) for s in args.slots.split(",")]
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        for B in slots:
            prof = profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA])
            run(model, apool, B, args.ticks, args.warmup, args.seed + B, CFG["look_ahead"], audio=True, prof=prof)
            kern = {}
            for e in prof.key_averages():
                if e.device_time_total > 0 and e.device_type == torch.autograd.DeviceType.CUDA:
                    kern[e.key] = round(e.device_time_total / args.ticks, 2)
            r = {"profile": "audio", "slots": B, "ticks": args.ticks, "gpu": info,
                 "device_us_per_tick": dict(sorted(kern.items(), key=lambda kv: -kv[1]))}
            print(json.dumps(r), flush=True)
            rows.append(r)
        summary = {"gpu": info, "profile": True}
    else:
        for B in slots:
            for rep in range(args.reps if args.audio else 1):
                for audio in ([False, True] if args.audio else [False]):
                    r = run(model, apool if audio else pool, B, args.ticks, args.warmup, args.seed + B, CFG["look_ahead"], audio=audio)
                    r["gpu"] = info
                    r["rep"] = rep
                    print(json.dumps(r), flush=True)
                    rows.append(r)
        summary = {"gpu": info, "hop_ms": HOP_MS, "slot_counts": slots}
        for arm in (["mask", "audio"] if args.audio else ["mask"]):
            ok = [B for B in slots if all(r["meets_hop_p99"] for r in rows if r["slots"] == B and r["arm"] == arm)]
            summary["largest_slots_p99_under_hop" + ("" if arm == "mask" else "_audio")] = max(ok) if ok else 0
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "stream_sessions.json"), "w") as f:
            json.dump({"rows": rows, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
