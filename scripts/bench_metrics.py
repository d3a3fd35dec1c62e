"""Cost of the device metrics (fsnplus_b200.metrics, DESIGN.md §3.20 and §3.21) on three workloads at 16 kHz: a DNS-test-set-shaped
batch (150 clips x 10 s), 64 clips x 3 s, and one 60-minute clip.

  * device time per call (SI-SDR, STOI, SDR) with CUDA events: the median and min over --iters calls after a warm-up call;
  * SDR's achieved fp64 rate: the work counted from the shapes (2 x 512 L_b multiply-adds of correlations and 512 (L_b + 511) of
    projection per clip, 2 FLOP each) over the median call time;
  * per-kernel device time from torch.profiler, in a separate pass;
  * baseline: the float64 numpy / scipy restatements (tests/metrics_ref.py, not pystoi; tests/sdr_ref.py, not mir_eval) on the
    host's cores with joblib, one clip per job as the reference's scorer runs, timed once.
Prints one JSON line per workload with the GPU name, power limit and max SM clock read in the same run; with --out, also writes
them to DIR/bench_metrics.json.

    python scripts/bench_metrics.py [--iters 10] [--out DIR] [--no-baseline]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200"), os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")]
from bench_stream_audio_chunks import gpu_info, timed  # noqa: E402
from fsnplus_b200 import metrics  # noqa: E402

DEV = "cuda:0"
SR = 16000
WORKLOADS = {"dns_150x10s": (150, 10.0), "64x3s": (64, 3.0), "1x60min": (1, 3600.0)}


def clips(B, seconds, seed):
    """Speech-like references (tests/audio_ref.speech) with white noise at 5 dB SNR as the estimates."""
    import audio_ref as A
    n = int(seconds * SR)
    rng = np.random.default_rng(seed)
    ref = np.stack([A.speech(n, seed + b) for b in range(B)])
    est = (ref + rng.standard_normal(ref.shape).astype(np.float32) * ref.std(axis=1, keepdims=True) * 10 ** (-5 / 20)).astype(np.float32)
    return ref, est


def baseline(ref, est):
    import metrics_ref as R
    from joblib import Parallel, delayed
    Parallel(n_jobs=-1)(delayed(R.si_sdr)(r, e) for r, e in zip(ref[:1], est[:1]))   # start the workers outside the timed window
    t = time.perf_counter()
    Parallel(n_jobs=-1)(delayed(R.si_sdr)(r, e) for r, e in zip(ref, est))
    t_sdr = time.perf_counter() - t
    t = time.perf_counter()
    Parallel(n_jobs=-1)(delayed(R.stoi)(r, e, SR) for r, e in zip(ref, est))
    return t_sdr * 1e3, (time.perf_counter() - t) * 1e3


def baseline_sdr(ref, est):
    import sdr_ref as S
    from joblib import Parallel, delayed
    Parallel(n_jobs=-1)(delayed(S.sdr)(r, e) for r, e in zip(ref[:1, :1000], est[:1, :1000]))
    t = time.perf_counter()
    Parallel(n_jobs=-1)(delayed(S.sdr)(r, e) for r, e in zip(ref, est))
    return (time.perf_counter() - t) * 1e3


def sdr_flop(B, n):
    return 2 * B * (2 * 512 * n + 512 * (n + 511))


def kernel_times(r, e):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            metrics.si_sdr(r, e)
            metrics.stoi(r, e, sr=SR)
            metrics.sdr(r, e)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if "kernel" in ev.key and ("sdr" in ev.key or "stoi" in ev.key):
            out[ev.key.split("(")[0].replace("void fsn::", "")] = round(ev.device_time_total / 3 / 1e3, 4)   # ms per call
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()
    gpu = gpu_info()
    rows = []
    for name, (B, seconds) in WORKLOADS.items():
        ref, est = clips(B, seconds, 1)
        r, e = torch.from_numpy(ref).to(DEV), torch.from_numpy(est).to(DEV)
        row = {"workload": name, "clips": B, "seconds_per_clip": seconds, "sr": SR, "gpu": gpu}
        for mname, fn in (("si_sdr", lambda i: metrics.si_sdr(r, e)), ("stoi", lambda i: metrics.stoi(r, e, sr=SR)),
                          ("sdr", lambda i: metrics.sdr(r, e))):
            fn(0)
            torch.cuda.synchronize()
            t = timed(fn, args.iters)
            row[f"{mname}_ms_median"] = float(np.median(t))
            row[f"{mname}_ms_min"] = float(np.min(t))
        row["sdr_tflops"] = sdr_flop(B, ref.shape[1]) / (row["sdr_ms_median"] * 1e-3) / 1e12
        row["kernels_ms_per_call"] = kernel_times(r, e)
        if not args.no_baseline:
            sdr_ms, stoi_ms = baseline(ref, est)
            row.update(baseline_numpy_si_sdr_ms=sdr_ms, baseline_numpy_stoi_ms=stoi_ms, baseline_cores=os.cpu_count())
            row["baseline_numpy_sdr_ms"] = baseline_sdr(ref, est)
        print(json.dumps(row), flush=True)
        rows.append(row)
        del r, e
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_metrics.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
