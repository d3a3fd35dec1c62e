"""The sub-band LSTM's input-projection GEMM (Gin = X W_ih^T, fp16 in / fp32 accumulate / fp16 out) alone, 128 x 128 tiles against
128 x 256 tiles on CTA pairs, at the shapes the layer-wise path runs it with.

    python scripts/bench_gin_gemm.py [--iters 20] [--rounds 3]            # the GEMM alone, CUDA events
    python scripts/bench_gin_gemm.py --profile [--batch 64]                 # through a model forward, torch.profiler

Prints one JSON line with the card's name and power limit (read in the same run).  GEMM alone: per shape and N tile, alternated
round by round on the same seeded operands, the ms per call (CUDA events over `iters` back-to-back calls), TFLOP/s, the HBM
bytes the GEMM must move (A and B read once, C written once) per second, and the bytes the kernel's tiles pull from L2 into
shared memory per second, counted from the tile geometry: per 128-row A tile and k-block 16 KB of A, plus 16 KB of B per 128
columns of the N tile, fetched once per tile (128 x 128) or once per CTA pair (128 x 256: each CTA fetches one half of the B block
and multicasts it).  Both tilings must give the same bits; the run checks that too.  --profile: the default FullSubNet+ at config
#2's geometry (B clips x 3 s), one model per setting of FSN_GIN_GEMM, the GEMM kernels' time per forward from torch.profiler.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]

HBM_BYTES_PER_S = 3.35e12          # H100 SXM data sheet
FP16_FLOPS = 989e12                # H100 SXM data sheet, dense FP16 (700 W, 1.83 GHz)

# (name, M, N, K) = (ntp x T' x 128, 4 hidden, hidden): config #2 (64 x 257 rows in ntp = 130 tiles of 128, T' = 190, hidden 384)
# and config #5 (32 x 513 rows, 130 tiles, T' = 96, hidden 512)
SHAPES = [("config2_layer1", 130 * 190 * 128, 1536, 384), ("config5_layers12", 130 * 96 * 128, 2048, 512)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clk = (q.stdout.strip().split(", ") + ["", "", ""])[:3] if q.returncode == 0 else ("", "", "")
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi_name": name, "power_limit_w": float(power) if power else None,
            "max_sm_clock_mhz": float(clk) if clk else None}


def counts(M, N, K, tile_n):
    flop = 2.0 * M * N * K
    hbm = 2.0 * (M * K + N * K + M * N)
    l2_smem = (M / 128) * (N / tile_n) * 2.0 * (128 * K + tile_n * K) if tile_n == 128 else (M / 256) * (N / 256) * 2.0 * (2 * 128 * K + 256 * K)
    return flop, hbm, l2_smem


def gemm_alone(args, lib):
    dev = torch.device("cuda:0")
    stream = torch.cuda.current_stream(dev)
    out = {}
    for name, M, N, K in SHAPES:
        g = torch.Generator(device=dev).manual_seed(7)
        A = (torch.randn(M, K, device=dev, generator=g) * 0.5).half()
        B = (torch.randn(N, K, device=dev, generator=g) * (1.0 / K ** 0.5)).half()
        Cs = {t: torch.empty(M, N, device=dev, dtype=torch.half) for t in (128, 256)}

        def call(t):
            rc = lib.fsn_gemm_f16(C.c_void_p(A.data_ptr()), C.c_void_p(B.data_ptr()), C.c_void_p(Cs[t].data_ptr()), M, N, K, t,
                                  C.c_void_p(stream.cuda_stream))
            if rc:
                raise RuntimeError(lib.fsn_last_error().decode())

        def timed(t):
            for _ in range(3):
                call(t)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                call(t)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.iters

        ms = {128: [], 256: []}
        for _ in range(args.rounds):
            for t in (128, 256):
                ms[t].append(timed(t))
        r = {"M": M, "N": N, "K": K, "bit_identical": bool(torch.equal(Cs[128], Cs[256]))}
        for t in (128, 256):
            med = statistics.median(ms[t])
            flop, hbm, l2 = counts(M, N, K, t)
            r[f"tile_128x{t}"] = {"ran_with_tile_n": int(lib.fsn_gemm_f16_tile_n(M, N, K, t)), "ms": med, "rounds_ms": ms[t],
                                  "tflop_s": flop / med / 1e9, "hbm_gb_s": hbm / med / 1e6, "l2_to_smem_gb_s": l2 / med / 1e6,
                                  "flop": flop, "hbm_bytes": hbm, "l2_to_smem_bytes": l2}
        r["hbm_bound_ms"] = hbm / HBM_BYTES_PER_S * 1e3
        r["tensor_bound_ms_datasheet"] = flop / FP16_FLOPS * 1e3
        out[name] = r
        del A, B, Cs
        torch.cuda.empty_cache()
    return out


def through_model(args):
    from fsnplus_b200.model import FullSubNet_Plus
    from fsnplus_b200.synth import synth_clips
    from fsnplus_b200 import inference as inf
    from torch.profiler import ProfilerActivity, profile

    dev = torch.device("cuda:0")
    B, nsamp = args.batch, 48000
    cfg = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM", fb_output_activate_function="ReLU",
               sb_output_activate_function=False, channel_attention_model="TSSE", fb_model_hidden_size=512, sb_model_hidden_size=384,
               norm_type="offline_laplace_norm", num_groups_in_drop_band=2, kersize=[3, 5, 10], subband_num=1)
    X = inf.stft(synth_clips(B, nsamp, 16000, seed=1000).to(dev), 512, 256, 512)
    mag, real, imag = X.abs().unsqueeze(1).contiguous(), X.real.unsqueeze(1).contiguous(), X.imag.unsqueeze(1).contiguous()
    res = {}
    for knob in ("128", None):
        if knob is None:
            os.environ.pop("FSN_GIN_GEMM", None)
        else:
            os.environ["FSN_GIN_GEMM"] = knob
        torch.manual_seed(0)
        m = FullSubNet_Plus(**cfg).to(dev).eval()
        with torch.no_grad():
            for _ in range(2):
                out = m.enhance_spectrum(mag, real, imag)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.steps):
                    m.enhance_spectrum(mag, real, imag)
                torch.cuda.synchronize()
        os.environ.pop("FSN_GIN_GEMM", None)
        kern = {}
        for e in prof.key_averages():
            if "gemm_f16_pair_kernel" in e.key or "gemm_tc5_kernel<4, 128>" in e.key:
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                kern[e.key.split("(")[0]] = {"calls_per_forward": e.count / args.steps, "ms_per_forward": t / 1e3 / args.steps}
        res["FSN_GIN_GEMM=128" if knob else "default"] = {"gin_gemm_kernels": kern, "launches_per_forward": m.last_launch_count(),
                                                          "enhanced": out.cpu()}
        del m
        torch.cuda.empty_cache()
    same = torch.equal(res["default"].pop("enhanced"), res["FSN_GIN_GEMM=128"].pop("enhanced"))
    return {"workload": f"default FullSubNet+, B = {B} x 3 s clips (config #2 geometry), enhance_spectrum, {args.steps} profiled forwards",
            "enhanced_bit_identical": same, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", action="store_true", help="time the GEMM inside a model forward with torch.profiler")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    from fsnplus_b200 import _lib
    lib = _lib.load_library()
    out = {"card": card()}
    if args.profile:
        out["model"] = through_model(args)
    else:
        out.update({"iters": args.iters, "rounds": args.rounds, "timing": "CUDA events, median over the alternated rounds"})
        out["gemm"] = gemm_alone(args, lib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
