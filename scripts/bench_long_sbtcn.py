"""Long clips with the sub-band TCN (DESIGN.md §3.8): the cost of bin chunks and end-to-end times of single long recordings.

    python scripts/bench_long_sbtcn.py [--minutes 10,30,60] [--skip-batch]

(a) one 90 s clip, unchunked vs FSN_SB_CHUNK=64, arms alternated: the cost of chunking;
(b) 10 / 30 / 60 min single clips through enhance_batch at the default cap: wall time, RTF, plan and workspace_bytes();
(c) 4 x 30 min clips in one call.
Default FullSubNet+ config with sequence_model = "TCN", reference weight init, synthetic audio; prints one line per measurement.
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]

import torch  # noqa: E402

from fsnplus_b200 import inference as H  # noqa: E402
from fsnplus_b200.model import FullSubNet_Plus  # noqa: E402

DEV = "cuda:0"
# the reference's config/inference.toml model arguments, with the TCN sub-band model
DEFAULT_CONFIG = dict(num_freqs=257, look_ahead=2, sequence_model="TCN", fb_num_neighbors=0, sb_num_neighbors=15,
                      fb_output_activate_function="ReLU", sb_output_activate_function=False, channel_attention_model="TSSE",
                      fb_model_hidden_size=512, sb_model_hidden_size=384, norm_type="offline_laplace_norm", num_groups_in_drop_band=2,
                      kersize=[3, 5, 10], subband_num=1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(0)


def make_model(chunk=None):
    if chunk:
        os.environ["FSN_SB_CHUNK"] = str(chunk)
    else:
        os.environ.pop("FSN_SB_CHUNK", None)
    torch.manual_seed(0)
    m = FullSubNet_Plus(**DEFAULT_CONFIG).to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    os.environ.pop("FSN_SB_CHUNK", None)
    return m


def timed(m, noisy):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        y = H.enhance_batch(m, noisy)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", default="10,30,60")
    ap.add_argument("--skip-batch", action="store_true")
    args = ap.parse_args()
    print(f"card: {card()}")
    g = torch.Generator().manual_seed(0)
    clip = lambda B, s: (torch.randn(B, int(s * 16000), generator=g) * 0.05).to(DEV)

    x = clip(1, 90)
    arms = {"unchunked": make_model(), "chunks of 64 bins": make_model(64)}
    for m in arms.values():
        timed(m, x)                                                   # warm-up: allocations
    res = {k: [] for k in arms}
    for _ in range(3):
        for k, m in arms.items():
            res[k].append(timed(m, x)[0])
    for k, m in arms.items():
        print(f"(a) 90 s clip, {k}: {', '.join(f'{t * 1e3:.1f}' for t in res[k])} ms, plan {m.last_plan_bins()}, "
              f"{m.last_launch_count()} launches")
    del arms
    torch.cuda.empty_cache()

    m = make_model()
    timed(m, clip(1, 5))
    for mins in [float(v) for v in args.minutes.split(",")]:
        dt, y = timed(m, clip(1, 60 * mins))
        print(f"(b) {mins:g} min clip: {dt:.2f} s, RTF {dt / (60 * mins):.2e}, plan {m.last_plan_bins()}, "
              f"workspace {m.workspace_bytes() / 1e9:.2f} GB, finite {bool(torch.isfinite(y).all())}")
        del y
    if not args.skip_batch:
        dt, y = timed(m, clip(4, 1800))
        print(f"(c) 4 x 30 min clips: {dt:.2f} s, RTF {dt / 7200:.2e}, plan {m.last_plan_bins()}, "
              f"workspace {m.workspace_bytes() / 1e9:.2f} GB, finite {bool(torch.isfinite(y).all())}")


if __name__ == "__main__":
    main()
