import os, sys, time, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "fullsubnet-plus_b200")]
from fsnplus_b200.model import Model, FullSubNet_Plus
import bench
torch.manual_seed(0)
dev = "cuda:0"
cfg = dict(sb_num_neighbors=15, fb_num_neighbors=0, num_freqs=257, look_ahead=2, sequence_model="LSTM", fb_output_activate_function="ReLU",
           sb_output_activate_function=False, fb_model_hidden_size=512, sb_model_hidden_size=384, weight_init=False)
def timeit(fn, n=5):
    for _ in range(3): fn()
    torch.cuda.synchronize(); e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize(); return e0.elapsed_time(e1) / n
with torch.no_grad():
    m = Model(**cfg).to(dev).eval()
    for B in (1, 8, 64):
        x = torch.rand(B, 1, 257, 188, device=dev)
        print(f"fullsubnet.Model B={B}: {timeit(lambda: m(x)):.2f} ms  (sub-band LSTM {m.last_lstm_ms():.2f} ms)")
    # FullSubNet+ from one clip to the flagship batch
    p = FullSubNet_Plus(**bench.default_cfg()).to(dev).eval()
    for B in (1, 2, 4, 8, 16, 24, 32, 48, 64):
        x = torch.rand(B, 1, 257, 188, device=dev)
        ta = timeit(lambda: p(x, x - 0.5, x - 0.3)); la = p.last_lstm_ms()
        print(f"FullSubNet_Plus B={B:2d}: {ta:6.2f} ms (sub-band LSTM {la:5.2f})   {ta / B:6.3f} ms/clip")
    # other constructor values: GRU sub-band model (tensor-core LSTM path with the GRU cell), SE attention, and BASELINE config #5
    # (F = 513, H = 512, 3 layers, B = 32, T = 94)
    x = torch.rand(64, 1, 257, 188, device=dev)
    g = FullSubNet_Plus(**dict(bench.default_cfg(), sequence_model="GRU")).to(dev).eval()
    print(f"FullSubNet_Plus GRU B=64: {timeit(lambda: g(x, x - 0.5, x - 0.3)):.2f} ms  (sub-band GRU {g.last_lstm_ms():.2f} ms, {g.last_lstm_impl()})")
    del g
    a = FullSubNet_Plus(**dict(bench.default_cfg(), channel_attention_model="SE")).to(dev).eval()
    print(f"FullSubNet_Plus SE attention B=64: {timeit(lambda: a(x, x - 0.5, x - 0.3)):.2f} ms")
    del a
    big = dict(bench.default_cfg(), num_freqs=513, sb_model_hidden_size=512, fb_model_hidden_size=512)
    l = FullSubNet_Plus(**big, num_layers=3).to(dev).eval()
    xl = torch.rand(32, 1, 513, 94, device=dev)
    ms = timeit(lambda: l(xl, xl - 0.5, xl - 0.3), n=3)
    flop = 32 * 525.9e9
    print(f"config #5 (F=513, H=512, L=3, B=32, T=94): {ms:.2f} ms  (sub-band LSTM {l.last_lstm_ms():.2f} ms, {l.last_lstm_impl()}; "
          f"{flop / ms / 1e9:.0f} TFLOP/s algorithmic)")
