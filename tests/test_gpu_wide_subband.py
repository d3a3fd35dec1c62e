"""Wide sub-band inputs (64 < Isb <= 128, DESIGN.md §3.3) on the GPU: the layer-wise path (layer 0 projected by the input-projection
GEMM from rows of 128 halves) and the generic kernel (Ipad = 128), offline and streaming.

  * every wide golden (tests/golden/make_golden_wide.py) within cIRM rel-L2 1e-3 of the reference's fp64 output, on both paths;
  * the sub-band stage alone (fsn_model_sb_forward) element by element against fp64 with the rule of tests/sb_rnn_ref.py at Isb 66, 96
    and 128, hidden 64 / 384 / 512, 1 and 3 layers, LSTM and GRU, fast and accurate gate math; the rule catches planted packer faults
    (the two 64-channel k-blocks swapped, channel 64 dropped);
  * bit identity: windows of 32 and 64 frames and a cap-triggered plan against the unwindowed forward, ragged batches against each
    clip's lone forward, enhance_audio of a ragged batch against each clip alone;
  * streaming fullsubnet.Model (small and default geometry, 3 and 80 slots): step_slots, step_chunk, step_audio and step_audio_chunk
    sessions with staggered starts and holds are bit-identical to their lone runs, the masks within 1e-3 of the fp64 oracle;
    save_slots / load_slots round trips continue bit-identically."""
import numpy as np
import pytest
import torch

import sb_rnn_ref as R
from oracle import fsn_oracle as O
from test_wide_subband_cpu import GOLDENS, golden_cfg, golden_inputs, isb

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASK_TOL = 1e-3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _build(kind, cfg, params, monkeypatch=None, cap_gb=None, **kw):
    from fsnplus_b200.model import FullSubNet_Plus, Model
    if cap_gb is not None:
        monkeypatch.setenv("FSN_WS_CAP_GB", str(cap_gb))
    m = (FullSubNet_Plus if kind == "plus" else Model)(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    if cap_gb is not None:
        monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
    return m


def _params(kind, cfg, seed, scale=1.0, L=2):
    f = O.make_params_plus if kind == "plus" else O.make_params_fsn
    return f(cfg, seed=seed, lstm_scale=scale, num_layers=L)


def _fwd(m, kind, mag, real, imag, **kw):
    with torch.no_grad():
        return m(mag, real, imag, **kw) if kind == "plus" else m(mag, **kw)


# ---------------------------------------------------------------------------------------------------------------------------------
# goldens
@pytest.mark.parametrize("impl", ["auto", "mma"])
@pytest.mark.parametrize("name", list(GOLDENS))
def test_golden(golden, name, impl):
    kind, cfg = golden_cfg(name)
    g = golden(name)
    params = _params(kind, cfg, int(g["seed"]), float(g["lstm_scale"]) if "lstm_scale" in g else 1.0)
    m = _build(kind, cfg, params, lstm_impl=impl)
    mag, real, imag = (_t(x) for x in golden_inputs(golden, name))
    out = _fwd(m, kind, mag, real, imag).cpu().numpy()
    err = O.rel_l2(out, g["out"])
    want_impl = "tcgen05" if impl == "auto" else "mma"
    print(f"\n{name} (Isb {isb(kind, cfg)}) {m.last_lstm_impl()}: cIRM rel-L2 vs fp64 reference {err:.2e}")
    assert m.last_lstm_impl() == want_impl
    assert err <= MASK_TOL


# ---------------------------------------------------------------------------------------------------------------------------------
# the sub-band stage alone, element by element (the helpers of tests/test_gpu_sb_recurrence.py, restated for wide inputs)
WIDE_ISB = {66: (4, 9), 96: (16, 10), 128: (2, 20)}            # Isb: (sb_num_neighbors, fb_num_neighbors) of FullSubNet+
STAGE = [(i, H, 1 + 2 * (n % 2), kind, n % 3 != 2) for n, (i, H, kind) in
         enumerate((i, H, kind) for i in WIDE_ISB for H in (64, 384, 512) for kind in ("LSTM", "GRU"))]
STAGE_MMA = [(128, 64, 2, "LSTM", True), (96, 384, 3, "GRU", False), (128, 512, 4, "LSTM", True)]


def _stage_model(Isb, H, L, kind, fast, impl="auto", F=64, la=2, seed=0):
    cfg = O.default_plus_config()
    Ns, Nf = WIDE_ISB[Isb]
    cfg.update(num_freqs=F, sb_model_hidden_size=H, sequence_model=kind, look_ahead=la, sb_num_neighbors=Ns, fb_num_neighbors=Nf)
    params = _params("plus", cfg, seed, L=L)
    return _build("plus", cfg, params, num_layers=L, lstm_impl=impl, fast_math=fast), params, cfg


def _input(B, F, I, Tp, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(B, F, I, Tp, device=DEV, generator=g)).half().float()      # fp16 values: the packer's rounding is exact


def _sb(m, x, T, Tw=0, frames=None):
    import ctypes as C
    from fsnplus_b200 import _lib
    B, F = x.shape[0], x.shape[1]
    fr = (C.c_int32 * B)(*frames) if frames is not None else None
    out = torch.full((B, 2, F, T), float("nan"), device=DEV)
    with torch.cuda.device(DEV):
        stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
        _lib.check(_lib.load_library().fsn_model_sb_forward(m._handle, C.c_void_p(x.data_ptr()), B, T, Tw, fr, C.c_void_p(out.data_ptr()),
                                                            C.c_void_p(), C.c_void_p(), C.c_void_p(), stream))
    torch.cuda.synchronize()
    return out


def _rule(params, cfg, x, got, fast, xref=None):
    """sb_rnn_ref's rule on every row: got [B, 2, F, T] against fp64 of xref (default x)"""
    B, F, I, Tp = x.shape
    la, kind = cfg["look_ahead"], cfg["sequence_model"]
    xs = (x if xref is None else xref).reshape(B * F, I, Tp)
    dev = DEV if B * F * Tp * cfg["sb_model_hidden_size"] > 2e6 else "cpu"
    want = R.truth(params, kind, xs.to(dev), la, False, device=dev)
    emu = R.emulate(params, kind, xs.to(dev), la, False, device=dev)
    g = got.permute(0, 2, 1, 3).reshape(B * F, 2, Tp - la)
    return R.compare(g, want, emu, R.FAST_FACTOR if fast else 1.0)


def _stage_case(Isb, H, L, kind, fast, impl):
    m, params, cfg = _stage_model(Isb, H, L, kind, fast, impl)
    B, Tp = 2, 41
    x = _input(B, cfg["num_freqs"], Isb, Tp, seed=Isb + H + L)
    got = _sb(m, x, Tp - cfg["look_ahead"])
    r = _rule(params, cfg, x, got, fast)
    print(f"\n[{impl}] Isb={Isb} {kind} H={H} L={L} {'fast' if fast else 'acc '} {m.last_lstm_impl()}: max err/RMS {r['err']:.2e} "
          f"emu {r['emu']:.2e} bound {r['bound']:.2e} ratio {r['ratio']:.2f} rel-L2 {r['rel']:.2e}")
    assert m.last_lstm_impl() == ("tcgen05" if impl == "auto" else "mma")
    assert r["finite"] and r["ok"], r


@pytest.mark.parametrize("Isb,H,L,kind,fast", STAGE)
def test_stage_layerwise(Isb, H, L, kind, fast):
    _stage_case(Isb, H, L, kind, fast, "auto")


@pytest.mark.parametrize("Isb,H,L,kind,fast", STAGE_MMA)
def test_stage_mma(Isb, H, L, kind, fast):
    _stage_case(Isb, H, L, kind, fast, "mma")


@pytest.mark.parametrize("impl", ["auto", "mma"])
def test_rule_catches_planted_faults(impl):
    """The kernel fed a wrongly packed input (what a packer bug would hand it) fails the rule against the true input's fp64."""
    m, params, cfg = _stage_model(128, 64, 1, "LSTM", False, impl)
    B, Tp = 1, 41
    x = _input(B, cfg["num_freqs"], 128, Tp, seed=5)
    T = Tp - cfg["look_ahead"]
    assert _rule(params, cfg, x, _sb(m, x, T), False)["ok"]
    swapped = torch.cat([x[:, :, 64:], x[:, :, :64]], 2).contiguous()       # the two 64-channel k-blocks swapped
    dropped = x.clone()
    dropped[:, :, 64] = 0                                                    # channel 64 (the second block's first) dropped
    for label, bad in (("k-blocks swapped", swapped), ("channel 64 dropped", dropped)):
        r = _rule(params, cfg, bad, _sb(m, bad, T), False, xref=x)
        print(f"\n[{impl}] planted fault '{label}': max err/RMS {r['err']:.2e} bound {r['bound']:.2e}")
        assert not r["ok"], label


# ---------------------------------------------------------------------------------------------------------------------------------
# bit identity
def test_windows_bit_identical(monkeypatch):
    m, params, cfg = _stage_model(128, 384, 3, "LSTM", True)
    x = _input(3, cfg["num_freqs"], 128, 150, seed=9)
    T = 150 - cfg["look_ahead"]
    ref = _sb(m, x, T)
    for tw in (32, 64):
        assert torch.equal(_sb(m, x, T, Tw=tw), ref), tw
    # a full forward whose plan windows under a small cap, against the unwindowed plan
    cfg = O.default_plus_config()
    cfg.update(sb_num_neighbors=15, fb_num_neighbors=15)
    params = _params("plus", cfg, 3)
    rng = np.random.default_rng(1)
    re, im = rng.standard_normal((2, 1, 257, 400)).astype(np.float32) * 0.05, rng.standard_normal((2, 1, 257, 400)).astype(np.float32) * 0.05
    mag, real, imag = _t(np.sqrt(re ** 2 + im ** 2)), _t(re), _t(im)
    full = _fwd(_build("plus", cfg, params), "plus", mag, real, imag)
    mc = _build("plus", cfg, params, monkeypatch, cap_gb=0.3)
    win = _fwd(mc, "plus", mag, real, imag)
    bs, tw = mc.last_plan()
    print(f"\ncap-triggered plan: sub-batch {bs}, window {tw}")
    assert tw > 0
    assert torch.equal(win, full)


def test_ragged_and_audio_bit_identical():
    name = "plus_small_wide128"
    kind, cfg = golden_cfg(name)
    params = _params(kind, cfg, 7)
    m = _build(kind, cfg, params)
    rng = np.random.default_rng(2)
    B, F, T = 4, cfg["num_freqs"], 50
    re, im = rng.standard_normal((B, 1, F, T)).astype(np.float32) * 0.05, rng.standard_normal((B, 1, F, T)).astype(np.float32) * 0.05
    mag, real, imag = _t(np.sqrt(re ** 2 + im ** 2)), _t(re), _t(im)
    frames = [50, 8, 33, 17]                                     # >= 8: frames + look_ahead covers the TSSE kernel (10)
    out = _fwd(m, kind, mag, real, imag, frames=frames)
    for b, n in enumerate(frames):
        lone = _fwd(m, kind, mag[b:b + 1, :, :, :n].contiguous(), real[b:b + 1, :, :, :n].contiguous(), imag[b:b + 1, :, :, :n].contiguous())
        assert torch.equal(out[b:b + 1, :, :, :n], lone), b
        assert not out[b, :, :, n:].any()
    hop = F - 1
    wave = _t((rng.standard_normal((3, 60 * hop)) * 0.1).astype(np.float32))
    lens = [60 * hop, 17 * hop + 5, 33 * hop]
    with torch.no_grad():
        y = m.enhance_audio(wave, lens)
        assert torch.isfinite(y).all()
        for b, n in enumerate(lens):
            assert torch.equal(y[b, :n], m.enhance_audio(wave[b:b + 1, :n].contiguous())[0]), b


# ---------------------------------------------------------------------------------------------------------------------------------
# streaming (fullsubnet.Model with a cumulative norm)
def _stream_cfg(default):
    cfg = O.default_fsn_config()
    if default:                                                  # F = 257, hidden 384 / 512: Isb 31 + 61 = 92
        cfg.update(sb_num_neighbors=15, fb_num_neighbors=30, norm_type="cumulative_laplace_norm")
    else:
        _, cfg = golden_cfg("fsn_small_wide128")
    return cfg


GEOMS = [(False, 3), (True, 3), (True, 80)]


def _schedule(nslots, T, la, ncalls, seed):
    """Per slot: (start call, holds): staggered starts, a few holds inside each session"""
    rng = np.random.default_rng(seed)
    out = []
    for b in range(nslots):
        start = int(rng.integers(0, 3))
        holds = set(int(v) for v in rng.integers(start + 1, start + T, size=2))
        out.append((start, holds))
    return out


def _flags(sched, steps_needed, ncalls):
    """call -> flags per slot (HOLD 0 / STEP 1 / START 2); a slot steps until it has made steps_needed steps"""
    from fsnplus_b200.streaming import HOLD, STEP, START
    flags, done = [], [0] * len(sched)
    for c in range(ncalls):
        f = []
        for b, (start, holds) in enumerate(sched):
            if c < start or done[b] >= steps_needed or c in holds:
                f.append(HOLD)
            else:
                f.append(START if c == start else STEP)
                done[b] += 1
        flags.append(f)
    return flags


@pytest.mark.parametrize("default,nslots", GEOMS)
def test_stream_slots_and_chunks(default, nslots):
    from fsnplus_b200.streaming import StreamingFullSubNet, HOLD
    cfg = _stream_cfg(default)
    params = _params("fsn", cfg, 31)
    F, la = cfg["num_freqs"], cfg["look_ahead"]
    T = 24 if default else 20
    rng = np.random.default_rng(nslots)
    clips = (np.abs(rng.standard_normal((nslots, F, T))) * 0.05 + 0.01).astype(np.float32)
    want = O.fullsubnet_forward(params, cfg, clips[:, None])                      # [nslots, 2, F, T] fp64 oracle
    for impl in ("auto", "mma"):
        m = _build("fsn", cfg, params, lstm_impl=impl)
        # ---- step_slots: one frame per tick
        steps = T + la
        sched = _schedule(nslots, steps, la, 0, 1)
        ncalls = max(s for s, _ in sched) + steps + 4
        flags = _flags(sched, steps, ncalls)
        st = StreamingFullSubNet(m, nslots)
        n = [0] * nslots
        got = [[] for _ in range(nslots)]
        saved = None
        for c, f in enumerate(flags):
            x = torch.full((nslots, F), float("nan"), device=DEV)
            for b in range(nslots):
                if f[b] != HOLD:
                    x[b] = _t(clips[b, :, n[b]] if n[b] < T else np.zeros(F, np.float32))
                    n[b] += 1
            mask, valid = st.step_slots(x, f)
            for b in range(nslots):
                if valid[b]:
                    got[b].append(mask[b].clone())
            if c == ncalls // 2:
                saved = (c, st.save_slots([0]), n[0], len(got[0]))
        res = torch.stack([torch.stack(g, -1) for g in got])                     # [nslots, 2, F, T]
        err = O.rel_l2(res.cpu().numpy(), want)
        print(f"\nstep_slots {impl} F={F} slots={nslots}: rel-L2 vs fp64 {err:.2e}")
        assert err <= MASK_TOL
        # lone run of each of a few sessions: its own ticks on a 1-slot handle
        for b in sorted({0, nslots - 1}):
            lone = StreamingFullSubNet(m, 1)
            out = []
            for c, f in enumerate(flags):
                if f[b] == HOLD:
                    continue
                k = len([1 for cc in range(c) if flags[cc][b] != HOLD])
                x = _t(clips[b:b + 1, :, k] if k < T else np.zeros((1, F), np.float32))
                mask, valid = lone.step_slots(x, [f[b]])
                if valid[0]:
                    out.append(mask[0].clone())
            assert torch.equal(torch.stack(out, -1), res[b]), b
        # save / load: slot 0's session continued from its snapshot in slot 1 of a fresh handle
        c0, state, k0, v0 = saved
        st2 = StreamingFullSubNet(m, 2)
        st2.load_slots([1], state)
        out = []
        for c in range(c0 + 1, ncalls):
            f0 = flags[c][0]
            if f0 == HOLD:
                continue
            x = torch.full((2, F), float("nan"), device=DEV)
            x[1] = _t(clips[0, :, k0] if k0 < T else np.zeros(F, np.float32))
            k0 += 1
            mask, valid = st2.step_slots(x, [HOLD, f0])
            if valid[1]:
                out.append(mask[1].clone())
        assert torch.equal(torch.stack(out, -1), res[0, ..., v0:])
        # ---- step_chunk: K frames per call, staggered; each session against one call over all its frames on a 1-slot handle
        Ks = [3, 4, 1, 9, 32, 4]
        st = StreamingFullSubNet(m, nslots)
        n = [0] * nslots
        got = [[] for _ in range(nslots)]
        c = 0
        while min(n) < steps and c < 64:
            K = Ks[c % len(Ks)]
            f = []
            x = torch.full((nslots, F, K), float("nan"), device=DEV)
            for b in range(nslots):
                start = b % 3
                if c < start or n[b] >= steps or (c == start + 2 and b % 2):
                    f.append(HOLD)
                    continue
                f.append(2 if n[b] == 0 else 1)
                seg = np.zeros((F, K), np.float32)
                take = max(0, min(K, T - n[b]))
                if take:
                    seg[:, :take] = clips[b, :, n[b]:n[b] + take]
                x[b] = _t(seg)
                n[b] += K
            mask, nvalid = st.step_chunk(x, f)
            for b in range(nslots):
                if f[b] != HOLD and nvalid[b]:
                    got[b].append(mask[b, ..., K - int(nvalid[b]):].clone())
            c += 1
        for b in range(nslots):
            g = torch.cat(got[b], -1)[..., :T]
            assert O.rel_l2(g.cpu().numpy(), want[b]) <= MASK_TOL, b
        for b in sorted({0, nslots - 1}):
            lone = StreamingFullSubNet(m, 1)
            seg = np.zeros((1, F, steps), np.float32)
            seg[0, :, :T] = clips[b]
            mask, nvalid = lone.step_chunk(_t(seg), [2])
            assert torch.equal(torch.cat(got[b], -1)[..., :T], mask[0, ..., steps - int(nvalid[0]):][..., :T]), b


@pytest.mark.parametrize("default,nslots", GEOMS)
def test_stream_audio(default, nslots):
    from fsnplus_b200.streaming import StreamingFullSubNet, HOLD, STEP, START, FLUSH
    cfg = _stream_cfg(default)
    params = _params("fsn", cfg, 32)
    F, la = cfg["num_freqs"], cfg["look_ahead"]
    hop = F - 1
    nh = 12
    rng = np.random.default_rng(3 + nslots)
    wave = (rng.standard_normal((nslots, nh * hop)) * 0.1).astype(np.float32)
    m = _build("fsn", cfg, params)
    # per-hop call: slot b starts at tick b % 3, holds one tick, then flushes look_ahead + 2 ticks
    def plan(b):
        seq = [START] + [STEP] * (nh - 1) + [FLUSH] * (la + 2)
        seq = [HOLD] * (b % 3) + seq[:4] + [HOLD] + seq[4:]
        return seq
    plans = [plan(b) for b in range(nslots)]
    ticks = max(len(p) for p in plans)
    st = StreamingFullSubNet(m, nslots)
    outs = [[] for _ in range(nslots)]
    k = [0] * nslots
    for t in range(ticks):
        f = [plans[b][t] if t < len(plans[b]) else HOLD for b in range(nslots)]
        x = torch.full((nslots, hop), float("nan"), device=DEV)
        for b in range(nslots):
            if f[b] in (START, STEP):
                x[b] = _t(wave[b, k[b] * hop:(k[b] + 1) * hop])
                k[b] += 1
        y, valid = st.step_audio(x, f)
        for b in range(nslots):
            if valid[b]:
                outs[b].append(y[b].clone())
    for b in sorted({0, nslots - 1}):
        lone = StreamingFullSubNet(m, 1)
        got, kk = [], 0
        for f in plans[b]:
            if f == HOLD:
                continue
            x = _t(wave[b:b + 1, kk * hop:(kk + 1) * hop]) if f in (START, STEP) else torch.full((1, hop), float("nan"), device=DEV)
            kk += f in (START, STEP)
            y, valid = lone.step_audio(x, [f])
            if valid[0]:
                got.append(y[0].clone())
        assert len(got) == nh and torch.equal(torch.stack(got), torch.stack(outs[b])), b
    # K-hop call: START 4, STEP 4, STEP 2 (then HOLD), FLUSH 0 (look_ahead + 2 = 4 flush ticks), staggered and held per slot
    K = 4
    calls = [(START, 4), (STEP, 4), (STEP, 2), (FLUSH, 0)]
    plans = [[(HOLD, 0)] * (b % 3) + calls[:2] + [(HOLD, 0)] * (b % 2) + calls[2:] for b in range(nslots)]
    ncalls = max(len(p) for p in plans)
    st = StreamingFullSubNet(m, nslots)
    outs = [[] for _ in range(nslots)]
    k = [0] * nslots
    for c in range(ncalls):
        fl = [plans[b][c] if c < len(plans[b]) else (HOLD, 0) for b in range(nslots)]
        x = torch.full((nslots, K * hop), float("nan"), device=DEV)
        for b, (f, h) in enumerate(fl):
            if f != HOLD and h:
                x[b, :h * hop] = _t(wave[b, k[b] * hop:(k[b] + h) * hop])
                k[b] += h
        y, nout = st.step_audio_chunk(x, [f for f, _ in fl], [h for _, h in fl])
        for b in range(nslots):
            if int(nout[b]):
                outs[b].append(y[b, :int(nout[b]) * hop].clone())
    for b in sorted({0, nslots - 1}):
        lone = StreamingFullSubNet(m, 1)
        got, kk = [], 0
        for f, h in plans[b]:
            if f == HOLD:
                continue
            x = torch.full((1, K * hop), float("nan"), device=DEV)
            if h:
                x[0, :h * hop] = _t(wave[b, kk * hop:(kk + h) * hop])
                kk += h
            y, nout = lone.step_audio_chunk(x, [f], [h])
            if int(nout[0]):
                got.append(y[0, :int(nout[0]) * hop].clone())
        a, o = torch.cat(got), torch.cat(outs[b])
        assert a.numel() == 10 * hop and torch.isfinite(a).all() and torch.equal(a, o), b      # 4 + 4 + 2 hops
