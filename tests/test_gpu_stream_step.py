"""The streaming step (fsn_stream_step / _step_slots / _step_chunk, DESIGN.md §3.9, §3.13) element by element against fp64, stage by
stage, from each stage's own input and carried state (tests/stream_ref.py):

* fb_in (get_stage) against the reference's cumulative norm of the session's frames since its START; the payload's cum_in against
  the fp64 sums (within 1e-12 of the sums of |x| and x^2);
* fb_out and the full band's (h, c) after the call against the fp64 LSTM / GRU from the call's own fb_in and the (h, c) saved before;
* the sub-band input (generic path: the decoded sb_img) against the fp64 unfold + cumulative norm of the session's magnitude and the
  kernels' fb_out; cum_sb against its fp64 sums;
* the mask columns and the sub band's (h, c) after the call against the fp64 LSTM / GRU from the decoded images (layer-wise path: the
  emulated pack, so a fault of the compact-row or window pack or of the carry shows up here) and the (h, c) saved before.  Columns of
  a negative frame and held rows must be exactly 0; a held slot's payload must not change.
The audio calls (per hop and chunk, per-slot hop counts so kf < K) add the analysis: "mag" against |rfft| in fp64 of the session's
samples (reflect at 0 and, after the FLUSH, at L - 1; zero frames past the last hop), emulated by an fp32 FFT, factor AUDIO_FACTOR;
then every model stage from those frames; columns past a slot's kf must be exactly 0.
Slots, not rows, are sampled: at 80 slots the checked slots are 0, 1, 63, 64 and 79 (the 64-slot and tile boundaries), every bin of
each, instead of sb_rnn_ref.sample_rows over B F rows.
The lockstep call is checked through the hook and the masks only, from zero state over the whole session (a save would switch the
handle to slot counts), and saved once at the end.
Rule (sb_rnn_ref.compare): max |kernel - fp64| <= factor * (3 max |emulation - fp64| + 1e-6 RMS), factor 1 (accurate gates and the
norm / pack) or sb_rnn_ref.FAST_FACTOR (fast gates).  One printed line per stage and case; the last test prints the worst case per
stage (DESIGN.md §2).  test_stream_step_cpu.py checks that the case lists reach the edges they claim and that the rule catches the
planted faults."""
import numpy as np
import pytest
import torch

import front_ref as FR
import sb_rnn_ref as R
import stream_ref as S
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WORST = {}
SUM_TOL = 1e-12

# ---- case lists (test_stream_step_cpu.py checks their reach) -----------------------------------------------------------------------
GEOMETRY = [(33, 3), (65, 2), (129, 1), (257, 3), (513, 1), (257, 80)]               # (F, B): B F straddles 128-row tiles at 257 x 3 / 80
MMA_H = [(64, 2), (384, 3), (512, 4)]                                                 # (Hsb, L) of the generic kernel: R = 64, 32, 16
WIDE = [(32, 0), (31, 32)]                                                            # (Ns, Nf): Isb 66, 128
KS = [3, 4, 1, 37, 1, 32, 5]                                                          # chunk calls: 1-frame calls and K = 37
LONG_T, LONG_K = 1876, 32                                                             # the 30 s config #4 clip, in 32-frame calls


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _record(stage, label, r):
    if r["err"] >= WORST.get(stage, (-1.0,))[0]:
        WORST[stage] = (r["err"], r["ratio"], label)


def _check(stage, label, got, want, emu, factor, extra=""):
    r = R.compare(got, want, emu, factor)
    print(f"\n[{label}] {stage}{extra}: max err/RMS {r['err']:.2e} emu {r['emu']:.2e} bound {r['bound']:.2e} ratio {r['ratio']:.2f} "
          f"rel-L2 {r['rel']:.2e}")
    _record(stage, label, r)
    assert r["finite"] and r["ok"], (label, stage, r)


def _sums_ok(label, got, x):
    """payload sums [.., 2] against the fp64 sums of x's values (float64 [.., n]): within SUM_TOL of sum |x| and sum x^2"""
    want = np.stack([x.sum(-1), (x * x).sum(-1)], -1)
    tol = SUM_TOL * np.stack([np.abs(x).sum(-1), (x * x).sum(-1)], -1) + 1e-300
    assert np.all(np.abs(got - want) <= tol), (label, float(np.max(np.abs(got - want) / tol)))


def _model(F=257, Hfb=512, Hsb=384, L=2, kind="LSTM", norm="cumulative_laplace_norm", fast=True, impl="auto", Ns=7, Nf=0, la=2,
           seed=0, monkeypatch=None, env=None):
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=F, fb_model_hidden_size=Hfb, sb_model_hidden_size=Hsb, sequence_model=kind, norm_type=norm,
               sb_num_neighbors=Ns, fb_num_neighbors=Nf, look_ahead=la)
    params = O.make_params_fsn(cfg, seed=seed, num_layers=L)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    m = Model(**cfg, num_layers=L, lstm_impl=impl, fast_math=fast)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    for k in (env or {}):
        monkeypatch.delenv(k, raising=False)
    return m, params, cfg, dict(L=L, Hfb=Hfb, Hsb=Hsb, kind=kind, norm=norm, fast=fast, Ns=Ns, Nf=Nf, la=la,
                                act=cfg["fb_output_activate_function"], sb_act=cfg["sb_output_activate_function"])


def _clip(F, T, seed, scale=1.0, zero_open=0):
    rng = np.random.default_rng(seed)
    re, im = rng.standard_normal((F, T)) * 0.05 + 0.004, rng.standard_normal((F, T)) * 0.05 - 0.003
    x = (np.sqrt(re ** 2 + im ** 2) * scale).astype(np.float32)
    x[:, :zero_open] = 0
    return x


class Sess:
    """one session on one slot: its clip (then zero frames), and what the kernels fed it so far (magnitude and fb_out frames)"""
    def __init__(self, clip):
        self.clip, self.n, self.mag, self.fb = clip, 0, [], []

    def frames(self, K):
        F, T = self.clip.shape
        out = np.zeros((F, K), np.float32)
        if self.n < T:
            out[:, :min(K, T - self.n)] = self.clip[:, self.n:self.n + K]
        return out


def _img(st, m, cfg, K):
    """the call's decoded sub-band input [B F, Isb, K] (float64) of the generic path"""
    F, B = cfg["num_freqs"], st.B
    I = 2 * cfg["sb_num_neighbors"] + 1 + 2 * cfg["fb_num_neighbors"] + 1
    wide = I > 64
    rows = B * F
    nb = (rows + 127) // 128 * K * 128 * (256 if wide else 128)
    raw = st.get_stage("sb_img", (nb // 4,)).cpu().numpy().view(np.uint8)
    full = np.zeros(FR.img_bytes(rows, K, wide), np.uint8)
    full[:nb] = raw
    vals, _ = FR.decode_sb_img(full, rows, K, 128 if wide else 64, "wide_tm" if wide else "sw128")
    assert not np.any(vals[:, I:]), "channels past Isb of the sub-band images are not zero"   # rows past B F are never read
    return vals[:, :I].astype(np.float64)


def _rnn_check(label, stage, p, prefix, head, x, state, kf, got, got_state, fast, cols=None, dev=DEV):
    """the recurrence of one slot over kf frames from x [N, I, kf] and state (h, c) [L, N, H]: its outputs (columns `cols`) and final
    state against fp64"""
    act = p["act"] if head == "fb" else p["sb_act"]
    xt = torch.as_tensor(x[..., :kf]).to(dev, torch.float64)
    st = tuple(torch.as_tensor(v).to(dev, torch.float64) for v in state)
    want, (hw, cw) = R.truth(p["params"], p["kind"], xt, 0, act, dev, prefix, head, state=st, return_state=True)
    emu, (he, ce) = R.emulate(p["params"], p["kind"], xt, 0, act, dev, prefix=prefix, head=head, state=st, return_state=True)
    f = R.FAST_FACTOR if fast else 1.0
    c = slice(None) if cols is None else cols
    if want[..., c].numel():
        _check(f"{stage} out", label, got[..., c], want[..., c], emu[..., c], f)
    if got_state is not None:
        _check(f"{stage} h", label, got_state[0], hw, he, f)
        _check(f"{stage} c", label, got_state[1], cw, ce, f)


def gru_c_is_fp32(c):
    """the GRU carries its h in fp32 (the payload's c): most nonzero values are not fp16 numbers, as they would all be had the carry
    been rounded to fp16"""
    c = np.asarray(c, np.float64)
    nz = c[c != 0]
    return nz.size > 0 and float(np.mean(nz.astype(np.float16).astype(np.float64) == nz)) < 0.5


def _slot_state(pl, p, F):
    d = S.decode(pl, F, p["L"], p["Hfb"], p["Hsb"])
    d["h_fb"], d["c_fb"] = d["h_fb"][:, None], d["c_fb"][:, None]                       # [L, 1, H]: one sequence
    return d


def _check_slot(label, p, F, s, K, fb_in, fb_out, img, mask, before, after, layerwise):
    """one stepping slot's call: norm, full band, pack and sub band, each from its own input and the state saved before"""
    la, kind = p["la"], p["norm"]
    n0 = s.n - K                                                                       # frames before this call
    xs = np.concatenate(s.mag, axis=1).astype(np.float64)                              # [F, n]
    _check("norm", label, fb_in, S.norm_truth(xs, kind)[:, n0:], S.norm_emulate(xs, kind)[:, n0:], 1.0)
    _sums_ok(label + " cum_in", after["cum_in"], xs.reshape(1, -1))
    _rnn_check(label, "full band", p, "fb_model", "fb", fb_in[None], (before["h_fb"], before["c_fb"]), K, fb_out[None],
               (after["h_fb"], after["c_fb"]), p["fast"])
    fbs = np.concatenate(s.fb, axis=1).astype(np.float64)
    want = S.sb_truth(xs, fbs, p["Ns"], p["Nf"], kind)[..., n0:]
    emu = S.sb_emulate(xs, fbs, p["Ns"], p["Nf"], kind)[..., n0:]
    if img is not None:
        _check("sub-band input", label, img, want, emu, 1.0)
    _sums_ok(label + " cum_sb", after["cum_sb"], S.unfold(xs.astype(np.float32), fbs.astype(np.float32), p["Ns"], p["Nf"])
             .astype(np.float64).reshape(F, -1))
    if p["kind"] == "GRU":
        assert gru_c_is_fp32(after["c_fb"]) and gru_c_is_fp32(after["c_sb"]), (label, "the GRU's carried h was rounded to fp16")
    x = emu if img is None else img
    cols = [k for k in range(K) if n0 + k - la >= 0]
    assert np.all(mask[:, :, [k for k in range(K) if k not in cols]] == 0), (label, "columns of negative frames are not zero")
    if cols:
        cols = slice(cols[0], K)
    else:
        cols = slice(K, K)
    _rnn_check(label, "sub band", p, "sb_model", "sb", x, (before["h_sb"], before["c_sb"]), K, torch.as_tensor(mask).permute(1, 0, 2),
               (after["h_sb"], after["c_sb"]), p["fast"], cols)


def _run_slots(label, m, p, cfg, B, schedule, chunk, check=None, check_from=0, lw=False, ws=None):
    """schedule: [(K, {slot: ("start", clip) | "step"}), ...] (slots not listed HOLD, fed NaN).  Every call is checked on the slots
    of `check` (default: all) from call check_from on; held slots' payloads must not change and their rows must be zero.  lw: the
    sub band must run layer-wise (else on the generic kernel); ws: None, or whether the full band must run weight-stationary."""
    from fsnplus_b200.streaming import HOLD, START, STEP, StreamingFullSubNet
    F = cfg["num_freqs"]
    st = StreamingFullSubNet(m, B, DEV)
    if ws is not None:
        assert st.lib.fsn_stream_fb_ws(st._st) == int(ws), (label, "full-band kernel")
    sess = {}
    chk = list(range(B)) if check is None else list(check)
    layerwise = None
    for ci, (K, acts) in enumerate(schedule):
        flags = np.full(B, HOLD, np.int32)
        mag = np.full((B, F, K), np.nan, np.float32)
        for b, a in acts.items():
            if isinstance(a, tuple):
                sess[b] = Sess(a[1])
                flags[b] = START
            else:
                flags[b] = STEP
            mag[b] = sess[b].frames(K)
        live = ci >= check_from
        before = st.save_slots(chk).payload.cpu().numpy() if live and ci else None      # a fresh handle has no mode to save in yet
        if chunk:
            mask, _ = st.step_chunk(_t(mag), torch.from_numpy(flags))
        else:
            assert K == 1
            mask, _ = st.step_slots(_t(mag[..., 0]), torch.from_numpy(flags))
            mask = mask[..., None]
        fb_in = st.get_stage("fb_in", (B, F, K)).cpu().numpy()
        fb_out = st.get_stage("fb_out", (B, F, K)).cpu().numpy()
        if layerwise is None:
            layerwise = _layerwise(st)
            assert layerwise == lw, (label, "sub-band route", layerwise)
        img = None if layerwise or not live else _img(st, m, cfg, K)
        mask = mask.cpu().numpy()
        for b, a in acts.items():
            s = sess[b]
            s.mag.append(mag[b])
            s.fb.append(fb_out[b])
            s.n += K
        if not live:
            continue
        after = st.save_slots(chk).payload.cpu().numpy()
        for i, b in enumerate(chk):
            if b not in acts:
                assert before is None or np.array_equal(before[i], after[i]), (label, ci, b, "a held slot's state changed")
                assert not np.any(mask[b]), (label, ci, b, "a held slot's mask row is not zero")
                continue
            started = isinstance(acts[b], tuple)                                         # a START runs from zero state
            _check_slot(f"{label} call {ci} slot {b} K={K}", p, F, sess[b], K, fb_in[b], fb_out[b],
                        None if img is None else img[b * F:(b + 1) * F], mask[b],
                        _slot_state(np.zeros_like(after[i]) if started else before[i], p, F), _slot_state(after[i], p, F), layerwise)
    return st


def _layerwise(st):
    """whether the handle's last call ran the sub band layer-wise: get_stage("sb_img") refuses it as FSN_ESTATE (the generic path's
    images are refused for the wrong numel instead)"""
    import ctypes as C
    probe = torch.zeros(1, device=DEV)
    rc = st.lib.fsn_stream_get_stage(st._st, b"sb_img", C.c_void_p(probe.data_ptr()), 0, None)
    assert rc in (-1, -3), rc
    return rc == -3


def _staggered(B, F, Ks, seed, T=40):
    """B sessions: slot b STARTs at call b % 3, slot 1 holds at call 3, slot 0 ends and restarts a quiet session (slot reuse)"""
    clip = lambda i, sc=1.0: _clip(F, T, seed + i, sc)
    sched = []
    for ci, K in enumerate(Ks):
        acts = {}
        for b in range(B):
            if ci == b % 3:
                acts[b] = ("start", clip(b, 30.0 if b == 0 else 1.0))
            elif ci > b % 3 and not (b == 1 and ci == 3):
                acts[b] = "step"
        if ci == len(Ks) - 2 and B > 0:
            acts[0] = ("start", clip(99, 1e-3))                                       # slot reuse: a quiet session after a loud one
        sched.append((K, acts))
    return sched


def _p(params, extra):
    return dict(extra, params=params)


# ---- slot calls ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F,B", GEOMETRY)
def test_step_slots_geometry(built_lib, F, B):
    m, params, cfg, p = _model(F=F, Hfb=96 if F != 257 else 512, Hsb=64, impl="mma", seed=F + B)
    _run_slots(f"slots F={F} B={B}", m, cfg=cfg, p=_p(params, p), B=B, schedule=_staggered(B, F, [1] * 6, F), chunk=False,
               check=sorted({0, 1, B - 1} & set(range(B))))


@pytest.mark.parametrize("kind,norm,fast", [("LSTM", "cumulative_layer_norm", False), ("GRU", "cumulative_laplace_norm", True),
                                            ("GRU", "cumulative_layer_norm", False)])
def test_step_chunk_layerwise_variants(built_lib, kind, norm, fast):
    m, params, cfg, p = _model(F=257, kind=kind, norm=norm, fast=fast, seed=3)
    _run_slots(f"chunk lw {kind} {norm[11:]} {'fast' if fast else 'acc'}", m, cfg=cfg, p=_p(params, p), B=3,
               schedule=_staggered(3, 257, KS, 5), chunk=True, lw=True)


@pytest.mark.parametrize("Hsb,L", MMA_H)
def test_step_chunk_mma_rows(built_lib, Hsb, L):
    m, params, cfg, p = _model(F=65, Hfb=96, Hsb=Hsb, L=L, impl="mma", fast=Hsb != 384, seed=Hsb)
    rows = built_lib.fsn_lstm_mma_rows(L, Hsb, 16, 2)
    _run_slots(f"chunk mma R={rows} H={Hsb} L={L}", m, cfg=cfg, p=_p(params, p), B=2, schedule=_staggered(2, 65, KS, 7), chunk=True)


def test_step_chunk_low_cap_windows(built_lib, monkeypatch):
    """FSN_WS_CAP_GB low enough that a 37-frame call runs one session at a time (sub-batches) in windows with k0 > 0"""
    m, params, cfg, p = _model(F=257, seed=11)
    cap, Tw = _window_cap(built_lib, m._cfg, 3, 37)
    m, params, cfg, p = _model(F=257, seed=11, monkeypatch=monkeypatch, env={"FSN_WS_CAP_GB": repr(cap / 1e9)})
    _run_slots(f"chunk lw cap windows Tw={Tw}", m, cfg=cfg, p=_p(params, p), B=3, schedule=_staggered(3, 257, [4, 37, 37, 5, 37], 13),
               chunk=True, lw=True)


def _window_cap(lib, cfg, n, K):
    """the largest cap (bytes, fsn_stream_chunk_plan) under which n sessions of a K-frame call run one at a time in windows of Tw < K
    frames, and that Tw"""
    import ctypes as C
    Bs, Tw, nb = C.c_int32(), C.c_int32(), C.c_int64()
    assert lib.fsn_stream_chunk_plan(C.byref(cfg), 1, K, 1e15, None, None, C.byref(nb)) == 0
    for f in np.linspace(0.99, 0.05, 95):
        cap = float(int(nb.value * f))
        assert lib.fsn_stream_chunk_plan(C.byref(cfg), n, K, cap, C.byref(Bs), C.byref(Tw), None) == 0
        if Bs.value == 1 and 0 < Tw.value < K:
            return cap, Tw.value
    raise AssertionError("no cap gives windows")


@pytest.mark.parametrize("Ns,Nf", WIDE)
@pytest.mark.parametrize("impl", ["mma", "auto"])
def test_step_chunk_wide(built_lib, Ns, Nf, impl):
    m, params, cfg, p = _model(F=129, Hfb=96, Hsb=128, Ns=Ns, Nf=Nf, impl=impl, seed=Ns + Nf)
    _run_slots(f"chunk wide Isb={2 * Ns + 2 * Nf + 2} {impl}", m, cfg=cfg, p=_p(params, p), B=2, schedule=_staggered(2, 129, KS, 17),
               chunk=True, lw=impl == "auto")


@pytest.mark.parametrize("no_ws", [False, True])
def test_step_full_band_paths(built_lib, monkeypatch, no_ws):
    """weight-stationary (B <= 64) and generic (FSN_NO_WS, and B = 80 > 64) full band; the handle's kernel (fsn_stream_fb_ws) must be
    the one ws_eligible (test_gpu_full_band.py) names"""
    import test_gpu_full_band as G
    env = {"FSN_NO_WS": "1"} if no_ws else None
    for B in ((4,) if no_ws else (4, 80)):
        m, params, cfg, p = _model(F=257, seed=B, monkeypatch=monkeypatch, env=env)
        ws = G.ws_eligible(2, 512, 257, B, G._num_sms()) and not no_ws
        _run_slots(f"full band {'ws' if ws else 'mma'} B={B}", m, cfg=cfg, p=_p(params, p), B=B,
                   schedule=_staggered(B, 257, [1, 4, 1, 3, 2], 19), chunk=True, check=sorted({0, 1, 63, 64, B - 1} & set(range(B))),
                   lw=True, ws=ws)


def test_step_edge_sessions(built_lib):
    """an all-zero opening (normaliser 1 / eps), x1e3 frames that reach the fp16 clamp of the sub-band input"""
    m, params, cfg, p = _model(F=257, seed=23)
    F = 257
    sched = [(4, {0: ("start", _clip(F, 30, 1, zero_open=6)), 1: ("start", _clip(F, 30, 2, scale=1e3))})]
    sched += [(K, {0: "step", 1: "step"}) for K in (1, 3, 8, 16)]
    _run_slots("edge zero opening / x1e3", m, cfg=cfg, p=_p(params, p), B=2, schedule=sched, chunk=True, lw=True)


def test_step_long_session(built_lib):
    """the 30 s config #4 clip (1876 frames) in 32-frame calls, checked at its last calls"""
    m, params, cfg, p = _model(F=257, seed=29)
    F = 257
    clip = np.abs(O.stft(O.synth_clips(1, num_samples=256 * (LONG_T - 1), seed0=7))[0]).astype(np.float32)
    n = -(-(LONG_T + 2) // LONG_K)
    sched = [(LONG_K, {0: ("start", clip)})] + [(LONG_K, {0: "step"})] * (n - 1)
    _run_slots("long session 1876 frames", m, cfg=cfg, p=_p(params, p), B=1, schedule=sched, chunk=True, check_from=n - 3, lw=True)


# ---- the audio calls: the analysis, then the model stages from the kernels' own magnitude frames ----------------------------------
AUDIO_FACTOR = 1.0                                                                    # the STFT's rule factor (the radix-2 fp32 FFT)


class AudioSess(Sess):
    """an audio session: its samples so far, its slot ticks t and hop count Kh (0 before its FLUSH), as the handle counts them"""
    def __init__(self, F, seed):
        super().__init__(np.zeros((F, 0), np.float32))
        self.rng, self.x, self.t, self.Kh = np.random.default_rng(seed), np.zeros(0, np.float32), 0, 0

    def hops(self, n, hop):
        new = (self.rng.standard_normal(n * hop) * 0.1).astype(np.float32)
        self.x = np.concatenate([self.x, new])
        return new


def _audio_plan(s, flag, n, K, la):
    """fsn_api.cu audio_slot_plan restated: (k0, na, start, Kh after the call)"""
    from fsnplus_b200.streaming import FLUSH, START, STEP
    if flag == START:
        return 0, n, 1, 0
    if flag == STEP:
        return s.t, n, 0, 0
    assert flag == FLUSH
    Kh = s.Kh or (s.t + n if n < K else 0)
    left = Kh + la + 2 - s.t if Kh else n
    return s.t, min(max(left, 0), K), 0, Kh


def _run_audio(label, m, p, cfg, B, schedule, chunk, lw):
    """schedule: [(K, {slot: (flag, hops)}), ...] (slots not listed HOLD, fed NaN).  Per call and stepping slot: "mag" against the fp64
    STFT of the session's samples, then every model stage as in _run_slots from that magnitude; the mask columns of the call's ticks
    outside its model frames, fb_in past the slot's kf and held slots' rows must be exactly 0, held slots' payloads unchanged."""
    from fsnplus_b200.streaming import HOLD, START, StreamingFullSubNet
    F, la = cfg["num_freqs"], p["la"]
    hop = F - 1
    st = StreamingFullSubNet(m, B, DEV)
    sess = {}
    for ci, (K, acts) in enumerate(schedule):
        flags, nh = np.full(B, HOLD, np.int32), np.zeros(B, np.int32)
        x = np.full((B, K * hop), np.nan, np.float32)
        plan = {}
        for b, (flag, n) in acts.items():
            if flag == START:
                sess[b] = AudioSess(F, 100 * ci + b)
            flags[b], nh[b] = flag, n
            plan[b] = _audio_plan(sess[b], flag, n, K, la)
            x[b, :n * hop] = sess[b].hops(n, hop)
        before = st.save_slots(list(range(B))).payload.cpu().numpy() if ci else None
        if chunk:
            _, _, mask = st.step_audio_chunk(_t(x), torch.from_numpy(flags), torch.from_numpy(nh), return_mask=True)
        else:
            assert K == 1
            _, _, mask = st.step_audio(_t(x[:, :hop]), torch.from_numpy(flags), return_mask=True)
            mask = mask[..., None]
        mask = mask.cpu().numpy()
        kf = {b: max(na - start, 0) for b, (k0, na, start, _) in plan.items()}
        Km = max(kf.values(), default=0)
        after = st.save_slots(list(range(B))).payload.cpu().numpy()
        if Km:
            mag = st.get_stage("mag", (B, F, Km)).cpu().numpy()
            fb_in = st.get_stage("fb_in", (B, F, Km)).cpu().numpy()
            fb_out = st.get_stage("fb_out", (B, F, Km)).cpu().numpy()
            assert _layerwise(st) == (lw and chunk), (label, "sub-band route")
            img = None if lw and chunk else _img(st, m, cfg, Km)
        for b in range(B):
            if b not in plan or not kf[b]:
                if b not in plan and before is not None:
                    assert np.array_equal(before[b], after[b]), (label, ci, b, "a held slot's state changed")
                assert not np.any(mask[b]), (label, ci, b, "the mask row of a slot without model frames is not zero")
                if b in plan:
                    s = sess[b]
                    s.t, s.Kh = plan[b][0] + plan[b][1], plan[b][3]
                continue
            s, (k0, na, start, Kh) = sess[b], plan[b]
            s.Kh, n, j0 = Kh, kf[b], k0 + start - 1
            lab = f"{label} call {ci} slot {b} K={K} kf={n}"
            L = Kh * hop
            _check("stft mag", lab, mag[b][:, :n], S.stft_mag_truth(s.x, j0, n, hop, L), S.stft_mag_emulate(s.x, j0, n, hop, L),
                   AUDIO_FACTOR)
            assert not np.any(fb_in[b][:, n:]), (lab, "fb_in past the slot's frames is not zero")
            cols = np.arange(K)
            own = (cols >= start) & (cols < start + n)
            assert not np.any(mask[b][..., ~own]), (lab, "mask columns outside the slot's model frames are not zero")
            s.mag.append(mag[b][:, :n])
            s.fb.append(fb_out[b][:, :n])
            s.n += n
            _check_slot(lab, p, F, s, n, fb_in[b][:, :n], fb_out[b][:, :n], None if img is None else img[b * F:(b + 1) * F, :, :n],
                        mask[b][..., start:start + n], _slot_state(np.zeros_like(after[b]) if j0 == 0 else before[b], p, F),
                        _slot_state(after[b], p, F), lw and chunk)
            s.t = k0 + na


def test_audio_per_hop(built_lib):
    """the per-hop audio call: staggered STARTs, a mid-session HOLD, a FLUSH (frame K's right reflect, then zero frames)"""
    from fsnplus_b200.streaming import FLUSH, START, STEP
    m, params, cfg, p = _model(F=65, Hfb=96, Hsb=64, impl="mma", seed=41)
    sched = []
    for t in range(12):
        acts = {0: (START if t == 0 else FLUSH if t >= 6 else STEP, 1 if t < 6 else 0)}
        if t >= 2 and t != 5:
            acts[1] = (START if t == 2 else STEP, 1)
        if t < 9:
            acts[2] = (START if t == 0 else STEP, 1)
        sched.append((1, acts))
    _run_audio("audio per hop", m, _p(params, p), cfg, 3, sched, chunk=False, lw=False)


@pytest.mark.parametrize("impl", ["auto", "mma"])
def test_audio_chunk(built_lib, impl):
    """the audio chunk call with per-slot hop counts (kf < K): a START of 3 hops, STEPs of 8 / 5 / 1, a FLUSH of 2 hops that runs the
    look-ahead flush in the next calls, a held slot"""
    from fsnplus_b200.streaming import FLUSH, START, STEP
    m, params, cfg, p = _model(F=257, impl=impl, seed=43)
    sched = [(8, {0: (START, 8), 1: (START, 3)}),
             (8, {0: (STEP, 5), 1: (STEP, 8), 2: (START, 8)}),
             (8, {0: (STEP, 1), 1: (FLUSH, 2), 2: (STEP, 7)}),
             (8, {0: (STEP, 8), 1: (FLUSH, 0)}),
             (8, {0: (FLUSH, 3), 2: (STEP, 2)}),
             (8, {0: (FLUSH, 0), 2: (STEP, 8)})]
    _run_audio(f"audio chunk {impl}", m, _p(params, p), cfg, 3, sched, chunk=True, lw=impl == "auto")


# ---- the lockstep call: hook and masks only, from zero state over the whole session -----------------------------------------------
@pytest.mark.parametrize("kind,norm", [("LSTM", "cumulative_laplace_norm"), ("GRU", "cumulative_layer_norm")])
def test_lockstep_step(built_lib, kind, norm):
    from fsnplus_b200.streaming import StreamingFullSubNet
    F, B, T = 65, 3, 24
    m, params, cfg, p = _model(F=F, Hfb=96, Hsb=64, kind=kind, norm=norm, seed=31)
    p = _p(params, p)
    st = StreamingFullSubNet(m, B, DEV)
    clips = [_clip(F, T, 40 + b) for b in range(B)]
    fb_in, fb_out, img, mask = [], [], [], []
    for t in range(T):
        out = st.step(_t(np.stack([c[:, t] for c in clips])))
        fb_in.append(st.get_stage("fb_in", (B, F, 1)).cpu().numpy())
        fb_out.append(st.get_stage("fb_out", (B, F, 1)).cpu().numpy())
        img.append(_img(st, m, cfg, 1))
        mask.append(None if out is None else out.cpu().numpy()[..., None])
    fb_in, fb_out, img = (np.concatenate(v, axis=-1) for v in (fb_in, fb_out, img))
    label = f"lockstep {kind} {norm[11:]}"
    zero = np.zeros((p["L"], 1, p["Hfb"]))
    for b in range(B):
        xs = clips[b].astype(np.float64)
        _check("norm", label, fb_in[b], S.norm_truth(xs, norm), S.norm_emulate(xs, norm), 1.0)
        _rnn_check(label, "full band", p, "fb_model", "fb", fb_in[b][None], (zero, zero), T, fb_out[b][None], None, p["fast"])
        _check("sub-band input", label, img[b * F:(b + 1) * F], S.sb_truth(xs, fb_out[b], p["Ns"], p["Nf"], norm),
               S.sb_emulate(xs, fb_out[b], p["Ns"], p["Nf"], norm), 1.0)
    la = p["la"]
    assert sum(mk is not None for mk in mask) == T - la
    got = np.concatenate([np.zeros((B, 2, F, la), np.float32)] + [mk for mk in mask if mk is not None], axis=-1)   # step t: frame t - la
    zs = np.zeros((p["L"], B * F, p["Hsb"]))
    _rnn_check(label, "sub band", p, "sb_model", "sb", img, (zs, zs), T, torch.as_tensor(got).permute(0, 2, 1, 3).reshape(B * F, 2, -1),
               None, p["fast"], cols=slice(la, T))
    # saved at the end only: the final states against the same fp64 runs
    pl = st.save_slots(list(range(B))).payload.cpu().numpy()
    for b in range(B):
        d = S.decode(pl[b], F, p["L"], p["Hfb"], p["Hsb"])
        _sums_ok(label + " cum_in", d["cum_in"], clips[b].astype(np.float64).reshape(1, -1))


# ---- the hook's refusals -----------------------------------------------------------------------------------------------------------------
def test_get_stage_refusals(built_lib):
    import ctypes as C
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import HOLD, START, StreamingFullSubNet
    F, B = 65, 2
    m, params, cfg, p = _model(F=F, Hfb=96, Hsb=64, seed=37)
    lib = _lib.load_library()
    st = StreamingFullSubNet(m, B, DEV)
    buf = torch.zeros(B * F * 64, device=DEV)

    def call(name, numel, h=st._st, dst=buf):
        return lib.fsn_stream_get_stage(h, name if name is None else name.encode(), C.c_void_p(None if dst is None else dst.data_ptr()),
                                        numel, None)

    assert call("fb_in", B * F) == -3 and "no step" in lib.fsn_last_error().decode()         # FSN_ESTATE before any step
    st.step_chunk(_t(np.ones((B, F, 4), np.float32)), [START, START])
    assert call("fb_in", B * F * 4) == 0
    assert call("fb_in", B * F) == -1 and str(B * F * 4) in lib.fsn_last_error().decode()     # wrong numel: names the count
    assert call("bogus", B * F * 4) == -1 and "unknown" in lib.fsn_last_error().decode()
    assert call(None, B * F * 4) == -1 and call("fb_in", B * F * 4, dst=None) == -1 and call("fb_in", B * F * 4, h=None) == -1
    assert call("sb_img", 1) == -3 and "layer-wise" in lib.fsn_last_error().decode()          # layer-wise chunk call
    assert call("mag", B * F * 4) == -3 and "audio" in lib.fsn_last_error().decode()          # mask mode
    a = StreamingFullSubNet(m, B, DEV)
    hop = a.hop
    a.step_audio_chunk(_t(np.zeros((B, 2 * hop), np.float32)), [START, HOLD], [2, 0])
    assert lib.fsn_stream_get_stage(a._st, b"mag", C.c_void_p(buf.data_ptr()), B * F * 1, None) == 0
    a.step_audio_chunk(_t(np.zeros((B, 2 * hop), np.float32)), [HOLD, HOLD], [0, 0])         # no model step
    assert lib.fsn_stream_get_stage(a._st, b"mag", C.c_void_p(buf.data_ptr()), B * F * 1, None) == -3


def test_zz_worst_per_stage(built_lib):
    """The table DESIGN.md §2 quotes: the worst max err / RMS per stage."""
    if not WORST:
        pytest.skip("no case of this file ran before")
    print("\nworst max err / RMS per stage (ratio to the emulation's error, case):")
    for key in sorted(WORST):
        e, ratio, label = WORST[key]
        print(f"  {key:22s} {e:.2e} ({ratio:.2f}x, {label})")
