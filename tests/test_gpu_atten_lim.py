"""Attenuation limits (DESIGN.md §3.18) on every enhancement path: fsn_model_forward_enhance_lim, fsn_model_enhance_audio_lim, the
streaming audio calls (fsn_stream_set_atten_lim) and overlapped-chunk sessions (fsn_chunk_stream_set_atten_lim).

  * bit identity: clips and slots at +inf are the bits of the unlimited call, and a null array is the existing entry point;
  * the floor |Y| >= lam |X| in every bin, and the limited spectrum against an fp64 restatement of M' applied to the same call's own mask
    (fsn_model_forward on the same planes) and noisy spectrum, bin by bin -- on FullSubNet+ with the layer-wise LSTM, lstm_impl = "mma",
    the GRU and the sub-band TCN, and on fullsubnet.Model; under sub-batches, sub-band windows, TCN bin chunks and ragged frame counts;
  * the audio call against the fp64 iSTFT of the limited spectrum built from its own "stft" planes and the model's mask;
  * live sessions: +inf slots bit-identical, limited sessions against the offline limited call, masks and saved payloads unchanged, a
    limit changed mid-session leaving every earlier hop as it was; chunk sessions against the overlapped-chunk restatement;
  * every refusal, which changes no state."""
import ctypes as C

import numpy as np
import pytest
import torch

import chunk_stream_ref as R
import sbtcn_oracle as S
from oracle import fsn_oracle as O
from test_gpu_chunk_stream import STITCH_TOL, _bank, _drive as _chunk_drive, _schedule
from test_gpu_stream_audio_chunks import KS, WAVE_TOL, Session, _plan
from test_gpu_stream_audio import _clips
from test_gpu_stream_chunks import _fsn
from test_gpu_stream_sessions import _small_cfg

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
INF = float("inf")
LIMS = [INF, 0.0, 6.0, 20.0, INF, 12.0, 3.0, 40.0]      # one batch mixing +inf, 0 dB and finite limits
MASK_ABS = 2e-5           # fp32 decompress_cIRM and the product vs fp64, in mask units times |X|
AUDIO_TOL = 1e-4          # a limited waveform vs the fp64 iSTFT of the fp64-limited spectrum it was built from


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _floor(db):
    return np.float64(np.float32(10.0 ** (-db / 20.0)))


def _limited(crm, X, lams):
    """fp64: decompress_cIRM of crm [B, 2, F, T], M' per clip floor lams[b], times X [B, F, T]; also |M| and the floors [B, 1, 1]."""
    m = O.decompress_cIRM(crm.astype(np.float64))
    m0, m1 = m[:, 0], m[:, 1]
    a = np.hypot(m0, m1)
    lam = np.asarray(lams, np.float64)[:, None, None]
    low = a < lam
    s = np.where(low & (a > 0), lam / np.where(a > 0, a, 1.0), 1.0)
    m0, m1 = m0 * s, m1 * s
    m0 = np.where(low & (a == 0), lam, m0)
    Y = (m0 * X.real - m1 * X.imag) + 1j * (m1 * X.real + m0 * X.imag)
    return Y, a, lam, np.hypot(m0, m1)


def _build(kind, monkeypatch=None, env=None):
    from fsnplus_b200.model import FullSubNet_Plus
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    base = dict(num_freqs=129, sb_num_neighbors=7, sb_model_hidden_size=64)
    if kind == "fsn":
        cfg = O.default_fsn_config()
        cfg.update(num_freqs=129, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=128)
        m = _fsn(cfg, O.make_params_fsn(cfg, seed=21))
    else:
        cfg = O.default_plus_config()
        cfg.update(base)
        kw = {}
        if kind == "gru":
            cfg.update(sequence_model="GRU")
        if kind == "tcn":
            cfg.update(sequence_model="TCN", sb_model_hidden_size=32)
            params = S.make_params(cfg, seed=22)
        else:
            params = O.make_params_plus(cfg, seed=23)
        if kind == "mma":
            kw["lstm_impl"] = "mma"
        m = FullSubNet_Plus(**cfg, **kw)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
        m = m.to(DEV).eval()
        with torch.cuda.device(DEV):
            m._ensure_handle(torch.device(DEV))
    for k in (env or {}):
        monkeypatch.delenv(k, raising=False)
    return m, cfg


def _spectra(B, F, T, seed):
    n_fft, hop = 2 * (F - 1), F - 1
    x = O.synth_clips(B, num_samples=(T - 1) * hop, seed0=seed)
    X = O.stft(x.astype(np.float64), n_fft, hop, n_fft).astype(np.complex64)
    assert X.shape == (B, F, T)
    return X


def _check_spectrum(m, X, frames, lims, what):
    """The limited call on planes X against the unlimited call and the fp64 restatement over the same call's mask."""
    B, F, T = X.shape
    mag, re, im = (_t(v[:, None].astype(np.float32)) for v in (np.abs(X), X.real, X.imag))
    with torch.no_grad():
        base = m.enhance_spectrum(mag, re, im, frames=frames).cpu().numpy()
        n_base = m.last_launch_count()
        got = m.enhance_spectrum(mag, re, im, frames=frames, atten_lim_db=lims).cpu().numpy()
        n_got = m.last_launch_count()
        crm = (m(mag, re, im, frames=frames) if m._cfg.model_kind == 0 else m(mag, frames=frames)).cpu().numpy()
    assert n_got == n_base, (what, n_got, n_base)
    fr = frames or [T] * B
    Xd = X.astype(np.complex128)
    Y, a, lam, amp = _limited(crm, Xd, [_floor(v) for v in lims])
    worst, excl = 0.0, 0
    for b in range(B):
        n = fr[b]
        assert not got[b, :, n:].any(), (what, b)
        if lims[b] == INF:
            assert np.array_equal(got[b], base[b]), (what, b, "an unlimited clip differs from the unlimited call")
            continue
        g, y, x = got[b, :, :n].astype(np.complex128), Y[b, :, :n], np.abs(Xd[b, :, :n])
        assert (np.abs(g) >= lam[b] * x * (1 - 1e-5)).all(), (what, b, "floor")
        near = np.abs(a[b, :, :n] - lam[b]) <= MASK_ABS * (1 + lam[b])
        # a raised mask keeps M's direction: the fp32 mask's error grows by lam / |M| with it
        gain = np.maximum(1.0, lam[b] / np.maximum(a[b, :, :n], 1e-30))
        err = np.abs(g - y) / (x * (1 + amp[b, :, :n]) * gain + 1e-30)
        bad = (err > MASK_ABS) & ~near
        assert not bad.any(), (what, b, float(err[~near].max()))
        worst = max(worst, float(err[~near].max()))
        excl += int(near.sum())
        if lims[b] == 0.0:
            assert (np.abs(g) >= x * (1 - 1e-5)).all()
    print(f"\n[{what}] worst |Y - Y64| / (|X| (1 + |M'|)) {worst:.2e}, {excl} bins within rounding of lam excluded; launches {n_got}")
    return got


VARIANTS = ["lstm", "mma", "gru", "tcn", "fsn"]


@pytest.mark.parametrize("kind", VARIANTS)
def test_spectrum_floor_and_identity(built_lib, kind):
    from fsnplus_b200 import _lib
    m, cfg = _build(kind)
    F, T = cfg["num_freqs"], 96
    X = _spectra(8, F, T, seed=31)
    _check_spectrum(m, X, None, LIMS, f"{kind} whole")
    assert m.last_lstm_impl() == {"lstm": "tcgen05", "mma": "mma", "gru": "tcgen05", "tcn": "tcn", "fsn": "tcgen05"}[kind]
    _check_spectrum(m, X, [96, 37, 96, 64, 90, 96, 51, 77], LIMS, f"{kind} ragged")
    # a null array and all-+inf limits are the existing entry point, bit for bit and launch for launch
    mag, re, im = (_t(v[:, None].astype(np.float32)) for v in (np.abs(X), X.real, X.imag))
    lib = _lib.load_library()
    with torch.no_grad():
        want = m.enhance_spectrum(mag, re, im)
        n_want = m.last_launch_count()
        out = torch.empty_like(want)
        stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
        p = lambda x: C.c_void_p(x.data_ptr())
        _lib.check(lib.fsn_model_forward_enhance_lim(m._handle, p(mag), p(re), p(im), 8, T, None, None, p(out), stream))
        assert torch.equal(out, want) and m.last_launch_count() == n_want
        out2 = m.enhance_spectrum(mag, re, im, atten_lim_db=INF)
        assert torch.equal(out2, want) and m.last_launch_count() == n_want


SPLITS = [("lstm", {"FSN_WS_CAP_GB": "0.02"}), ("lstm", {"FSN_SB_WINDOW": "32"}), ("mma", {"FSN_WS_CAP_GB": "0.02"}),
          ("tcn", {"FSN_SB_CHUNK": "7"}), ("tcn", {"FSN_WS_CAP_GB": "0.02"}), ("fsn", {"FSN_WS_CAP_GB": "0.02"})]


@pytest.mark.parametrize("kind,env", SPLITS, ids=[f"{k}-{'-'.join(f'{a}={b}' for a, b in e.items())}" for k, e in SPLITS])
def test_spectrum_under_splits(built_lib, monkeypatch, kind, env):
    """Every clip gets its own floor in every sub-batch, window and bin chunk: the same checks as unsplit, and the same bits."""
    m, cfg = _build(kind, monkeypatch, env)
    whole, _ = _build(kind)
    F, T = cfg["num_freqs"], 160
    X = _spectra(8, F, T, seed=32)
    frames = [160, 41, 160, 99, 130, 160, 64, 111]
    got = _check_spectrum(m, X, frames, LIMS, f"{kind} {env}")
    Bs, Tw, Fc = m.last_plan_bins()
    assert Bs < 8 or Tw or Fc, (Bs, Tw, Fc)
    mag, re, im = (_t(v[:, None].astype(np.float32)) for v in (np.abs(X), X.real, X.imag))
    with torch.no_grad():
        ref = whole.enhance_spectrum(mag, re, im, frames=frames, atten_lim_db=LIMS).cpu().numpy()
    print(f"plan Bs {Bs} Tw {Tw} Fc {Fc}; max |split - whole| {np.abs(got - ref).max():.2e}")
    if kind != "fsn" or "FSN_WS_CAP_GB" not in env:
        assert np.abs(got - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("kind", VARIANTS)
def test_audio_against_fp64(built_lib, kind):
    from fsnplus_b200.model import FullSubNet_Plus  # noqa: F401
    m, cfg = _build(kind)
    F = cfg["num_freqs"]
    n_fft, hop = 2 * (F - 1), F - 1
    lengths = [12000, 7001, 12000, 9 * hop + 3, 11111, 5000, 12000, 8192]
    x = O.synth_clips(8, num_samples=12000, seed0=41)
    rows = np.full((8, 12000), np.nan, np.float32)
    for b, n in enumerate(lengths):
        rows[b, :n] = x[b, :n]
    with torch.no_grad():
        base = m.enhance_audio(_t(rows), lengths).cpu().numpy()
        n_base = m.last_launch_count()
        got = m.enhance_audio(_t(rows), lengths, atten_lim_db=LIMS).cpu().numpy()
        assert m.last_launch_count() == n_base
        T = max(lengths) // hop + 1
        planes = m.get_stage("stft", (3, 8, 1, F, T), torch.device(DEV))
        frames = [n // hop + 1 for n in lengths]
        crm = (m(planes[0], planes[1], planes[2], frames=frames) if m._cfg.model_kind == 0 else m(planes[0], frames=frames)).cpu().numpy()
    planes = planes.cpu().numpy().astype(np.float64)
    Xd = planes[1, :, 0] + 1j * planes[2, :, 0]
    Y = _limited(crm, Xd, [_floor(v) for v in LIMS])[0]
    worst = 0.0
    for b, n in enumerate(lengths):
        assert not got[b, n:].any()
        if LIMS[b] == INF:
            assert np.array_equal(got[b], base[b]), b
            continue
        ref = O.istft(Y[b:b + 1, :, :frames[b]], n_fft, hop, n_fft, length=n)[0]
        e = O.rel_l2(got[b, :n], ref)
        worst = max(worst, e)
        assert e <= AUDIO_TOL, (b, e)
        if LIMS[b] == 0.0:
            assert O.rel_l2(got[b, :n], base[b, :n]) > 1e-3        # 0 dB: no bin attenuated, so not the unlimited output
    print(f"\n[{kind} audio] worst rel-L2 vs fp64 iSTFT of the limited spectrum {worst:.2e}")


# ---- live sessions ---------------------------------------------------------------------------------------------------------------
def _stream_model():
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    params = O.make_params_fsn(cfg, seed=51)
    return _fsn(cfg, params), cfg


def _sessions(hop):
    A, B_, Cc, D, E, G = _clips(6, [30, 61, 45, 26, 40, 33], hop, seed0=910, gains=[8.0, 1.0, 1.0, 0.05, 1.0, 2.0])
    return [Session(0, 0, A, hop, seed=1), Session(1, 1, B_, hop, holds=(3, 4, 9), extra=1, seed=2),
            Session(2, 3, Cc, hop, holds=(6,), seed=3), Session(0, 9, D, hop, holds=(11,), extra=2, seed=4),
            Session(3, 2, E, hop, seed=5), Session(2, 14, G, hop, seed=6)]


SLOT_DB = [INF, 12.0, 6.0, 0.0]


def _tail_offset(c, la):
    """Byte offset of the overlap tail in an audio-mode payload (include/fsnplus_b200.h: the segments in order, 16-byte aligned)."""
    F, hop, L = c.num_freqs, c.num_freqs - 1, c.num_layers
    o = 0
    for size in (16, F * 16, L * c.fb_hidden * 2, L * c.fb_hidden * 4, L * F * c.sb_hidden * 2, L * F * c.sb_hidden * 4,
                 3 * hop * 4, (la + 1) * F * 8):
        o += (size + 15) // 16 * 16
    return o


def _run(st, sessions, la, per_hop, before=None, save_at=None):
    """The schedule of test_gpu_stream_audio_chunks through chunk calls or their per-hop expansion, with before(c) ahead of call c.
    Returns each session's waveform, the calls' (out, nout, mask) and the payload of every slot saved after call save_at."""
    from test_gpu_stream_audio_chunks import expand
    from fsnplus_b200.streaming import HOLD, START, STEP
    calls = _plan(sessions, KS, la)
    B, hop = st.B, st.hop
    wav, res, saved = [[] for _ in sessions], [], None
    for c, K in enumerate(KS):
        if before:
            before(c)
        flags, hops = np.full(B, HOLD, np.int32), np.zeros(B, np.int32)
        x = np.full((B, K * hop), np.nan, np.float32)
        for slot, (i, f, q, n) in calls[c].items():
            flags[slot], hops[slot] = f, n
            x[slot, :n * hop] = sessions[i].x[q * hop:(q + n) * hop]
        if per_hop:
            out, nout, mask = torch.zeros((B, K * hop)), torch.zeros(B, dtype=torch.int32), torch.zeros((B, 2, st.F, K))
            ticks = [expand(int(flags[b]), int(hops[b]), K) for b in range(B)]
            for k in range(K):
                fk = np.array([ticks[b][k] for b in range(B)], np.int32)
                xk = np.full((B, hop), np.nan, np.float32)
                for b in range(B):
                    if fk[b] in (START, STEP):
                        xk[b] = x[b, k * hop:(k + 1) * hop]
                o, v, mk = st.step_audio(_t(xk), torch.from_numpy(fk), return_mask=True)
                o, mk = o.cpu(), mk.cpu()
                for b in np.nonzero(v.numpy())[0]:
                    out[b, nout[b] * hop:(nout[b] + 1) * hop] = o[b]
                    nout[b] += 1
                mask[..., k] = mk
        else:
            out, nout, mask = st.step_audio_chunk(_t(x), torch.from_numpy(flags), torch.from_numpy(hops), return_mask=True)
            out, mask = out.cpu(), mask.cpu()
        res.append((out, nout.clone(), mask))
        for slot, (i, f, q, n) in calls[c].items():
            wav[i].append(out[slot, :int(nout[slot]) * hop])
        if c == save_at:
            saved = st.save_slots(list(range(B))).payload.cpu()
    return [torch.cat(w).numpy() for w in wav], res, saved


@pytest.mark.parametrize("per_hop", [False, True], ids=["chunk", "per_hop"])
def test_stream_slots(built_lib, per_hop):
    from fsnplus_b200.streaming import StreamingFullSubNet
    m, cfg = _stream_model()
    la = cfg["look_ahead"]
    st0 = StreamingFullSubNet(m, batch_size=4, device=DEV)
    hop = st0.hop
    want, wres, wsaved = _run(st0, _sessions(hop), la, per_hop, save_at=10)    # a schedule consumes its sessions' seeded draws
    st0.close()
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    st.set_atten_lim([0, 1, 2, 3], SLOT_DB)
    sessions = _sessions(hop)
    got, gres, gsaved = _run(st, sessions, la, per_hop, save_at=10)
    st.close()
    # the saved sessions: the same layout, and the same bytes up to the overlap tail -- a limited slot's tail is its limited synthesis
    assert gsaved.shape == wsaved.shape
    t0 = _tail_offset(m._cfg, la)
    for b, db in enumerate(SLOT_DB):
        assert torch.equal(gsaved[b, :t0], wsaved[b, :t0]), b
        if db == INF:
            assert torch.equal(gsaved[b], wsaved[b]), b
    for (o, n, mk), (o2, n2, mk2) in zip(gres, wres):
        assert torch.equal(n, n2) and torch.equal(mk, mk2), "the limit changed the hop counts or the masks"
    worst = 0.0
    for i, s in enumerate(sessions):
        db = SLOT_DB[s.slot]
        if db == INF:
            assert np.array_equal(got[i], want[i]), i
            continue
        with torch.no_grad():
            off = m.enhance_audio(_t(s.x[None]), atten_lim_db=db)[0].cpu().numpy()
        e = O.rel_l2(got[i], off)
        worst = max(worst, e)
        assert e < WAVE_TOL, (i, s.slot, e)
    print(f"\n[stream {'per-hop' if per_hop else 'chunk'}] limited sessions vs offline enhance_audio_lim: worst {worst:.2e}")


def test_stream_limit_changed_mid_session(built_lib):
    """A limit set before call 8 leaves every hop emitted before it bit-identical; afterwards the slot's hops differ."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    m, cfg = _stream_model()
    la = cfg["look_ahead"]
    st0 = StreamingFullSubNet(m, batch_size=4, device=DEV)
    _, wres, _ = _run(st0, _sessions(st0.hop), la, False)
    st0.close()
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    _, gres, _ = _run(st, _sessions(st.hop), la, False, before=lambda c: c == 8 and st.set_atten_lim([1], 6.0))
    st.close()
    for c, ((o, n, _), (o2, n2, _)) in enumerate(zip(gres, wres)):
        if c < 8:
            assert torch.equal(o, o2), c
        else:
            assert torch.equal(o[[0, 2, 3]], o2[[0, 2, 3]]), c
    assert any(not torch.equal(o[1], o2[1]) for (o, _, _), (o2, _, _) in zip(gres[8:], wres[8:]))


@pytest.mark.parametrize("kind", ["plus", "tcn"])
def test_chunk_sessions(built_lib, kind):
    from test_gpu_chunk_stream import _build as chunk_build
    from fsnplus_b200.streaming import ChunkStream
    m, cfg, _, _ = chunk_build(kind)
    C_, B = 512, 12
    H = C_ // 2
    sched = _schedule(B, H, 30, seed=61, S_choices=[1, 37, 160, 320, 700], special=(1, H, 2 * H, 3 * H))
    cs0 = ChunkStream(m, B, C_, DEV)
    want = _chunk_drive(cs0, sched, _bank(7), seed=62)
    cs0.close()
    dbs = [INF if b % 3 == 0 else [12.0, 3.0][b % 2] for b in range(B)]
    cs = ChunkStream(m, B, C_, DEV)
    cs.set_atten_lim(list(range(B)), dbs)
    got = _chunk_drive(cs, sched, _bank(7), seed=62)
    cs.close()
    assert len(got) == len(want)
    worst = 0.0
    for s, w in zip(got, want):
        db = dbs[s["slot"]]
        if db == INF:
            assert np.array_equal(s["y"], w["y"]), s["slot"]
            continue

        def enhance(rows, db=db):
            with torch.no_grad():
                return m.enhance_audio(_t(rows), atten_lim_db=db).cpu().numpy()
        want_y = R.chunk_stream_ref(s["x"], C_, enhance)[:s["y"].shape[0]]
        if s["y"].size and np.abs(want_y).max() > 0:
            e = O.rel_l2(s["y"], want_y)
            worst = max(worst, e)
            assert e <= STITCH_TOL, (s["slot"], e)
    print(f"\n[chunk {kind}] limited sessions vs the overlapped-chunk restatement over enhance_audio_lim: worst {worst:.2e}")


# ---- refusals --------------------------------------------------------------------------------------------------------------------
def test_errors_change_nothing(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200._lib import FsnError
    from fsnplus_b200.streaming import ChunkStream, StreamingFullSubNet
    lib = _lib.load_library()
    m, cfg = _build("lstm")
    F = cfg["num_freqs"]
    X = _spectra(3, F, 64, seed=71)
    mag, re, im = (_t(v[:, None].astype(np.float32)) for v in (np.abs(X), X.real, X.imag))
    rows = _t(O.synth_clips(3, num_samples=8000, seed0=72).astype(np.float32))
    with torch.no_grad():
        for bad, msg in ((-1.0, r"clip 2: h_atten_db\[2\] = -1"), (float("nan"), r"clip 2: h_atten_db\[2\] = nan")):
            with pytest.raises(FsnError, match=msg):
                m.enhance_audio(rows, atten_lim_db=[0.0, INF, bad])
            with pytest.raises(FsnError, match=msg):
                m.enhance_spectrum(mag, re, im, atten_lim_db=[0.0, INF, bad])
        with pytest.raises(ValueError, match="pipelined"):
            m.enhance_spectrum(mag, re, im, pipelined=True, atten_lim_db=6.0)
        with pytest.raises(ValueError, match="entries"):
            m.enhance_audio(rows, atten_lim_db=[1.0, 2.0])

    sm, scfg = _stream_model()
    for make, setter in ((lambda: StreamingFullSubNet(sm, batch_size=4, device=DEV), "fsn_stream_set_atten_lim"),
                         (lambda: ChunkStream(sm, 4, 512, DEV), "fsn_chunk_stream_set_atten_lim")):
        h = make()
        raw = h._st if hasattr(h, "_st") else h._cs
        fn = getattr(lib, setter)
        one = (C.c_int32 * 1)(0)
        val = (C.c_float * 1)(6.0)
        assert fn(raw, 1, None, val) == -1 and b"h_slots is null" in lib.fsn_last_error()
        assert fn(raw, 1, one, None) == -1 and b"h_atten_db is null" in lib.fsn_last_error()
        assert fn(raw, 0, one, val) == -1 and b"n = 0" in lib.fsn_last_error()
        cases = [([4], [6.0], r"h_slots\[0\] = 4 is out of range"), ([1, 1], [6.0, 6.0], r"slot 1 is named twice"),
                 ([0, 2], [6.0, -3.0], r"slot 2: h_atten_db\[1\] = -3"), ([0, 3], [6.0, float("nan")], r"slot 3: h_atten_db\[1\] = nan")]
        for slots, dbs, msg in cases:
            with pytest.raises(FsnError, match=msg):
                h.set_atten_lim(slots, dbs)
        h.close()
    # a failed call changes no state: slot 0 is still unlimited (bit-identical to a handle that never saw a limit)
    hop = scfg["num_freqs"] - 1
    x = _clips(1, [12], hop, seed0=73)[0]
    outs = []
    for fail in (False, True):
        st = StreamingFullSubNet(sm, batch_size=4, device=DEV)
        if fail:
            with pytest.raises(FsnError):
                st.set_atten_lim([0, 2], [6.0, -1.0])
        xs = np.full((4, 12 * hop), np.nan, np.float32)
        xs[0] = x
        o, n = st.step_audio_chunk(_t(xs), [2, 0, 0, 0], [12, 0, 0, 0])
        outs.append(o.cpu())
        st.close()
    assert torch.equal(outs[0], outs[1])
