"""The audio transforms element by element against fp64 (audio_ref.py), each from the kernels' own input:

  * offline analysis: the "stft" planes of fsn_model_enhance_audio against the fp64 rfft of the input rows, each frame's errors over
    its windowed samples' norm, digital silence exactly 0, frames past T_b exactly 0; the magnitude plane against hypot of the kernel's
    own real / imaginary planes;
  * offline synthesis: the waveform against the fp64 iSTFT of the call's own "enh", each sample times its overlap-add envelope, samples
    past L_b exactly 0;
  * streaming synthesis (the per-hop audio call): every emitted hop of a session against the fp64 cIRM product and iSTFT of the masks
    and spectra the calls' "mask" / "spec" hooks return, and those spectra against the fp64 rfft of the session's samples;
  * the cIRM product: fsn_apply_cirm, and the generic kernel's apply_cirm_planar through fullsubnet.Model's enhance_spectrum, per element
    over |X| (|M| + 10);
  * a batch of more clips than the launch grids hold: sub-batched, bit-identical to the same clips in smaller calls.

The rule is sb_rnn_ref.compare with FACTOR.  One line per case; the last test prints the worst case per stage."""
import numpy as np
import pytest
import torch

import audio_ref as A
import sb_rnn_ref as R
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Measured once on one H100 80GB HBM3 SXM (700 W power limit): see DESIGN.md §2 for the worst err / bound of every stage.
FACTOR = 1.0
WORST = {}
HOLD, STEP, START, FLUSH = 0, 1, 2, 3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _check(stage, label, got, want, emu):
    r = R.compare(got, want, emu, FACTOR)
    q = r["err"] / r["bound"]
    if q >= WORST.get(stage, (-1.0, ""))[0]:
        WORST[stage] = (q, label, r["emu"] / max(r["bound"], 1e-300) * FACTOR)
    assert r["finite"] and r["ok"], (stage, label, r)
    return q


def _load(cls, cfg, params, **kw):
    m = cls(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    return m


def _fsn(F, seed, la=2, **kw):
    from fsnplus_b200.model import Model
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=F, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=96, look_ahead=la,
               norm_type="cumulative_laplace_norm")
    return _load(Model, cfg, O.make_params_fsn(cfg, seed=seed), **kw)


def _plus(seed, **over):
    from fsnplus_b200.model import FullSubNet_Plus
    cfg = O.default_plus_config()
    cfg.update(over)
    return _load(FullSubNet_Plus, cfg, O.make_params_plus(cfg, seed=seed))


# ---- offline --------------------------------------------------------------------------------------------------------------------------
def _offline(label, m, clips, L=None, atten=None):
    """One ragged call of the clips (rows NaN past each length, L samples long): both transforms of every clip"""
    F = m._cfg.num_freqs
    hop = F - 1
    lengths = [len(c) for c in clips]
    B, L = len(clips), L or max(lengths) + 77
    rows = np.full((B, L), np.nan, np.float32)
    for b, c in enumerate(clips):
        rows[b, :len(c)] = c
    with torch.no_grad():
        got = m.enhance_audio(_t(rows), lengths, atten_lim_db=atten).cpu().numpy()
    assert m.last_plan_bins()[0] == B                                   # one sub-batch: the stages are this call's
    T = max(lengths) // hop + 1
    planes = m.get_stage("stft", (3, B, 1, F, T), torch.device(DEV)).cpu().numpy()[:, :, 0]
    enh = torch.view_as_complex(m.get_stage("enh", (B, F, T, 2), torch.device(DEV))).cpu().numpy()
    qa = qs = 0.0
    for b, Lb in enumerate(lengths):
        Tb = Lb // hop + 1
        X, nrm = A.stft_truth(rows[b], Lb, hop)
        emu = A.stft_emulate(rows[b], Lb, hop)
        re, im = planes[1, b, :, :Tb], planes[2, b, :, :Tb]
        g, w, e, silent = A.stft_arrays(re, im, X, emu, nrm)
        assert silent == 0, (label, b, "digital silence analysed to nonzero")
        qa = max(qa, _check("offline stft", f"{label} clip {b} L={Lb}", g, w, e))
        assert not planes[:, b, :, Tb:].any(), (label, b)
        hyp = np.hypot(re, im, dtype=np.float32)
        assert np.all(np.abs(planes[0, b, :, :Tb] - hyp) <= 2.4e-7 * hyp), (label, b, "mag != hypot(re, im)")
        y, ye = A.istft_truth(enh[b], Lb, hop), A.istft_emulate(enh[b], Lb, hop)
        qs = max(qs, _check("offline istft", f"{label} clip {b} L={Lb}", *A.istft_arrays(got[b], y, ye, Lb, hop)))
        assert (got[b, Lb:] == 0).all(), (label, b)
    print(f"\n[{label}] F={F} B={B} L={L}: err/bound stft {qa:.3f}  istft {qs:.3f}")


@pytest.mark.parametrize("n_fft", A.N_FFTS)
def test_offline_every_n_fft(built_lib, n_fft):
    """fullsubnet.Model (no TSSE: every clip length from hop + 1): the shortest clips, both sides of the first and second run
    boundary in frames and output hops at every L mod hop class, and a clip of more than three runs, in one ragged call"""
    hop = n_fft // 2
    lengths = A.offline_lengths(n_fft)
    _offline(f"fsn n_fft {n_fft}", _fsn(hop + 1, seed=n_fft), [A.speech(n, 100 + i) for i, n in enumerate(lengths)])


def test_offline_levels_plus(built_lib):
    """FullSubNet+: digital silence in the middle and at the end, a -80 dB clip, a x1e3 clip and run-boundary lengths"""
    hop = 256
    clips = [A.with_silence(20000, 1), A.speech(9 * hop - 1, 2, 1e-4), A.speech(16 * hop + 1, 3, 1e3)]
    runs = [n for n in A.run_lengths(512) if n // hop + 1 + 2 >= 10]              # T_b + look_ahead >= the TSSE kernel size 10
    clips += [A.speech(n, 10 + i) for i, n in enumerate(runs[::3])]
    _offline("plus levels", _plus(seed=3), clips)


def test_offline_limits(built_lib):
    """Finite attenuation limits on some clips, infinite on the others"""
    hop = 256
    clips = [A.speech(n, 20 + i) for i, n in enumerate([7 * hop + 1, 8 * hop + 128, 17 * hop - 1, 24000])]
    _offline("plus limits", _plus(seed=4), clips, atten=[6.0, float("inf"), 20.0, 0.0])
    _offline("fsn limits", _fsn(129, seed=5), [A.speech(n, 30 + i) for i, n in enumerate([129, 16 * 128 + 1, 3000])],
             atten=[float("inf"), 3.0, 12.0])


# ---- streaming synthesis ----------------------------------------------------------------------------------------------------------------
def _stream(label, m, B, sessions, atten=None):
    """Per-hop audio calls over sessions {slot: (first tick, K hops)} with random HOLDs; each slot's tick k (HOLDs not counted) analyses
    frame k - 1 and synthesises frame k - 1 - look_ahead (stream_audio_ref's schedule).  Collects every slot's spectra and masks from
    the hooks, then checks each session's output against the fp64 product and synthesis of them, and the spectra against the fp64
    rfft of its samples.  A mirror handle that is never read runs the same calls: the hooks change no output."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    F, la = m._cfg.num_freqs, m._cfg.look_ahead
    hop = F - 1
    st, mirror = StreamingFullSubNet(m, B, DEV), StreamingFullSubNet(m, B, DEV)
    if atten:
        slots = sorted(atten)
        for s_ in (st, mirror):
            s_.set_atten_lim(slots, [atten[b] for b in slots])
    rng = np.random.default_rng(F + B)
    x = {b: A.speech(K * hop, 200 + b) for b, (_, K) in sessions.items()}
    tick = {b: 0 for b in sessions}
    spec = {b: np.zeros((F, K + 1), np.complex64) for b, (_, K) in sessions.items()}
    mask = {b: np.zeros((2, F, K + 1), np.float32) for b, (_, K) in sessions.items()}
    out = {b: [] for b in sessions}
    for c in range(10 ** 6):
        if all(tick[b] > K + 1 + la for b, (_, K) in sessions.items()):
            break
        flags, rows, what = [HOLD] * B, np.full((B, hop), np.nan, np.float32), {}
        for b, (t0, K) in sessions.items():
            k = tick[b]
            if c < t0 or k > K + 1 + la or (k and rng.random() < 0.2):
                continue
            flags[b] = START if k == 0 else STEP if k < K else FLUSH
            if k < K:
                rows[b] = x[b][k * hop:(k + 1) * hop]
            what[b] = (k - 1, k - 1 - la)                               # (frame analysed, frame synthesised)
            tick[b] += 1
        got, valid, um = st.step_audio(_t(rows), flags, return_mask=True)
        again, _ = mirror.step_audio(_t(rows), flags)
        assert torch.equal(got, again), (label, c)
        got, um = got.cpu().numpy(), um.cpu().numpy()
        if any(k >= 0 for k, _ in what.values()):                       # some slot stepped the model
            sp = st.get_stage("spec", (B, 1, F)).cpu().numpy()
            mk = st.get_stage("mask", (B, 2, F, 1)).cpu().numpy()
            for b, (j, mm) in what.items():
                if j < 0:
                    continue
                if mm >= 0:
                    assert np.array_equal(mk[b, :, :, 0], um[b]), (label, c, b, "the mask hook is not the call's mask")
                if j <= sessions[b][1]:
                    spec[b][:, j] = sp[b, 0]
                else:
                    assert not sp[b, 0].any(), (label, b, j, "frame past the end is not zero")
                if 0 <= mm <= sessions[b][1]:
                    mask[b][:, :, mm] = mk[b, :, :, 0]
        for b in sessions:
            if valid[b]:
                out[b].append(got[b])
    lam = {b: np.float32(10.0 ** (-atten[b] / 20.0)) for b in (atten or {})}
    qa = qs = 0.0
    for b, (_, K) in sessions.items():
        L = K * hop
        X, nrm = A.stft_truth(x[b], L, hop)
        emu = A.stft_emulate(x[b], L, hop)
        g, w, e, _ = A.stft_arrays(spec[b].real, spec[b].imag, X, emu, nrm)
        qa = max(qa, _check("stream spec", f"{label} slot {b}", g, w, e))
        y = np.concatenate(out[b])
        assert y.shape == (L,), (label, b, y.shape)
        lm = None if b not in lam else np.array([lam[b]], np.float32)
        E, _ = A.cirm_truth(mask[b][None], spec[b][None], lm)
        Ee = A.cirm_emulate(mask[b][None], spec[b][None], lm)[0].astype(np.complex64)
        yt = A.istft_truth(E[0], L, hop)
        qs = max(qs, _check("stream synthesis", f"{label} slot {b}", *A.istft_arrays(y, yt, A.istft_emulate(Ee, L, hop), L, hop)))
    print(f"\n[{label}] F={F} la={la} B={B}: err/bound spec {qa:.3f}  synthesis {qs:.3f}")
    return st


@pytest.mark.parametrize("F,la", [(33, 1), (257, 2), (513, 3)])
def test_stream_per_hop(built_lib, F, la):
    """Staggered STARTs, random HOLDs, a finite limit on one slot, at three look-aheads (ring sizes 2, 3, 4)"""
    m = _fsn(F, seed=F, la=la)
    _stream(f"stream F={F}", m, 3, {0: (0, 21), 1: (2, 12), 2: (5, 17)}, atten={1: 10.0})


def test_stream_80_slots(built_lib):
    m = _fsn(65, seed=80)
    st = _stream("stream 80 slots", m, 80, {b: (b % 4, 14 + b % 5) for b in (0, 1, 63, 64, 79)}, atten={63: 6.0})
    from fsnplus_b200 import _lib
    with pytest.raises(_lib.FsnError, match="spec needs"):
        st.get_stage("spec", (80, 2, 65))
    with pytest.raises(_lib.FsnError, match="mask needs"):
        st.get_stage("mask", (80, 2, 65, 2))
    with pytest.raises(_lib.FsnError, match="unknown stage"):
        st.get_stage("masks", (80, 2, 65, 1))
    from fsnplus_b200.streaming import StreamingFullSubNet
    masks = StreamingFullSubNet(m, 80, DEV)                                   # a handle of the mask calls
    with torch.no_grad():
        masks.step_slots(torch.zeros((80, 65), device=DEV), [START] * 80)
    with pytest.raises(_lib.FsnError, match="mask is kept only by the audio calls"):
        masks.get_stage("mask", (80, 2, 65, 1))
    with pytest.raises(_lib.FsnError, match="spec is kept only by the audio calls"):
        masks.get_stage("spec", (80, 1, 65))


def _session_check(label, x, L, hop, spec, mask, y, lam):
    """One session of L samples: its spectra of frames 0 .. L // hop against the fp64 rfft of its samples, and its output y (L samples)
    against the fp64 product and synthesis of its own masks and spectra (the one-frame end included when L mod hop > 0)"""
    X, nrm = A.stft_truth(x, L, hop)
    g, w, e, _ = A.stft_arrays(spec.real, spec.imag, X, A.stft_emulate(x, L, hop), nrm)
    qa = _check("stream spec", label, g, w, e)
    assert y.shape == (L,), (label, y.shape)
    lm = None if lam is None else np.array([lam], np.float32)
    E, _ = A.cirm_truth(mask[None], spec[None], lm)
    Ee = A.cirm_emulate(mask[None], spec[None], lm)[0].astype(np.complex64)
    qs = _check("stream synthesis", label, *A.istft_arrays(y, A.istft_truth(E[0], L, hop), A.istft_emulate(Ee, L, hop), L, hop))
    return qa, qs


def _drive(label, m, B, sessions, kind, K=4, S=None, atten=None, seed=0):
    """The chunk call (kind "chunk": rows of K hops, per-slot hop counts 1 .. K) or the sample call (kind "samples": rows of S
    samples, per-slot counts 1 .. S) over sessions {slot: (first call, L samples, flush)}: staggered STARTs and random HOLDs; flush
    "with" ends a session in the call that carries its last samples, "alone" in a call of its own.  Slot tick k (k = 0 the START,
    HOLDs not counted) stores hop k, analyses frame k - 1 and synthesises frame k - 1 - look_ahead; a session of L samples has
    L // hop + 2 + look_ahead ticks, the ticks after the FLUSH draining it.  Each call's model column c of slot b is its c-th tick
    after the START, read from the "spec" / "mask" hooks.  A mirror handle that is never read runs the same calls."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    F, la = m._cfg.num_freqs, m._cfg.look_ahead
    hop = F - 1
    st, mirror = StreamingFullSubNet(m, B, DEV), StreamingFullSubNet(m, B, DEV)
    if atten:
        for s_ in (st, mirror):
            s_.set_atten_lim(sorted(atten), [atten[b] for b in sorted(atten)])
    rng = np.random.default_rng(seed)
    x = {b: A.speech(L, 300 + b) for b, (_, L, _) in sessions.items()}
    pos = {b: 0 for b in sessions}
    tick = {b: 0 for b in sessions}
    end = {b: None for b in sessions}                                   # ticks of the session, known at its FLUSH
    spec = {b: np.zeros((F, L // hop + 1), np.complex64) for b, (_, L, _) in sessions.items()}
    mask = {b: np.zeros((2, F, L // hop + 1), np.float32) for b, (_, L, _) in sessions.items()}
    out = {b: [] for b in sessions}
    width = K * hop if kind == "chunk" else S
    ring_reads = scratch_reads = 0
    for c in range(10 ** 5):
        if all(end[b] is not None and tick[b] >= end[b] for b in sessions):
            break
        flags, cnt, rows, new = [HOLD] * B, [0] * B, np.full((B, width), np.nan, np.float32), {}
        for b, (c0, L, flush) in sessions.items():
            if c < c0 or (end[b] is not None and tick[b] >= end[b]) or (pos[b] and rng.random() < 0.2):
                continue
            left = L - pos[b]
            if kind == "chunk":
                n = min(int(rng.integers(1, K + 1)), left // hop) if left else 0
                if pos[b] == 0:
                    n = max(n, 2)                                       # a session needs two hops before its FLUSH
            else:
                n = min(int(rng.integers(1, S + 1)), left)
                if pos[b] == 0:
                    n = max(n, min(2 * hop + 1, S))
            if end[b] is not None:
                n = 0
            done = pos[b] + n == L
            if pos[b] == 0:
                flags[b] = START
            elif end[b] is not None or (done and flush == "with") or (left == 0):
                flags[b] = FLUSH
            else:
                flags[b] = STEP
            if flags[b] == FLUSH and end[b] is None:
                end[b] = L // hop + 2 + la
            cnt[b] = n
            rows[b, :n * (hop if kind == "chunk" else 1)] = x[b][pos[b]:pos[b] + n * (hop if kind == "chunk" else 1)]
            pos[b] += n * (hop if kind == "chunk" else 1)
            if kind == "chunk":
                t1 = tick[b] + n if end[b] is None else min(tick[b] + K, end[b])
            else:
                t1 = pos[b] // hop if end[b] is None else end[b]
            new[b] = (tick[b], t1)
            tick[b] = t1
        if kind == "chunk":
            got, nout = st.step_audio_chunk(_t(rows), flags, cnt)
            again, _ = mirror.step_audio_chunk(_t(rows), flags, cnt)
            n_out = {b: int(nout[b]) * hop for b in sessions}
        else:
            got, nout = st.step_audio_samples(_t(rows), cnt, flags)
            again, _ = mirror.step_audio_samples(_t(rows), cnt, flags)
            n_out = {b: int(nout[b]) for b in sessions}
        assert torch.equal(got, again), (label, c)
        got = got.cpu().numpy()
        cols = {b: [k for k in range(t0, t1) if k >= 1] for b, (t0, t1) in new.items()}
        Km = max([len(v) for v in cols.values()] + [0])
        if Km:
            sp = st.get_stage("spec", (B, Km, F)).cpu().numpy()
            mk = st.get_stage("mask", (B, 2, F, Km)).cpu().numpy()
            for b, ks in cols.items():
                L = sessions[b][1]
                j0 = ks[0] - 1 if ks else 0
                for i, k in enumerate(ks):
                    j, mm = k - 1, k - 1 - la
                    if j <= L // hop:
                        spec[b][:, j] = sp[b, i]
                    else:
                        assert not sp[b, i].any(), (label, b, j, "frame past the end is not zero")
                    if 0 <= mm <= L // hop:
                        mask[b][:, :, mm] = mk[b, :, :, i]
                        scratch_reads += mm >= j0
                        ring_reads += mm < j0
        for b in sessions:
            out[b].append(got[b, :n_out[b]])
            assert not got[b, n_out[b]:].any(), (label, c, b, "output past nout")
    assert scratch_reads and ring_reads, (scratch_reads, ring_reads)
    qa = qs = 0.0
    for b, (_, L, flush) in sessions.items():
        lam = None if b not in (atten or {}) else np.float32(10.0 ** (-atten[b] / 20.0))
        a, s_ = _session_check(f"{label} slot {b} L={L} ({L % hop} past a hop, flush {flush})", x[b], L, hop, spec[b], mask[b],
                               np.concatenate(out[b]), lam)
        qa, qs = max(qa, a), max(qs, s_)
    print(f"\n[{label}] F={F} la={la} B={B}: err/bound spec {qa:.3f}  synthesis {qs:.3f}  (frames read from the scratch "
          f"{scratch_reads}, from the ring {ring_reads})")


@pytest.mark.parametrize("F,la,K", [(33, 1, 4), (65, 2, 5), (257, 2, 3)])
def test_stream_chunks(built_lib, F, la, K):
    """The chunk call: K > look_ahead hops per call, per-slot hop counts, staggered STARTs, HOLDs, FLUSH with and without hops, a
    limit on one slot"""
    m = _fsn(F, seed=F + 7, la=la)
    hop = F - 1
    sessions = {0: (0, 23 * hop, "with"), 1: (1, 11 * hop, "alone"), 2: (3, 17 * hop, "with"), 3: (2, 9 * hop, "alone")}
    _drive(f"chunk F={F} K={K}", m, 4, sessions, "chunk", K=K, atten={2: 8.0}, seed=F)


@pytest.mark.parametrize("F,la", [(65, 2), (513, 2), (33, 1)])
def test_stream_samples(built_lib, F, la):
    """The sample call: sessions ending at 13 hop + r for r in {0, 1, hop / 2, hop - 1}, each with its FLUSH in the call carrying its
    last samples and in a call of its own; any count per call, staggered STARTs, HOLDs, a limit on one slot"""
    m = _fsn(F, seed=F + 11, la=la)
    hop = F - 1
    sessions, b = {}, 0
    for r in A.residues(hop):
        for flush in ("with", "alone"):
            sessions[b] = (b % 3, 13 * hop + r, flush)
            b += 1
    _drive(f"samples F={F}", m, len(sessions), sessions, "samples", S=3 * hop + 17, atten={5: 10.0}, seed=F)


# ---- the cIRM product -------------------------------------------------------------------------------------------------------------------
def _masks(rng, shape):
    m = rng.uniform(-12, 12, shape).astype(np.float32)
    lim = np.float32(9.9)
    special = np.array([lim, -lim, np.nextafter(lim, np.float32(20)), np.nextafter(lim, np.float32(0)),
                        -np.nextafter(lim, np.float32(20)), -np.nextafter(lim, np.float32(0)), 0.0, 1e-30, -1e-30], np.float32)
    flat = m.reshape(-1)
    flat[rng.choice(flat.size, 20 * special.size, replace=False)] = np.repeat(special, 20)
    return m


def _spectrum(rng, shape):
    mag = 10.0 ** rng.uniform(-20, 6, shape)
    X = (mag * np.exp(2j * np.pi * rng.random(shape))).astype(np.complex64)
    flat = X.reshape(-1)
    i = rng.choice(flat.size, 300, replace=False)
    flat[i[:100]] = flat[i[:100]].imag * 1j
    flat[i[100:200]] = flat[i[100:200]].real
    flat[i[200:]] = 0
    return X


def test_apply_cirm(built_lib):
    """fsn_apply_cirm: masks over [-12, 12] with +-9.9f and their fp32 neighbours, 0 and +-1e-30; |X| from 1e-20 to 1e6 with zero real
    or imaginary parts and zeros; B F T = 3 x 257 x 101, not a multiple of 256"""
    from fsnplus_b200 import inference as inf
    rng = np.random.default_rng(0)
    B, F, T = 3, 257, 101
    mask, X = _masks(rng, (B, 2, F, T)), _spectrum(rng, (B, F, T))
    got = inf.apply_cirm(_t(mask), _t(X)).cpu().numpy()
    E, sc = A.cirm_truth(mask, X)
    g, w, e, zero = A.cirm_arrays(got, E, A.cirm_emulate(mask, X), sc)
    assert zero == 0
    q = _check("cirm apply_cirm", "fsn_apply_cirm", g, w, e)
    print(f"\n[fsn_apply_cirm] B F T = {B * F * T}: err/bound {q:.3f}")


@pytest.mark.parametrize("limits", [None, [6.0, float("inf"), 0.5]])
def test_apply_cirm_planar(built_lib, limits):
    """The generic kernel's fused pass: enhance_spectrum against the mask of a forward of the same input, ragged; everything past each
    clip's frames is exactly 0"""
    m = _fsn(65, seed=9, lstm_impl="mma")
    rng = np.random.default_rng(1)
    B, F, T = 3, 65, 77
    frames = [77, 40, 13]
    X = _spectrum(rng, (B, F, T))
    mag, re, im = (np.ascontiguousarray(a[:, None]).astype(np.float32) for a in (np.abs(X), X.real, X.imag))
    with torch.no_grad():
        m1 = m(_t(mag), frames=frames).cpu().numpy()
        m2 = m(_t(mag), frames=frames).cpu().numpy()
        assert np.array_equal(m1, m2), "two mask forwards differ"
        enh = m.enhance_spectrum(_t(mag), _t(re), _t(im), frames=frames, atten_lim_db=limits).cpu().numpy()
    assert m.last_lstm_impl() == "mma"
    lam = None if limits is None else np.array([10.0 ** (-d / 20.0) for d in limits], np.float32)
    q = 0.0
    for b, n in enumerate(frames):
        Xb = (re[b, 0, :, :n] + 1j * im[b, 0, :, :n]).astype(np.complex64)[None]
        lb = None if lam is None else lam[b:b + 1]
        E, sc = A.cirm_truth(m1[b:b + 1, :, :, :n], Xb, lb)
        g, w, e, zero = A.cirm_arrays(enh[b:b + 1, :, :n], E, A.cirm_emulate(m1[b:b + 1, :, :, :n], Xb, lb), sc)
        assert zero == 0
        q = max(q, _check("cirm planar", f"planar limits={limits} clip {b}", g, w, e))
        # the kernel's extent tlen[b] is frames[b] + look_ahead (stage_lengths), so tlen - look_ahead is the clip's own n frames
        assert not enh[b, :, n:].any(), (b, "enhanced spectrum past tlen - look_ahead")
    print(f"\n[apply_cirm_planar limits={limits}] err/bound {q:.3f}")


# ---- the batch grid limit ---------------------------------------------------------------------------------------------------------------
def test_more_clips_than_the_launch_grid(built_lib):
    """66 000 short clips at num_freqs 33 in one audio call: sub-batches of at most 65 535 clips (the launch grids' y / z limit), each
    bit-identical to the same clips in a call of their own"""
    from fsnplus_b200 import _lib
    m = _fsn(33, seed=66)
    B, L = 66000, 200
    lengths = [L - (b % 7) * 23 for b in range(B)]
    rows = np.tile(A.speech(L, 5), (B, 1)) * np.linspace(0.5, 2.0, B, dtype=np.float32)[:, None]
    x = _t(rows)
    with torch.no_grad():
        got = m.enhance_audio(x, lengths)
        Bs = m.last_plan_bins()[0]
        assert Bs == 33000, Bs
        assert _lib.plan_audio(m._cfg, B, L)[0] == Bs
        for b0 in (0, Bs):
            part = m.enhance_audio(x[b0:b0 + Bs].contiguous(), lengths[b0:b0 + Bs])
            assert m.last_plan_bins()[0] == Bs
            assert torch.equal(got[b0:b0 + Bs], part), b0
    print(f"\n[grid limit] B = {B}: sub-batches of {Bs}, bit-identical to two calls of {Bs}")


def test_zz_worst_per_stage(built_lib):
    print("\nworst err / bound per stage (FACTOR = %.2f; the emulation's share of the bound in brackets):" % FACTOR)
    for k, (q, label, eq) in sorted(WORST.items()):
        print(f"  {k:18s} {q:.3f}  [{eq:.3f}]  {label}")
