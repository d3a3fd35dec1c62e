"""Audio chunk call (fsn_stream_step_audio_chunk, DESIGN.md §3.14): K hops per slot and call, each slot with its own hop count.

A schedule is a list of calls, each with its own K, and of sessions, each on one slot: a session STARTs at its first call, then STEPs
(or, with its last hops, FLUSHes) a seeded number of its remaining hops at every call that is not one of its holds, then FLUSHes with 0
hops until its output is complete, plus optional extra FLUSH calls (which act as HOLD).  Every sample the call must not read is NaN.
  * lstm_impl = "mma": every call's output rows, hop counts and mask columns are the bits of the same calls expanded into per-hop
    fsn_stream_step_audio_slots ticks on a second handle, and so are saved payloads;
  * layer-wise path: every session's waveform and masks are the bits of its lone run (one chunk call over all its hops on a 1-slot
    handle), under caps that force sub-batches and windows too; its waveform is the fp64 iSTFT pipeline fed with the returned masks
    within 2e-5, and end to end within the offline bars."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O
from test_gpu_stream_audio import _clips
from test_gpu_stream_chunks import _fsn
from test_gpu_stream_sessions import DEV, MASK_TOL, _small_cfg, _t

pytestmark = pytest.mark.gpu
XFORM_TOL = 2e-5          # chunked waveform vs the fp64 pipeline fed with the returned masks
WAVE_TOL = 2e-3           # vs the offline enhancement (fp64 oracle, offline GPU forward)
KS = [1, 2, 3, 8, 37, 5, 1, 16, 4, 9, 2, 32, 3, 7, 1, 12, 6, 20, 3, 8, 8, 2, 11, 5]


class Session:
    def __init__(self, slot, start, x, hop, holds=(), extra=0, seed=0):
        self.slot, self.start, self.x, self.holds, self.extra = slot, start, np.asarray(x, np.float32), set(holds), extra
        self.T = len(self.x) // hop
        assert self.T * hop == len(self.x) and self.T >= 2
        self.rng = np.random.default_rng(seed)


def expand(flag, n, K):
    from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP
    if flag == HOLD:
        return [HOLD] * K
    if flag == START:
        return [START] + [STEP] * (n - 1) + [HOLD] * (K - n)
    return [STEP] * n + [HOLD if flag == STEP else FLUSH] * (K - n)


def _advance(tr, f, la):
    """One per-hop tick of a session tracker [slot tick, hops K (0 before the FLUSH)]: the frame whose mask the tick returns, or None."""
    from fsnplus_b200.streaming import FLUSH, START, STEP
    if f == START:
        tr[:] = [1, 0]
        return None
    if f not in (STEP, FLUSH):
        return None
    if f == FLUSH and not tr[1]:
        tr[1] = tr[0]
    if tr[1] and tr[0] > tr[1] + la + 1:                        # a FLUSH past the session's end is a HOLD
        return None
    tr[0] += 1
    return tr[0] - 2 - la


def _plan(sessions, Ks, la):
    """call -> {slot: (session, flag, first hop, n)}."""
    from fsnplus_b200.streaming import FLUSH, START, STEP
    calls = [dict() for _ in Ks]
    for i, s in enumerate(sessions):
        q, tr, extra, c = 0, [-1, 0], s.extra, s.start
        while True:
            assert c < len(Ks), "the schedule ends before a session"
            if c in s.holds:
                c += 1
                continue
            K, r = Ks[c], s.T - q
            if tr[1] and tr[0] == tr[1] + la + 2:               # complete: extra FLUSH calls act as HOLD
                if not extra:
                    break
                extra -= 1
                flag, n = FLUSH, 0
            elif tr[0] < 0:
                flag, n = START, int(min(K, r) if s.rng.random() < 0.7 else s.rng.integers(1, min(K, r) + 1))
            elif r > 0:
                n = int(min(K, r) if s.rng.random() < 0.6 else s.rng.integers(1, min(K, r) + 1))
                flag = FLUSH if n == r and s.rng.random() < 0.5 else STEP
            else:
                flag, n = FLUSH, 0
            assert s.slot not in calls[c], "sessions overlap on a slot"
            calls[c][s.slot] = (i, flag, q, n)
            for f in expand(flag, n, K):
                _advance(tr, f, la)
            q += n
            c += 1
    return calls


def _drive(st, sessions, Ks, la, per_hop=False):
    """Run the schedule through chunk calls (or their per-hop expansion).  Returns the calls' (out, nout, masks) and each session's
    (waveform [L], masks [2, F, T + 1])."""
    from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP
    calls = _plan(sessions, Ks, la)
    B, F, hop = st.B, st.F, st.hop
    res, wav = [], [[] for _ in sessions]
    masks = [dict() for _ in sessions]
    tick = [[-1, 0] for _ in sessions]           # per session: slot tick, hops K (0 before the FLUSH)
    for c, K in enumerate(Ks):
        flags, hops = np.full(B, HOLD, np.int32), np.zeros(B, np.int32)
        x = np.full((B, K * hop), np.nan, np.float32)
        for slot, (i, f, q, n) in calls[c].items():
            flags[slot], hops[slot] = f, n
            x[slot, :n * hop] = sessions[i].x[q * hop:(q + n) * hop]
        if per_hop:
            out, nout, mask = torch.zeros((B, K * hop)), torch.zeros(B, dtype=torch.int32), torch.zeros((B, 2, F, K))
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
        for b in range(B):
            if b not in calls[c]:
                assert int(nout[b]) == 0 and torch.count_nonzero(out[b]) == 0 and torch.count_nonzero(mask[b]) == 0, f"call {c} slot {b}"
                continue
            i = calls[c][b][0]
            wav[i].append(out[b, :int(nout[b]) * hop])
            assert torch.count_nonzero(out[b, int(nout[b]) * hop:]) == 0, f"call {c} slot {b}: output past nout is not zero"
            for k, f in enumerate(expand(int(flags[b]), int(hops[b]), K)):
                m = _advance(tick[i], f, la)
                if m is not None and m >= 0:
                    masks[i][m] = mask[b, ..., k].clone()
                else:
                    assert torch.count_nonzero(mask[b, ..., k]) == 0, f"call {c} slot {b} tick {k}: a mask without a frame"
    sess = []
    for i, s in enumerate(sessions):
        w = torch.cat(wav[i])
        assert w.numel() == len(s.x) and sorted(masks[i]) == list(range(s.T + 1)), f"session {i} incomplete"
        sess.append((w, torch.stack([masks[i][m] for m in range(s.T + 1)], dim=-1)))
    return res, sess


def _lone(m, s, la):
    """The session alone on a 1-slot handle: one START call with all its hops, then one FLUSH call of 0 hops."""
    from fsnplus_b200.streaming import FLUSH, START, StreamingFullSubNet
    st = StreamingFullSubNet(m, batch_size=1, device=DEV)
    hop = st.hop
    a, n1, m1 = st.step_audio_chunk(_t(s.x[None]), [START], [s.T], return_mask=True)
    b, n2, m2 = st.step_audio_chunk(_t(np.full((1, (la + 2) * hop), np.nan, np.float32)), [FLUSH], [0], return_mask=True)
    st.close()
    assert int(n1[0]) + int(n2[0]) == s.T
    w = torch.cat([a[0, :int(n1[0]) * hop].cpu(), b[0, :int(n2[0]) * hop].cpu()])
    masks = torch.cat([m1[0, ..., 1 + la:].cpu(), m2[0].cpu()], dim=-1)   # tick k of the first call is frame k - 1 - la
    return w, masks


def _check_pipeline(sessions, sess, n_fft, tol=XFORM_TOL):
    hop = n_fft // 2
    for i, (s, (w, mk)) in enumerate(zip(sessions, sess)):
        X = O.stft(s.x[None].astype(np.float64), n_fft, hop, n_fft)
        ref = O.istft(O.enhance(X, mk.numpy()[None].astype(np.float64)), n_fft, hop, n_fft, length=len(s.x))[0]
        e = O.rel_l2(w.numpy(), ref)
        print(f"\n[session {i}, slot {s.slot}, T={s.T}] waveform vs fp64 iSTFT of its masks {e:.2e}")
        assert e < tol


def _check_e2e(m, params, cfg, s, w, mk):
    from fsnplus_b200 import inference as inf
    n_fft = 2 * (cfg["num_freqs"] - 1)
    hop = n_fft // 2
    X = O.stft(s.x[None].astype(np.float64), n_fft, hop, n_fft)
    crm = O.fullsubnet_forward(params, cfg, np.abs(X)[:, None])
    ref = O.istft(O.enhance(X, crm), n_fft, hop, n_fft, length=len(s.x))[0]
    with torch.no_grad():
        off = inf.enhance_batch(m, _t(s.x[None]), n_fft, hop, n_fft, complex_inputs=False)[0].cpu().numpy()
    e_mask, e_ref, e_off = O.rel_l2(mk.numpy(), crm[0]), O.rel_l2(w.numpy(), ref), O.rel_l2(w.numpy(), off)
    print(f"masks vs oracle {e_mask:.2e}  waveform vs fp64 pipeline {e_ref:.2e}  vs offline GPU {e_off:.2e}")
    assert e_mask < MASK_TOL and e_ref < WAVE_TOL and e_off < WAVE_TOL


def _small_sessions(hop):
    """4 slots: staggered joins, holds mid-session, slot 0 reused by a quiet session after a loud one, slot 3 never started."""
    A, B_, Cc, D, E = _clips(5, [30, 61, 45, 26, 3], hop, seed0=900, gains=[8.0, 1.0, 1.0, 0.05, 1.0])
    return [Session(0, 0, A, hop, seed=1), Session(1, 1, B_, hop, holds=(3, 4, 9), extra=1, seed=2),
            Session(2, 3, Cc, hop, holds=(6,), seed=3), Session(0, 9, D, hop, holds=(11,), extra=2, seed=4),
            Session(1, 20, E, hop, seed=5)]


def _compare_calls(got, want):
    for c, ((o, n, mk), (o2, n2, mk2)) in enumerate(zip(got, want)):
        assert torch.equal(n, n2), f"call {c}: nout {n.tolist()} != {n2.tolist()}"
        assert torch.equal(o, o2), f"call {c}: output differs from the per-hop ticks"
        assert torch.equal(mk, mk2), f"call {c}: masks differ from the per-hop ticks"


SMALL = [("cumulative_laplace_norm", "LSTM"), ("cumulative_layer_norm", "LSTM"), ("cumulative_laplace_norm", "GRU")]


@pytest.mark.parametrize("norm,rnn", SMALL)
def test_mma_audio_chunks_match_per_hop_small(built_lib, norm, rnn):
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params, lstm_impl="mma")
    la = cfg["look_ahead"]
    sessions = _small_sessions(64)
    st, ref = StreamingFullSubNet(m, batch_size=4, device=DEV), StreamingFullSubNet(m, batch_size=4, device=DEV)
    got, gs = _drive(st, sessions, KS, la)
    want, _ = _drive(ref, _small_sessions(64), KS, la, per_hop=True)
    _compare_calls(got, want)
    p1, p2 = st.save_slots([0, 1, 2]), ref.save_slots([0, 1, 2])          # the slots that served sessions
    assert _meta(p1) == _meta(p2)
    for i in range(9):                                                   # the alignment gaps between segments are not written
        s0, s1 = _segment(m._cfg, i)
        assert torch.equal(p1.payload[:, s0:s1], p2.payload[:, s0:s1]), f"payload segment {i}"
    st.close(); ref.close()
    _check_pipeline(sessions, gs, 128, tol=1e-5)


@pytest.mark.parametrize("F,la", [(33, 1), (129, 3), (513, 2)])
def test_mma_audio_chunks_fft_sizes(built_lib, F, la):
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=F, look_ahead=la, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=96,
               norm_type="cumulative_laplace_norm")
    params = O.make_params_fsn(cfg, seed=41)
    m = _fsn(cfg, params, lstm_impl="mma")
    hop = F - 1

    def sessions():
        x = _clips(3, [40, 2, 23], hop, seed0=700 + F)
        return [Session(0, 0, x[0], hop, holds=(5,), seed=7), Session(1, 2, x[1], hop, extra=1, seed=8),
                Session(1, 8, x[2], hop, holds=(10,), seed=9)]
    st, ref = StreamingFullSubNet(m, batch_size=2, device=DEV), StreamingFullSubNet(m, batch_size=2, device=DEV)
    got, gs = _drive(st, sessions(), KS, la)
    want, _ = _drive(ref, sessions(), KS, la, per_hop=True)
    _compare_calls(got, want)
    st.close(); ref.close()
    _check_pipeline(sessions(), gs, 2 * hop, tol=1e-5)


@pytest.mark.parametrize("norm,rnn", SMALL)
def test_layerwise_audio_chunks_small(built_lib, norm, rnn):
    """Every session bit-identical to its lone run; waveform vs the fp64 pipeline of its masks; end to end for two sessions."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params)
    la = cfg["look_ahead"]
    sessions = _small_sessions(64)
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    _, gs = _drive(st, sessions, KS, la)
    st.close()
    for i, s in enumerate(sessions):
        lw, lm = _lone(m, s, la)
        assert torch.equal(gs[i][0], lw) and torch.equal(gs[i][1], lm), f"session {i} differs from its lone run"
    _check_pipeline(sessions, gs, 128)
    for i in (1, 2):
        _check_e2e(m, params, cfg, sessions[i], *gs[i])


def test_layerwise_audio_chunks_under_a_low_cap(built_lib, monkeypatch):
    """Caps that force sub-batches of one session and windows: the same bits as the uncapped handle."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    params = O.make_params_fsn(cfg, seed=13)
    la = cfg["look_ahead"]
    st = StreamingFullSubNet(_fsn(cfg, params), batch_size=4, device=DEV)
    _, want = _drive(st, _small_sessions(64), KS, la)
    st.close()
    for cap_gb in (0.0015, 0.0004):
        st = StreamingFullSubNet(_fsn(cfg, params, monkeypatch, cap_gb), batch_size=4, device=DEV)
        _, got = _drive(st, _small_sessions(64), KS, la)
        st.close()
        for i in range(len(want)):
            assert torch.equal(got[i][0], want[i][0]) and torch.equal(got[i][1], want[i][1]), f"cap {cap_gb} GB, session {i}"


@pytest.mark.parametrize("B", [3, 80])
def test_audio_chunks_default_geometry(built_lib, B):
    """Config #4 geometry: 3 slots run the weight-stationary full band, 80 the generic one.  Layer-wise sessions bit-identical to their
    lone runs and within the bars; the history and spectrum rings of a saved session are the per-hop run's; with lstm_impl = "mma" every
    call is bit-identical to its per-hop expansion."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    la = cfg["look_ahead"]
    Ks = [3, 32, 4, 1, 37, 4, 32, 8, 16, 2, 32, 8, 5, 16, 3, 32, 8, 4]

    def sessions():
        if B == 3:
            x = _clips(4, [60, 90, 50, 40], 256, seed0=500, gains=[6.0, 1.0, 1.0, 0.1])
            return [Session(0, 0, x[0], 256, seed=1), Session(1, 1, x[1], 256, holds=(3,), seed=2),
                    Session(2, 2, x[2], 256, seed=3), Session(0, 7, x[3], 256, extra=1, seed=4)]
        n = B + 2
        x = _clips(n, [40 + i % 13 for i in range(n)], 256, seed0=600)
        out = [Session(i, i % 3, x[i], 256, holds=(3,) if i % 7 == 3 else (), seed=i) for i in range(B)]
        return out + [Session(j, 7, x[B + j], 256, seed=100 + j) for j in range(2)]
    m = _fsn(cfg, params)
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    _, gs = _drive(st, sessions(), Ks, la)
    st.close()
    ss = sessions()
    for i in ([0, 1, 3] if B == 3 else [1, 40, B]):
        lw, lm = _lone(m, ss[i], la)
        assert torch.equal(gs[i][0], lw) and torch.equal(gs[i][1], lm), f"session {i} differs from its lone run"
        _check_pipeline([ss[i]], [gs[i]], 512)
        _check_e2e(m, params, cfg, ss[i], *gs[i])
    # the history and spectrum rings of a saved session (after 3 calls) are those of the per-hop run
    st, ref = StreamingFullSubNet(m, batch_size=B, device=DEV), StreamingFullSubNet(m, batch_size=B, device=DEV)
    _drive_prefix(st, sessions(), Ks, la, 3)
    _drive_prefix(ref, sessions(), Ks, la, 3, per_hop=True)
    a, b = st.save_slots([1]), ref.save_slots([1])
    assert _meta(a) == _meta(b)
    for i in (6, 7):
        s0, s1 = _segment(m._cfg, i)
        assert torch.equal(a.payload[:, s0:s1], b.payload[:, s0:s1]), f"payload segment {i}"
    st.close(); ref.close()
    mm = _fsn(cfg, params, lstm_impl="mma")
    st, ref = StreamingFullSubNet(mm, batch_size=B, device=DEV), StreamingFullSubNet(mm, batch_size=B, device=DEV)
    got, _ = _drive(st, sessions(), Ks, la)
    want, _ = _drive(ref, sessions(), Ks, la, per_hop=True)
    _compare_calls(got, want)
    st.close(); ref.close()


def _meta(state):
    """The fields of each saved session's fsn_slot_meta (its raw bytes include the struct's padding)."""
    return [(x.magic, x.version, x.weights_id, x.mode, x.frames, x.tick, x.hops, x.payload_bytes) for x in state.meta]


def _segment(cfg, i):
    """[begin, end) of payload segment i of an audio payload (16-byte aligned each, include/fsnplus_b200.h)."""
    F, L = cfg.num_freqs, cfg.num_layers
    sizes = [16, F * 16, L * cfg.fb_hidden * 2, L * cfg.fb_hidden * 4, L * F * cfg.sb_hidden * 2, L * F * cfg.sb_hidden * 4,
             3 * (F - 1) * 4, (cfg.look_ahead + 1) * F * 8, (F - 1) * 4]
    off, at = [], 0
    for n in sizes:
        at = (at + 15) // 16 * 16
        off.append((at, at + n))
        at += n
    return off[i]


def _drive_prefix(st, sessions, Ks, la, ncalls, per_hop=False):
    """The first ncalls calls of a schedule (the sessions do not complete)."""
    from fsnplus_b200.streaming import HOLD
    calls = _plan(sessions, Ks, la)
    B, hop = st.B, st.hop
    for c in range(ncalls):
        K = Ks[c]
        flags, hops = np.full(B, HOLD, np.int32), np.zeros(B, np.int32)
        x = np.full((B, K * hop), np.nan, np.float32)
        for slot, (i, f, q, n) in calls[c].items():
            flags[slot], hops[slot] = f, n
            x[slot, :n * hop] = sessions[i].x[q * hop:(q + n) * hop]
        if per_hop:
            ticks = [expand(int(flags[b]), int(hops[b]), K) for b in range(B)]
            for k in range(K):
                fk = np.array([ticks[b][k] for b in range(B)], np.int32)
                st.step_audio(_t(np.ascontiguousarray(x[:, k * hop:(k + 1) * hop])), torch.from_numpy(fk))
        else:
            st.step_audio_chunk(_t(x), torch.from_numpy(flags), torch.from_numpy(hops))


@pytest.mark.parametrize("move", [3, 80])
def test_audio_chunks_mixed_with_per_hop_and_moved(built_lib, move):
    """Per-hop and chunk calls alternating on one session, then a save after a chunk call loaded into another handle that continues with
    chunks: within the bars, and bit-identical to the uninterrupted run when the new handle runs the same full-band kernel (3 slots:
    weight-stationary; 80: generic)."""
    from fsnplus_b200.streaming import FLUSH, START, STEP, StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    la = cfg["look_ahead"]
    m = _fsn(cfg, params)
    x = _clips(1, [70], 256, seed0=800)[0]
    s = Session(0, 0, x, 256)

    def run(move):
        st = StreamingFullSubNet(m, batch_size=3, device=DEV)
        out, masks = [], []
        q = 0

        def chunk(h, slot, flag, n, K):
            nonlocal q
            xs = np.full((h.B, K * 256), np.nan, np.float32)
            xs[slot, :n * 256] = x[q * 256:(q + n) * 256]
            fl, hp = np.zeros(h.B, np.int32), np.zeros(h.B, np.int32)
            fl[slot], hp[slot] = flag, n
            o, nn, mk = h.step_audio_chunk(_t(xs), torch.from_numpy(fl), torch.from_numpy(hp), return_mask=True)
            out.append(o[slot, :int(nn[slot]) * 256].cpu())
            q += n

        def hop1(h, slot, flag):
            nonlocal q
            xs = np.full((h.B, 256), np.nan, np.float32)
            if flag != FLUSH:
                xs[slot] = x[q * 256:(q + 1) * 256]
                q += 1
            fl = np.zeros(h.B, np.int32)
            fl[slot] = flag
            o, v = h.step_audio(_t(xs), torch.from_numpy(fl))
            if v[slot]:
                out.append(o[slot].cpu())
        chunk(st, 0, START, 9, 9)
        for _ in range(5):
            hop1(st, 0, STEP)
        chunk(st, 0, STEP, 16, 16)
        hop1(st, 0, STEP)
        chunk(st, 0, STEP, 7, 8)
        h, slot = st, 0
        if move:
            saved = st.save_slots([0])
            h, slot = StreamingFullSubNet(m, batch_size=move, device=DEV), move - 1
            h.load_slots([slot], saved)
        chunk(h, slot, STEP, 20, 20)
        chunk(h, slot, FLUSH, 70 - q, 32)
        chunk(h, slot, FLUSH, 0, 4)
        st.close()
        if move:
            h.close()
        return torch.cat(out)
    a, b = run(0), run(move)
    assert a.numel() == len(x) and b.numel() == len(x)
    X = O.stft(x[None].astype(np.float64), 512, 256, 512)
    crm = O.fullsubnet_forward(params, cfg, np.abs(X)[:, None])
    ref = O.istft(O.enhance(X, crm), 512, 256, 512, length=len(x))[0]
    ea, eb = O.rel_l2(a.numpy(), ref), O.rel_l2(b.numpy(), ref)
    print(f"\nmixed per-hop / chunk vs fp64 pipeline {ea:.2e}; moved to 80 slots {eb:.2e}; a vs b {O.rel_l2(b.numpy(), a.numpy()):.2e}")
    assert ea < WAVE_TOL and eb < WAVE_TOL
    if move == 3:
        assert torch.equal(a, b)


def test_audio_chunk_rejects_bad_arguments(built_lib):
    from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP, StreamingFullSubNet
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=21), lstm_impl="mma")
    st, twin = StreamingFullSubNet(m, batch_size=4, device=DEV), StreamingFullSubNet(m, batch_size=4, device=DEV)
    lib = st.lib
    K = 4
    x = _t(np.random.default_rng(0).standard_normal((4, K * 64)).astype(np.float32) * 0.1)
    out = torch.empty((4, K * 64), device=DEV)
    nout = (C.c_int32 * 4)()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(flags, hops, h=st, k=K, xp=None, op=None, np_=nout, hp=True):
        f = None if flags is None else (C.c_int32 * 4)(*flags)
        n = None if hops is None else (C.c_int32 * 4)(*hops)
        xp = C.c_void_p(x.data_ptr()) if xp is None else xp
        op = C.c_void_p(out.data_ptr()) if op is None else op
        return lib.fsn_stream_step_audio_chunk(h._st, xp, k, f, n, op, np_, None, stream)

    def err():
        return lib.fsn_last_error().decode()

    def same(flags, hops):
        """A valid call on both handles gives the same outputs: the failed calls before it changed nothing."""
        assert call(flags, hops) == 0
        a = out.clone()
        assert call(flags, hops, h=twin) == 0
        assert torch.equal(a, out)

    for flags, slot in (([0, 0, 4, 0], 2), ([-1, 0, 0, 0], 0), ([0, 0, 0, 7], 3)):
        assert call(flags, [1] * 4) == -1 and f"slot {slot}" in err() and "flag" in err()
    for hops, slot in (([0, 1, 1, 1], 0), ([1, 5, 1, 1], 1)):
        assert call([START] * 4, hops) == -1 and f"slot {slot}" in err() and "h_hops" in err()
    assert call([STEP, HOLD, HOLD, HOLD], [1] * 4) == -1 and "slot 0" in err() and "without a session" in err()
    assert call([HOLD, FLUSH, HOLD, HOLD], [0] * 4) == -1 and "slot 1" in err() and "without a session" in err()
    assert call(None, [1] * 4) == -1 and "h_flags" in err()
    assert call([START] * 4, None) == -1 and "h_hops" in err()
    assert call([START] * 4, [1] * 4, np_=None) == -1 and "h_nout" in err()
    assert call([START] * 4, [1] * 4, xp=C.c_void_p()) == -1 and "d_samples" in err()
    assert call([START] * 4, [1] * 4, op=C.c_void_p()) == -1 and "d_out" in err()
    assert call([START] * 4, [1] * 4, k=0) == -1 and "K = 0" in err()
    assert call([START] * 4, [1] * 4, k=65535 * 256) == -1 and "chunk limit" in err()
    same([START, START, START, HOLD], [1, 2, 4, 0])
    assert call([FLUSH, STEP, HOLD, HOLD], [0, 1, 0, 0]) == -1 and "slot 0" in err() and "at least 2" in err()   # a 1-hop session
    same([FLUSH, STEP, FLUSH, HOLD], [1, 3, 0, 0])
    assert call([HOLD, HOLD, STEP, HOLD], [0, 0, 1, 0]) == -1 and "slot 2" in err() and "FLUSH" in err()        # STEP after the flush
    assert call([FLUSH, HOLD, HOLD, HOLD], [2, 0, 0, 0]) == -1 and "slot 0" in err() and "h_hops = 2" in err()
    same([FLUSH, STEP, FLUSH, HOLD], [0, 4, 0, 0])
    same([START, STEP, START, HOLD], [3, 1, 4, 0])                                                               # START reuses slots
    # one handle serves masks or audio, not both
    assert lib.fsn_stream_step_chunk(st._st, C.c_void_p(x.data_ptr()), 4, C.c_void_p(torch.empty((4, 2, 65, 4), device=DEV).data_ptr()),
                                     (C.c_int32 * 4)(1, 1, 1, 1), nout, stream) == -3
    masks = StreamingFullSubNet(m, batch_size=4, device=DEV)
    masks.step_chunk(torch.zeros((4, 65, 4), device=DEV), [START] * 4)
    assert call([START] * 4, [1] * 4, h=masks) == -3
    torch.cuda.synchronize()
    for s in (st, twin, masks):
        s.close()
