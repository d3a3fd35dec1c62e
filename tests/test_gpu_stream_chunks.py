"""Streaming chunk call (fsn_stream_step_chunk, DESIGN.md §3.13): K frames per slot and call.

A schedule is a list of calls, each with its own K, and of sessions, each on one slot: a session STARTs at its first call, steps K
frames of its clip (then zero frames: the look_ahead flush, and any frames past it) at every call that is not one of its holds, and ends
once it has consumed T + look_ahead frames.  Held slots are fed NaN frames, which the call must never read.
  * lstm_impl = "mma": every session is bit-identical to the same schedule stepped frame by frame with fsn_stream_step_slots;
  * layer-wise path: every session is bit-identical to its lone run (one call over all its frames on a 1-slot handle), so the masks do
    not depend on the chunk splits, the slot, the neighbours or the full-band kernel; under a low cap (sub-batches, windows) too; and
    every session is within 1e-3 of the fp64 oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASK_TOL = 1e-3
KS = [3, 4, 1, 37, 32, 4, 3, 1, 37, 4, 32]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _fsn(cfg, params, monkeypatch=None, cap_gb=None, **kw):
    from fsnplus_b200.model import Model
    if monkeypatch is not None:
        monkeypatch.setenv("FSN_WS_CAP_GB", str(cap_gb))
    m = Model(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    if monkeypatch is not None:
        monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
    return m


def _small_cfg(norm="cumulative_laplace_norm", rnn="LSTM"):
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=65, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=96, norm_type=norm, sequence_model=rnn)
    return cfg


def _small_clips(lens, seed):
    rng = np.random.default_rng(seed)
    out = []
    for T in lens:
        re, im = rng.standard_normal((65, T)) * 0.05 + 0.004, rng.standard_normal((65, T)) * 0.05 - 0.003
        out.append(np.sqrt(re ** 2 + im ** 2).astype(np.float32))
    return out


def _speech_clips(lens, seed0):
    T = max(lens)
    mag = np.abs(O.stft(O.synth_clips(len(lens), num_samples=256 * (T - 1), seed0=seed0))).astype(np.float32)
    return [np.ascontiguousarray(mag[i, :, :n]) for i, n in enumerate(lens)]


class Session:
    def __init__(self, slot, start, clip, holds=()):
        self.slot, self.start, self.clip, self.holds = slot, start, clip, set(holds)
        self.T = clip.shape[1]

    def frames(self, n0, K):
        out = np.zeros((self.clip.shape[0], K), dtype=np.float32)
        if n0 < self.T:
            out[:, :min(K, self.T - n0)] = self.clip[:, n0:n0 + K]
        return out


def _plan(sessions, Ks, la):
    """call -> {slot: (session, n0)}: the session steps frames n0 .. n0 + K - 1 at that call."""
    steps = [dict() for _ in Ks]
    for i, s in enumerate(sessions):
        n, c = 0, s.start
        while n < s.T + la:
            assert c < len(Ks), "the schedule ends before a session"
            if c not in s.holds:
                assert s.slot not in steps[c], "sessions overlap on a slot"
                steps[c][s.slot] = (i, n)
                n += Ks[c]
            c += 1
        s.end = c
    return steps


def _collect(outs, i, n0, cols, la):
    """cols [2, F, K]: columns of frames n0 + k - la; keep the valid ones."""
    for k in range(cols.shape[-1]):
        if n0 + k - la >= 0:
            outs[i][n0 + k - la] = cols[..., k].clone()


def _result(sessions, outs):
    return [torch.stack([o[t] for t in range(s.T)], dim=-1) for s, o in zip(sessions, outs)]


def _run_chunks(st, sessions, Ks, la, per_frame=()):
    """Run the schedule with one chunk call per entry of Ks (calls listed in per_frame go through fsn_stream_step_slots instead, K
    ticks); check nvalid and the zero columns; return each session's masks [2, F, T]."""
    from fsnplus_b200.streaming import HOLD, START, STEP
    steps = _plan(sessions, Ks, la)
    B, F = st.B, st.F
    outs = [dict() for _ in sessions]
    for c, K in enumerate(Ks):
        flags = np.full(B, HOLD, dtype=np.int32)
        mag = np.full((B, F, K), np.nan, dtype=np.float32)
        for slot, (i, n0) in steps[c].items():
            flags[slot] = START if n0 == 0 else STEP
            mag[slot] = sessions[i].frames(n0, K)
        if c in per_frame:
            mask = torch.zeros((B, 2, F, K))
            for k in range(K):
                fk = np.where(flags == START, START if k == 0 else STEP, flags).astype(np.int32)
                m, _ = st.step_slots(_t(mag[:, :, k]), torch.from_numpy(fk))
                mask[..., k] = m.cpu()
        else:
            mask, nvalid = st.step_chunk(_t(mag), torch.from_numpy(flags))
            mask = mask.cpu()
            for b in range(B):
                want = 0 if b not in steps[c] else min(max(steps[c][b][1] + K - la, 0), K)
                assert int(nvalid[b]) == want, f"call {c} slot {b}: nvalid {int(nvalid[b])} != {want}"
                assert torch.count_nonzero(mask[b, ..., :K - want]) == 0, f"call {c} slot {b}: an invalid column is not zero"
        for slot, (i, n0) in steps[c].items():
            _collect(outs, i, n0, mask[slot], la)
    return _result(sessions, outs)


def _run_slots(st, sessions, Ks, la):
    """The same schedule through fsn_stream_step_slots, K ticks per call."""
    return _run_chunks(st, sessions, Ks, la, per_frame=range(len(Ks)))


def _lone(m, s, la):
    """The session alone: one chunk call over all its frames on a fresh 1-slot handle."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    st = StreamingFullSubNet(m, batch_size=1, device=DEV)
    out = _run_chunks(st, [Session(0, 0, s.clip)], [s.T + la], la)[0]
    st.close()
    return out


def _oracle_err(params, cfg, s, got):
    ref = O.fullsubnet_forward(params, cfg, s.clip[None, None])[0]
    return O.rel_l2(got.numpy(), ref)


def _small_schedule(seed):
    A, B_, Cc, D = _small_clips([18, 45, 60, 22], seed=seed)
    return [Session(0, 0, A), Session(1, 1, B_, holds=(3, 6)), Session(2, 3, Cc, holds=(5,)), Session(0, 6, D, holds=(8,))]


SMALL = [("cumulative_laplace_norm", "LSTM"), ("cumulative_layer_norm", "LSTM"), ("cumulative_laplace_norm", "GRU")]


@pytest.mark.parametrize("norm,rnn", SMALL)
def test_mma_chunks_match_slot_steps_small(built_lib, norm, rnn):
    """Generic sub-band path: 4 slots (slot 3 never started), staggered STARTs, holds and slot 0 reused: every session's masks are
    the bits of the same schedule stepped frame by frame."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params, lstm_impl="mma")
    la = cfg["look_ahead"]
    sessions = _small_schedule(9)
    st, ref = StreamingFullSubNet(m, batch_size=4, device=DEV), StreamingFullSubNet(m, batch_size=4, device=DEV)
    got, want = _run_chunks(st, sessions, KS, la), _run_slots(ref, sessions, KS, la)
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g, w), f"session {i}"
        assert _oracle_err(params, cfg, sessions[i], g) < MASK_TOL
    st.close(); ref.close()


@pytest.mark.parametrize("norm,rnn", SMALL)
def test_layerwise_chunks_small(built_lib, norm, rnn):
    """Layer-wise path: every session bit-identical to its lone run (any split, slot, neighbours), and within 1e-3 of the oracle."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params)
    la = cfg["look_ahead"]
    sessions = _small_schedule(9)
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    got = _run_chunks(st, sessions, KS, la)
    st.close()
    for i, s in enumerate(sessions):
        assert torch.equal(got[i], _lone(m, s, la)), f"session {i} differs from its lone run"
        e = _oracle_err(params, cfg, s, got[i])
        print(f"\n[{norm} {rnn} session {i}] vs oracle {e:.2e}")
        assert e < MASK_TOL


def test_layerwise_chunks_under_a_low_cap(built_lib, monkeypatch):
    """FSN_WS_CAP_GB low enough for sub-batches of one session and for windows: the same bits as the uncapped handle."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg()
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params)
    la = cfg["look_ahead"]
    sessions = _small_schedule(9)
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    want = _run_chunks(st, sessions, KS, la)
    st.close()
    for cap_gb in (0.0015, 0.0004):
        mc = _fsn(cfg, params, monkeypatch, cap_gb)
        c = mc._cfg
        bs, tw, _ = _lib.stream_chunk_plan(c, 3, 37, cap_bytes=cap_gb * 1e9)
        assert bs < 3 and (cap_gb > 0.001 or tw > 0), (bs, tw)
        st = StreamingFullSubNet(mc, batch_size=4, device=DEV)
        got = _run_chunks(st, sessions, KS, la)
        st.close()
        for i in range(len(sessions)):
            assert torch.equal(got[i], want[i]), f"cap {cap_gb} GB, session {i}"


@pytest.mark.parametrize("B", [3, 80])
def test_chunks_default_geometry(built_lib, B):
    """Config #4 geometry: 3 slots run the weight-stationary full band, 80 the generic one.  Layer-wise sessions bit-identical to their
    lone runs and within 1e-3 of the oracle; with lstm_impl = "mma" bit-identical to the per-frame schedule."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    la = cfg["look_ahead"]
    Ks = [3, 32, 4, 1, 37, 4, 32]
    if B == 3:
        clips = _speech_clips([40, 60, 36, 30], seed0=500)
        sessions = [Session(0, 0, clips[0]), Session(1, 1, clips[1], holds=(3,)), Session(2, 2, clips[2]), Session(0, 5, clips[3])]
    else:
        clips = _speech_clips([30 + i % 11 for i in range(B + 2)], seed0=600)
        sessions = [Session(i, i % 3, clips[i], holds=(3,) if i % 7 == 3 else ()) for i in range(B)]
        sessions += [Session(j, 5, clips[B + j]) for j in range(2)]
    m = _fsn(cfg, params)
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    got = _run_chunks(st, sessions, Ks, la)
    st.close()
    for i in ([0, 1, 3] if B == 3 else [1, 40, B]):
        assert torch.equal(got[i], _lone(m, sessions[i], la)), f"session {i} differs from its lone run"
        e = _oracle_err(params, cfg, sessions[i], got[i])
        print(f"\n[B={B} session {i}] layer-wise chunks vs oracle {e:.2e}")
        assert e < MASK_TOL
    mm = _fsn(cfg, params, lstm_impl="mma")
    st, ref = StreamingFullSubNet(mm, batch_size=B, device=DEV), StreamingFullSubNet(mm, batch_size=B, device=DEV)
    got, want = _run_chunks(st, sessions, Ks, la), _run_slots(ref, sessions, Ks, la)
    for i in range(len(sessions)):
        assert torch.equal(got[i], want[i]), f"mma session {i}"
    st.close(); ref.close()


def test_chunks_mixed_with_per_frame_steps(built_lib):
    """Layer-wise chunks alternating with per-frame steps on the same handle: every session within 1e-3 of the oracle; the chunk
    rel-L2 against the per-frame masks is printed."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    la = cfg["look_ahead"]
    clips = _speech_clips([50, 44, 61], seed0=700)
    sessions = [Session(0, 0, clips[0]), Session(1, 1, clips[1]), Session(2, 0, clips[2], holds=(2,))]
    Ks = [4, 3, 32, 5, 8, 16, 8, 32]
    m = _fsn(cfg, params)
    st = StreamingFullSubNet(m, batch_size=3, device=DEV)
    got = _run_chunks(st, sessions, Ks, la, per_frame=(1, 3, 5))
    st.close()
    st = StreamingFullSubNet(m, batch_size=3, device=DEV)
    frame = _run_slots(st, sessions, Ks, la)
    st.close()
    for i, s in enumerate(sessions):
        e, d = _oracle_err(params, cfg, s, got[i]), O.rel_l2(got[i].numpy(), frame[i].numpy())
        print(f"\n[mixed session {i}] vs oracle {e:.2e}, vs per-frame steps {d:.2e}")
        assert e < MASK_TOL


@pytest.mark.parametrize("B_from,B_to", [(3, 80), (80, 3)])
def test_save_after_chunk_and_move(built_lib, B_from, B_to):
    """A session saved right after a chunk call and loaded into a handle of another B continues bit-identically."""
    from fsnplus_b200.streaming import START, STEP, StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    m = _fsn(cfg, params)
    F = 257
    clip = _speech_clips([70], seed0=800)[0]
    s = Session(0, 0, clip)
    a, b = StreamingFullSubNet(m, batch_size=B_from, device=DEV), StreamingFullSubNet(m, batch_size=B_to, device=DEV)
    ref = StreamingFullSubNet(m, batch_size=1, device=DEV)

    def chunk(st, slot, n0, K, first):
        flags = [0] * st.B
        flags[slot] = START if first else STEP
        mag = torch.full((st.B, F, K), float("nan"), device=DEV)
        mag[slot] = _t(s.frames(n0, K))
        mask, nv = st.step_chunk(mag, flags)
        return mask[slot].cpu(), int(nv[slot])

    slot_a, slot_b = B_from - 1, B_to // 2
    r1, _ = chunk(ref, 0, 0, 33, True)
    g1, _ = chunk(a, slot_a, 0, 33, True)
    assert torch.equal(r1, g1)
    state = a.save_slots([slot_a])
    b.load_slots([slot_b], state)
    r2, n2 = chunk(ref, 0, 33, 39, False)
    g2, m2 = chunk(b, slot_b, 33, 39, False)
    assert n2 == m2 == 39 and torch.equal(r2, g2)
    for st in (a, b, ref):
        st.close()


def test_chunk_errors_change_nothing(built_lib):
    """Every error code and message; a failed call leaves the neighbours' state untouched (their next masks are the uninterrupted
    run's)."""
    from fsnplus_b200.streaming import START, STEP, StreamingFullSubNet
    cfg = _small_cfg()
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=21))
    st, ref = StreamingFullSubNet(m, batch_size=4, device=DEV), StreamingFullSubNet(m, batch_size=4, device=DEV)
    lib = st.lib
    x = _t(np.stack(_small_clips([12] * 4, seed=3)))                   # [4, 65, 12]
    out = torch.empty((4, 2, 65, 12), device=DEV)
    valid = (C.c_int32 * 4)()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(flags, K=12, mag=x, dst=out, v=valid, h=st):
        f = None if flags is None else (C.c_int32 * 4)(*flags)
        return lib.fsn_stream_step_chunk(h._st, None if mag is None else C.c_void_p(mag.data_ptr()), K,
                                         None if dst is None else C.c_void_p(dst.data_ptr()), f, v, stream)

    def err():
        return lib.fsn_last_error().decode()

    for s_ in (st, ref):
        s_.step_chunk(x[:, :, :4].contiguous(), [START] * 4)
    for flags, slot in (([1, 1, 3, 0], 2), ([-1, 1, 1, 1], 0), ([0, 0, 0, 7], 3)):
        assert call(flags) == -1 and f"slot {slot}" in err()
    for K in (0, -2):
        assert call([1] * 4, K=K) == -1 and f"K = {K}" in err()
    assert call([1] * 4, K=65535 * 256) == -1 and "chunk limit" in err()
    assert call(None) == -1 and "h_flags" in err()
    assert call([1] * 4, v=None) == -1 and "h_valid" in err()
    assert call([1] * 4, mag=None) == -1 and "d_mag" in err()
    assert call([1] * 4, dst=None) == -1 and "d_mask" in err()
    y = x[:, :, 4:].contiguous()
    a, na = st.step_chunk(y, [STEP] * 4)
    b, nb = ref.step_chunk(y, [STEP] * 4)
    assert torch.equal(a, b) and torch.equal(na, nb)
    au = StreamingFullSubNet(m, batch_size=4, device=DEV)
    au.step_audio(torch.zeros((4, 64), device=DEV), [START] * 4)
    assert call([1] * 4, K=4, h=au) == -3 and "audio" in err()
    torch.cuda.synchronize()
    for s_ in (st, ref, au):
        s_.close()
