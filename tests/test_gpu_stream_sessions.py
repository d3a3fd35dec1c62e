"""Independent streaming sessions on one handle (fsn_stream_step_slots, DESIGN.md §3.9): sessions that start, hold and end on their
own schedule must get exactly the masks they get streamed alone, and those must match the offline forward and the fp64 oracle.

A schedule is a list of sessions, each on one slot: it STARTs at its first step tick, consumes its clip and then look_ahead zero
frames (the flush), and skips its hold ticks.  Held slots are fed NaN frames, which the step must never read."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MASK_TOL = 1e-3


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _fsn(cfg, params, **kw):
    from fsnplus_b200.model import Model
    m = Model(**cfg, **kw)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    return m.to(DEV).eval()


def _small_cfg(norm, rnn):
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
    """Default-geometry clips: the first lens[i] frames of a synthetic noisy-speech STFT magnitude [257, T]."""
    T = max(lens)
    mag = np.abs(O.stft(O.synth_clips(len(lens), num_samples=256 * (T - 1), seed0=seed0))).astype(np.float32)
    return [np.ascontiguousarray(mag[i, :, :n]) for i, n in enumerate(lens)]


class Session:
    def __init__(self, slot, start, clip, holds=()):
        self.slot, self.start, self.clip, self.holds = slot, start, clip, set(holds)
        self.T = clip.shape[1]


def _plan(sessions, la):
    """tick -> {slot: (session index, k)}: the k-th step of the session (frame k for k < T, else a flush zero frame)."""
    steps = {}
    for i, s in enumerate(sessions):
        t, k = s.start, 0
        while k < s.T + la:
            if t not in s.holds:
                steps.setdefault(t, {})[s.slot] = (i, k)
                k += 1
            t += 1
        s.end = t
    for a in sessions:
        for b in sessions:
            assert a is b or a.slot != b.slot or a.end <= b.start or b.end <= a.start, "sessions overlap on a slot"
    return steps, max(s.end for s in sessions)


def _run(st, sessions, la, extra_ticks=0):
    """Step the schedule; return each session's valid masks [2, F, T] (CPU) and check every other row is zero and not valid."""
    from fsnplus_b200.streaming import HOLD, STEP, START
    steps, n_ticks = _plan(sessions, la)
    B, F = st.B, st.F
    outs = [[] for _ in sessions]
    for tick in range(n_ticks + extra_ticks):
        flags = np.full(B, HOLD, dtype=np.int32)
        frame = np.full((B, F), np.nan, dtype=np.float32)
        want = np.zeros(B, dtype=bool)
        for slot, (i, k) in steps.get(tick, {}).items():
            s = sessions[i]
            flags[slot] = START if k == 0 else STEP
            frame[slot] = s.clip[:, k] if k < s.T else 0.0
            want[slot] = k >= la
        mask, valid = st.step_slots(_t(frame), torch.from_numpy(flags))
        mask = mask.cpu()
        assert torch.equal(valid, torch.from_numpy(want)), f"tick {tick}: valid {valid.tolist()} != {want.tolist()}"
        assert torch.count_nonzero(mask[torch.from_numpy(~want)]) == 0, f"tick {tick}: a row without a valid mask is not zero"
        for slot, (i, k) in steps.get(tick, {}).items():
            if k >= la:
                outs[i].append(mask[slot].clone())
    for s, o in zip(sessions, outs):
        assert len(o) == s.T
    return [torch.stack(o, dim=-1) for o in outs]


def _lone(m, B, s, la):
    """The session streamed alone: same slot of a fresh B-slot handle, no holds, every other slot held."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    out = _run(st, [Session(s.slot, 0, s.clip)], la)[0]
    st.close()
    return out


def _check_sessions(m, params, cfg, B, sessions, got, oracle_idx, off_tol):
    la = cfg["look_ahead"]
    for i, s in enumerate(sessions):
        assert torch.equal(got[i], _lone(m, B, s, la)), f"session {i} (slot {s.slot}) differs from its lone run"
    for i in oracle_idx:
        clip = sessions[i].clip[None, None]
        with torch.no_grad():
            offline = m(_t(clip))[0].cpu().numpy()
        ref = O.fullsubnet_forward(params, cfg, clip)[0]
        g = got[i].numpy()
        e_off, e_ref = O.rel_l2(g, offline), O.rel_l2(g, ref)
        print(f"\n[session {i}, slot {sessions[i].slot}, T={sessions[i].T}] vs offline {e_off:.2e}  vs oracle {e_ref:.2e}")
        assert e_off < off_tol and e_ref < MASK_TOL


@pytest.mark.parametrize("norm,rnn", [("cumulative_laplace_norm", "LSTM"), ("cumulative_layer_norm", "LSTM"), ("cumulative_laplace_norm", "GRU")])
def test_session_schedule_small(built_lib, norm, rnn):
    """4 slots, weight-stationary full-band step: sessions of different lengths joining at different ticks, slot 0 reused after a
    START, a session with holds in the middle, a tick where every slot holds (27), and slot 3 never started."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params, lstm_impl="mma")
    la = cfg["look_ahead"]
    A, B_, Cc, D = _small_clips([18, 25, 30, 22], seed=9)
    sessions = [Session(0, 0, A), Session(1, 3, B_, holds=(10, 11, 12, 27)), Session(2, 8, Cc, holds=(27,)), Session(0, 24, D, holds=(27,))]
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    got = _run(st, sessions, la, extra_ticks=3)
    st.close()
    _check_sessions(m, params, cfg, 4, sessions, got, range(len(sessions)), 1e-4)


@pytest.mark.parametrize("B", [3, 80])
def test_session_schedule_default_geometry(built_lib, B):
    """F = 257, full-band H = 512, sub-band H = 384: 3 slots run the weight-stationary full-band step, 80 slots the generic one.
    Staggered joins, holds, and reuse of the first slots; every session bit-identical to its lone run."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    m = _fsn(cfg, params)
    la = cfg["look_ahead"]
    if B == 3:
        clips = _speech_clips([40, 38, 36, 34], seed0=500)
        sessions = [Session(0, 0, clips[0]), Session(1, 4, clips[1], holds=(10, 11)), Session(2, 9, clips[2]),
                    Session(0, 45, clips[3], holds=(50,))]
    else:
        n = B + 4
        clips = _speech_clips([34 + i % 9 for i in range(n)], seed0=600)
        sessions = [Session(i, i % 13, clips[i], holds=(i % 13 + 5, i % 13 + 6) if i % 7 == 3 else ()) for i in range(B)]
        sessions += [Session(j, 60, clips[B + j], holds=(70,) if j == 1 else ()) for j in range(4)]
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    got = _run(st, sessions, la)
    st.close()
    _check_sessions(m, params, cfg, B, sessions, got, [1, len(sessions) - 1], MASK_TOL)


@pytest.mark.parametrize("B", [3, 70])
def test_slot_call_matches_lockstep_step(built_lib, B):
    """On a fresh handle the slot call with every flag STEP gives fsn_stream_step's masks and valid flags, frame for frame; and so
    does fsn_stream_step on a handle that used the slot call with every slot stepping.  (Before a mask is valid, fsn_stream_step
    leaves d_mask unspecified and the slot call writes zeros, so masks are compared where they are valid.)"""
    from fsnplus_b200.streaming import STEP, StreamingFullSubNet
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=21), lstm_impl="mma")
    T = 15
    x = _t(np.stack(_small_clips([T] * B, seed=4)))          # [B, F, T]
    ref, slots, mixed = (StreamingFullSubNet(m, batch_size=B, device=DEV) for _ in range(3))
    all_step = [STEP] * B
    for t in range(T):
        y = ref.step(x[:, :, t])
        mask, valid = slots.step_slots(x[:, :, t], all_step)
        if t < 6:
            mask2, valid2 = mixed.step_slots(x[:, :, t], all_step)
            valid2 = bool(valid2.all())
        else:
            mask2 = mixed.step(x[:, :, t])
            valid2 = mask2 is not None
        assert bool(valid.all()) == (y is not None) and bool(valid.any()) == (y is not None) and valid2 == (y is not None)
        if y is not None:
            assert torch.equal(mask, y) and torch.equal(mask2, y), f"frame {t}"
    for s in (ref, slots, mixed):
        s.close()


def test_slot_call_rejects_bad_arguments(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=21), lstm_impl="mma")
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    lib = st.lib
    x = torch.zeros((4, 65), device=DEV)
    out = torch.empty((4, 2, 65), device=DEV)
    valid = (C.c_int32 * 4)()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(flags, v=valid):
        f = None if flags is None else (C.c_int32 * 4)(*flags)
        return lib.fsn_stream_step_slots(st._st, C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), f, v, stream)

    for flags, slot in (([1, 1, 3, 0], 2), ([-1, 1, 1, 1], 0), ([0, 0, 0, 7], 3)):
        assert call(flags) == -1
        assert f"slot {slot}" in lib.fsn_last_error().decode()
    assert call(None) == -1 and "h_flags" in lib.fsn_last_error().decode()
    assert call([1, 1, 1, 1], None) == -1 and "h_valid" in lib.fsn_last_error().decode()
    assert call([2, 1, 0, 1]) == 0
    torch.cuda.synchronize()
    st.close()
