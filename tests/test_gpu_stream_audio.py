"""Audio in, audio out on one streaming handle (fsn_stream_step_audio_slots, DESIGN.md §3.10): every session's waveform and masks
must be exactly those of its lone run, its waveform must be the fp64 iSTFT pipeline fed with the masks the call returned (the
transforms), and it must match the offline enhancement of the same audio (end to end).

A schedule is a list of sessions, each on one slot: it STARTs with its first hop, STEPs through the others, then FLUSHes look_ahead + 2
times (plus extra FLUSH ticks, which act as HOLD), skipping its hold ticks.  The sample rows of HOLD and FLUSH slots are NaN."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O
from test_gpu_stream_sessions import DEV, MASK_TOL, _fsn, _small_cfg, _t

pytestmark = pytest.mark.gpu
XFORM_TOL = 1e-5          # streamed waveform vs the fp64 pipeline fed with the returned masks
WAVE_TOL = 2e-3           # streamed waveform vs the offline enhancement (fp64 oracle, offline GPU forward)


class Session:
    def __init__(self, slot, start, x, holds=()):
        self.slot, self.start, self.x, self.holds = slot, start, np.asarray(x, np.float32), set(holds)


def _clips(n, K, hop, seed0, gains=None):
    """n synthetic noisy-speech clips of K[i] hops (O.synth_clips, -25 dBFS +- 10), times gains[i]."""
    x = O.synth_clips(n, num_samples=max(K) * hop, seed0=seed0)
    g = np.ones(n) if gains is None else np.asarray(gains)
    return [(x[i, :K[i] * hop] * g[i]).astype(np.float32) for i in range(n)]


def _plan(sessions, hop, la, extra_flush):
    """tick -> {slot: (session index, flag, hop index or -1)}; every session's ticks and the end of the schedule."""
    from fsnplus_b200.streaming import FLUSH, START, STEP
    steps = {}
    for i, s in enumerate(sessions):
        K = len(s.x) // hop
        assert K * hop == len(s.x) and K >= 2
        seq = [(START, 0)] + [(STEP, q) for q in range(1, K)] + [(FLUSH, -1)] * (la + 2 + extra_flush)
        t = s.start
        for f, q in seq:
            while t in s.holds:
                t += 1
            steps.setdefault(t, {})[s.slot] = (i, f, q)
            t += 1
        s.end = t
    for a in sessions:
        for b in sessions:
            assert a is b or a.slot != b.slot or a.end <= b.start or b.end <= a.start, "sessions overlap on a slot"
    return steps, max(s.end for s in sessions)


def _run(st, sessions, la, extra_flush=2, extra_ticks=0):
    """Step the schedule; return each session's (waveform [L], masks [2, F, K + 1]) on the CPU.  Checks every tick: valid exactly
    where hop q of a session is due (its tick q + la + 2), every other audio row zero, and mask rows zero where no frame is due."""
    from fsnplus_b200.streaming import HOLD
    hop, B, F = st.hop, st.B, st.F
    steps, n_ticks = _plan(sessions, hop, la, extra_flush)
    wav = [[] for _ in sessions]
    masks = [[] for _ in sessions]
    k = [0] * len(sessions)
    for tick in range(n_ticks + extra_ticks):
        flags = np.full(B, HOLD, dtype=np.int32)
        x = np.full((B, hop), np.nan, dtype=np.float32)
        want = np.zeros(B, dtype=bool)
        frame = {}
        for slot, (i, f, q) in steps.get(tick, {}).items():
            s = sessions[i]
            K = len(s.x) // hop
            flags[slot] = f
            if q >= 0:
                x[slot] = s.x[q * hop:(q + 1) * hop]
            want[slot] = 0 <= k[i] - la - 2 < K
            if 0 <= k[i] - la - 1 <= K:
                frame[slot] = i
            k[i] += 1
        out, valid, mask = st.step_audio(_t(x), torch.from_numpy(flags), return_mask=True)
        out, mask = out.cpu(), mask.cpu()
        assert torch.equal(valid, torch.from_numpy(want)), f"tick {tick}: valid {valid.tolist()} != {want.tolist()}"
        assert torch.count_nonzero(out[torch.from_numpy(~want)]) == 0, f"tick {tick}: an audio row without a hop is not zero"
        quiet = torch.ones(B, dtype=torch.bool)
        for slot in frame:
            quiet[slot] = False
        assert torch.count_nonzero(mask[quiet]) == 0, f"tick {tick}: a mask row without a frame is not zero"
        for slot in np.nonzero(want)[0]:
            wav[steps[tick][slot][0]].append(out[slot].clone())
        for slot, i in frame.items():
            masks[i].append(mask[slot].clone())
    res = []
    for s, w, m in zip(sessions, wav, masks):
        K = len(s.x) // hop
        assert len(w) == K and len(m) == K + 1
        res.append((torch.cat(w), torch.stack(m, dim=-1)))
    return res


def _lone(m, B, s, la):
    """The session streamed alone: same slot of a fresh B-slot handle, no holds, no extra FLUSH, every other slot held."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    out = _run(st, [Session(s.slot, 0, s.x)], la, extra_flush=0)[0]
    st.close()
    return out


def _check(m, params, cfg, B, sessions, got, e2e_idx):
    la, F = cfg["look_ahead"], cfg["num_freqs"]
    n_fft = 2 * (F - 1)
    hop = n_fft // 2
    from fsnplus_b200 import inference as inf
    for i, s in enumerate(sessions):
        wav, mask = got[i]
        lw, lm = _lone(m, B, s, la)
        assert torch.equal(wav, lw) and torch.equal(mask, lm), f"session {i} (slot {s.slot}) differs from its lone run"
        X = O.stft(s.x[None].astype(np.float64), n_fft, hop, n_fft)
        ref = O.istft(O.enhance(X, mask.numpy()[None].astype(np.float64)), n_fft, hop, n_fft, length=len(s.x))[0]
        e = O.rel_l2(wav.numpy(), ref)
        print(f"\n[session {i}, slot {s.slot}, K={len(s.x) // hop}] waveform vs fp64 iSTFT of its masks {e:.2e}")
        assert e < XFORM_TOL
    for i in e2e_idx:
        s = sessions[i]
        wav, mask = got[i]
        X = O.stft(s.x[None].astype(np.float64), n_fft, hop, n_fft)
        crm = O.fullsubnet_forward(params, cfg, np.abs(X)[:, None])
        ref = O.istft(O.enhance(X, crm), n_fft, hop, n_fft, length=len(s.x))[0]
        with torch.no_grad():
            off = inf.enhance_batch(m, _t(s.x[None]), n_fft, hop, n_fft, complex_inputs=False)[0].cpu().numpy()
        e_mask, e_ref, e_off = O.rel_l2(mask.numpy(), crm[0]), O.rel_l2(wav.numpy(), ref), O.rel_l2(wav.numpy(), off)
        print(f"[session {i}] masks vs oracle {e_mask:.2e}  waveform vs fp64 pipeline {e_ref:.2e}  vs offline GPU {e_off:.2e}")
        assert e_mask < MASK_TOL and e_ref < WAVE_TOL and e_off < WAVE_TOL


@pytest.mark.parametrize("norm,rnn", [("cumulative_laplace_norm", "LSTM"), ("cumulative_layer_norm", "LSTM"), ("cumulative_laplace_norm", "GRU")])
def test_audio_sessions_small(built_lib, norm, rnn):
    """F = 65 (n_fft 128, hop 64), 4 slots: staggered joins, holds mid-session, an all-held tick (27), slot 0 reused by a quiet
    session after a loud one, a 2-hop session on slot 1, slot 3 never started."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13)
    m = _fsn(cfg, params, lstm_impl="mma")
    la = cfg["look_ahead"]
    A, B_, Cc, D, E = _clips(5, [18, 25, 30, 22, 2], 64, seed0=900, gains=[8.0, 1.0, 1.0, 0.05, 1.0])
    sessions = [Session(0, 0, A), Session(1, 3, B_, holds=(10, 11, 12, 27)), Session(2, 8, Cc, holds=(27,)),
                Session(0, 26, D, holds=(27,)), Session(1, 40, E)]
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    got = _run(st, sessions, la, extra_ticks=3)
    st.close()
    _check(m, params, cfg, 4, sessions, got, range(len(sessions)))


@pytest.mark.parametrize("B", [3, 80])
def test_audio_sessions_default_geometry(built_lib, B):
    """F = 257 (n_fft 512, hop 256): 3 slots run the weight-stationary full-band step, 80 slots the generic one."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg["norm_type"] = "cumulative_laplace_norm"
    params = O.make_params_fsn(cfg, seed=33)
    m = _fsn(cfg, params)
    la = cfg["look_ahead"]
    if B == 3:
        x = _clips(4, [40, 38, 36, 34], 256, seed0=500, gains=[6.0, 1.0, 1.0, 0.1])
        sessions = [Session(0, 0, x[0]), Session(1, 4, x[1], holds=(10, 11)), Session(2, 9, x[2]), Session(0, 50, x[3], holds=(55,))]
        e2e = [1, 3]
    else:
        n = B + 4
        x = _clips(n, [34 + i % 9 for i in range(n)], 256, seed0=600)
        sessions = [Session(i, i % 13, x[i], holds=(i % 13 + 5, i % 13 + 6) if i % 7 == 3 else ()) for i in range(B)]
        sessions += [Session(j, 70, x[B + j], holds=(80,) if j == 1 else ()) for j in range(4)]
        e2e = [3, len(sessions) - 3]
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    got = _run(st, sessions, la)
    st.close()
    _check(m, params, cfg, B, sessions, got, e2e)


@pytest.mark.parametrize("F,la", [(33, 1), (129, 3), (513, 2)])
def test_audio_fft_sizes(built_lib, F, la):
    """One cheap model per remaining FFT size (n_fft 64, 256, 1024), with other look-aheads: 2 slots, one of them a 2-hop session."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg = O.default_fsn_config()
    cfg.update(num_freqs=F, look_ahead=la, sb_num_neighbors=7, sb_model_hidden_size=64, fb_model_hidden_size=96,
               norm_type="cumulative_laplace_norm")
    params = O.make_params_fsn(cfg, seed=41)
    m = _fsn(cfg, params, lstm_impl="mma")
    hop = F - 1
    x = _clips(3, [20, 2, 12], hop, seed0=700 + F)
    sessions = [Session(0, 0, x[0], holds=(5,)), Session(1, 2, x[1]), Session(1, 12, x[2], holds=(14,))]
    st = StreamingFullSubNet(m, batch_size=2, device=DEV)
    got = _run(st, sessions, la)
    st.close()
    _check(m, params, cfg, 2, sessions, got, range(len(sessions)))


def test_audio_call_rejects_bad_arguments(built_lib):
    from fsnplus_b200.streaming import FLUSH, HOLD, START, STEP, StreamingFullSubNet
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    m = _fsn(cfg, O.make_params_fsn(cfg, seed=21), lstm_impl="mma")
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    lib = st.lib
    x = torch.zeros((4, 64), device=DEV)
    out = torch.empty((4, 64), device=DEV)
    valid = (C.c_int32 * 4)()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(flags, v=valid, xp=None, op=None, h=st):
        f = None if flags is None else (C.c_int32 * 4)(*flags)
        xp = C.c_void_p(x.data_ptr()) if xp is None else xp
        op = C.c_void_p(out.data_ptr()) if op is None else op
        return lib.fsn_stream_step_audio_slots(h._st, xp, op, f, v, None, stream)

    def err():
        return lib.fsn_last_error().decode()

    for flags, slot in (([0, 0, 4, 0], 2), ([-1, 0, 0, 0], 0), ([0, 0, 0, 7], 3)):
        assert call(flags) == -1 and f"slot {slot}" in err()
    assert call([STEP, HOLD, HOLD, HOLD]) == -1 and "slot 0" in err() and "without a session" in err()
    assert call([HOLD, FLUSH, HOLD, HOLD]) == -1 and "slot 1" in err()
    assert call(None) == -1 and "h_flags" in err()
    assert call([START] * 4, None) == -1 and "h_valid" in err()
    assert call([START] * 4, xp=C.c_void_p()) == -1 and "d_samples" in err()
    assert call([START] * 4, op=C.c_void_p()) == -1 and "d_out" in err()
    assert call([START, START, HOLD, HOLD]) == 0
    assert call([FLUSH, STEP, HOLD, HOLD]) == -1 and "slot 0" in err() and "at least 2" in err()    # a 1-hop session
    assert call([STEP, STEP, HOLD, HOLD]) == 0
    assert call([FLUSH, STEP, HOLD, HOLD]) == 0
    assert call([STEP, STEP, HOLD, HOLD]) == -1 and "slot 0" in err() and "FLUSH" in err()          # STEP after the flush
    assert call([START, STEP, HOLD, HOLD]) == 0                                                     # a START reuses the slot
    # one handle serves masks or audio, not both
    assert st.lib.fsn_stream_step_slots(st._st, C.c_void_p(x.data_ptr()), C.c_void_p(torch.empty((4, 2, 65), device=DEV).data_ptr()),
                                        (C.c_int32 * 4)(1, 1, 1, 1), valid, stream) == -3
    masks = StreamingFullSubNet(m, batch_size=4, device=DEV)
    masks.step_slots(torch.zeros((4, 65), device=DEV), [START] * 4)
    assert call([START] * 4, h=masks) == -3
    masks2 = StreamingFullSubNet(m, batch_size=4, device=DEV)
    masks2.step(torch.zeros((4, 65), device=DEV))
    assert call([START] * 4, h=masks2) == -3
    torch.cuda.synchronize()
    for s in (st, masks, masks2):
        s.close()
    # n_fft = 2 (num_freqs - 1) must be a power of two from 64 to 1024
    cfg = _small_cfg("cumulative_laplace_norm", "LSTM")
    cfg["num_freqs"] = 100
    odd = StreamingFullSubNet(_fsn(cfg, O.make_params_fsn(cfg, seed=3), lstm_impl="mma"), batch_size=4, device=DEV)
    xo, oo = torch.zeros((4, 99), device=DEV), torch.empty((4, 99), device=DEV)
    assert call([START] * 4, xp=C.c_void_p(xo.data_ptr()), op=C.c_void_p(oo.data_ptr()), h=odd) == -1 and "num_freqs 100" in err()
    odd.close()
