"""Park, resume and move streaming sessions (fsn_stream_save_slots / fsn_stream_load_slots, DESIGN.md §3.11): a session saved from one
slot and loaded into another -- of the same handle, of another handle with the same B, or across B and full-band kernels -- must
continue exactly as its lone run (bit-identical where the kernels are the same, within the oracle bars across kernels), and nothing
else on either handle may change.

A Driver ticks one or more handles in lockstep; every live session feeds its next frame (mask mode: clip frames then look_ahead zero
frames; audio mode: START, STEP hops, then look_ahead + 2 FLUSH ticks) on whatever slot it lives in now.  Held rows are NaN."""
import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_stream_audio as A
from oracle import fsn_oracle as O
from test_gpu_stream_sessions import DEV, MASK_TOL, Session, _fsn, _lone, _small_cfg, _small_clips, _speech_clips, _t

pytestmark = pytest.mark.gpu


class Driver:
    def __init__(self, handles, la, audio=False):
        self.h, self.la, self.audio = handles, la, audio
        self.s, self.live, self.raw = {}, set(), []

    def start(self, sid, hn, slot, x):
        from fsnplus_b200.streaming import FLUSH, START, STEP
        st = self.h[hn]
        if self.audio:
            hop = st.hop
            K = len(x) // hop
            seq = [(START, x[:hop])] + [(STEP, x[q * hop:(q + 1) * hop]) for q in range(1, K)] + [(FLUSH, None)] * (self.la + 2)
        else:
            K = x.shape[1]
            seq = [(START if k == 0 else STEP, x[:, k] if k < K else np.zeros(x.shape[0], np.float32)) for k in range(K + self.la)]
        self.s[sid] = dict(h=hn, slot=slot, k=0, seq=seq, K=K, out=[], mask=[], x=x, slot0=slot, B0=st.B)
        self.live.add(sid)

    def tick(self):
        from fsnplus_b200.streaming import HOLD
        feed = {}
        for hn, st in self.h.items():
            W = st.hop if self.audio else st.F
            feed[hn] = (np.full(st.B, HOLD, np.int32), np.full((st.B, W), np.nan, np.float32))
        for sid in self.live:
            s = self.s[sid]
            f, row = s["seq"][s["k"]]
            flags, x = feed[s["h"]]
            assert flags[s["slot"]] == HOLD, f"two sessions on slot {s['slot']}"
            flags[s["slot"]] = f
            if row is not None:
                x[s["slot"]] = row
        res = {}
        for hn, st in self.h.items():
            flags, x = feed[hn]
            if self.audio:
                out, valid, mask = st.step_audio(_t(x), torch.from_numpy(flags), return_mask=True)
                res[hn] = (out.cpu(), valid, mask.cpu())
            else:
                mask, valid = st.step_slots(_t(x), torch.from_numpy(flags))
                res[hn] = (mask.cpu(), valid)
        self.raw.append(res)
        for sid in sorted(self.live):
            s = self.s[sid]
            r, k, slot = res[s["h"]], s["k"], s["slot"]
            if self.audio:
                if r[1][slot]:
                    s["out"].append(r[0][slot].clone())
                if 0 <= k - self.la - 1 <= s["K"]:
                    s["mask"].append(r[2][slot].clone())
            else:
                assert bool(r[1][slot]) == (k >= self.la)
                if k >= self.la:
                    s["out"].append(r[0][slot].clone())
            s["k"] += 1
        self.live -= {sid for sid in self.live if self.s[sid]["k"] == len(self.s[sid]["seq"])}

    def run(self, n):
        for _ in range(n):
            self.tick()

    def finish(self):
        while self.live:
            self.tick()

    def save(self, sids):
        hn = self.s[sids[0]]["h"]
        return self.h[hn].save_slots([self.s[i]["slot"] for i in sids])

    def place(self, sids, state, hn, slots):
        """Load `state` (session i = sids[i]) into `slots` of handle hn; the sessions continue there."""
        self.h[hn].load_slots(slots, state)
        for sid, slot in zip(sids, slots):
            self.s[sid].update(h=hn, slot=slot)
            self.live.add(sid)

    def fork(self, sid, new, hn, slot):
        state = self.save([sid])
        s = self.s[sid]
        self.s[new] = dict(s, out=list(s["out"]), mask=list(s["mask"]))
        self.place([new], state, hn, [slot])

    def park(self, sid):
        state = self.save([sid])
        self.live.discard(sid)
        return state

    def result(self, sid):
        s = self.s[sid]
        assert sid not in self.live
        if self.audio:
            assert len(s["out"]) == s["K"] and len(s["mask"]) == s["K"] + 1
            return torch.cat(s["out"]), torch.stack(s["mask"], dim=-1)
        assert len(s["out"]) == s["K"]
        return torch.stack(s["out"], dim=-1)


def _lone_of(m, d, sid):
    """The session streamed alone on a fresh handle of the B and slot it started on."""
    s = d.s[sid]
    if d.audio:
        return A._lone(m, s["B0"], A.Session(s["slot0"], 0, s["x"]), d.la)
    return _lone(m, s["B0"], Session(s["slot0"], 0, s["x"]), d.la)


def _same(a, b):
    return all(torch.equal(x, y) for x, y in zip(a, b)) if isinstance(a, tuple) else torch.equal(a, b)


def _rel(a, b):
    a, b = (a[0], b[0]) if isinstance(a, tuple) else (a, b)
    return O.rel_l2(a.numpy(), b.numpy())


def _model(kind):
    if kind == "default":
        cfg = O.default_fsn_config()
        cfg["norm_type"] = "cumulative_laplace_norm"
        params = O.make_params_fsn(cfg, seed=33)
        return cfg, params, _fsn(cfg, params)
    norm, rnn, layers = {"laplace": ("cumulative_laplace_norm", "LSTM", 2), "layer": ("cumulative_layer_norm", "LSTM", 2),
                         "gru": ("cumulative_laplace_norm", "GRU", 2), "lstm3": ("cumulative_laplace_norm", "LSTM", 3)}[kind]
    cfg = _small_cfg(norm, rnn)
    params = O.make_params_fsn(cfg, seed=13, num_layers=layers)
    return cfg, params, _fsn(cfg, params, lstm_impl="mma", num_layers=layers)


def _clips(kind, lens, seed):
    return _speech_clips(lens, seed0=seed) if kind == "default" else _small_clips(lens, seed)


CASES = [("laplace", 4), ("layer", 4), ("gru", 4), ("lstm3", 4), ("default", 3), ("default", 80)]


@pytest.mark.parametrize("kind,B", CASES)
@pytest.mark.parametrize("wait", [0, 1])
def test_fork_park_resume(built_lib, kind, B, wait):
    """On one handle: a fork inside the look-ahead (after 2 frames), a park mid-clip with another session STARTed in the parked slot,
    the parked session resumed into a different slot `wait` ticks later (both tick parities of the weight-stationary step), and a fork
    mid-flush.  Every session, forks included, is bit-identical to its lone run."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model(kind)
    la = cfg["look_ahead"]
    a, b, c = _clips(kind, [20, 22, 6], 71)
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    d = Driver({"h": st}, la)
    d.start(0, "h", 0, a)
    d.start(1, "h", 1, b)
    d.run(2)
    d.fork(0, 10, "h", 2)                       # frames consumed: 2 <= look_ahead
    d.run(8)
    parked = d.park(1)                          # mid-clip (10 of 22 frames)
    d.start(2, "h", 1, c)                       # another session in the parked slot: 6 frames + flush, ticks 10..17
    assert la >= 2
    while d.s[0]["k"] < d.s[0]["K"] + la - 1:   # session 0 inside its flush, one zero frame to go
        d.tick()
    assert 2 not in d.live
    d.fork(0, 11, "h", 1)                       # mid-flush, into the slot session 2 has left
    d.run(1 + wait)                             # sessions 0, 10 and 11 end: slot 2 is free
    d.place([1], parked, "h", [2])              # resumed in another slot, at tick parity 22 + wait
    d.finish()
    st.close()
    for sid in (0, 10, 11, 1, 2):
        assert _same(d.result(sid), _lone_of(m, d, sid)), f"session {sid} differs from its lone run"
    if kind == "default":
        ref = O.fullsubnet_forward(params, cfg, b[None, None])[0]
        e = O.rel_l2(d.result(1).numpy(), ref)
        print(f"\n[{kind} B={B}] parked session vs oracle {e:.2e}")
        assert e < MASK_TOL


@pytest.mark.parametrize("B,slots", [(3, [0, 1, 2]), (80, [0, 37, 64, 79])])
def test_start_after_random_load(built_lib, B, slots):
    """A START zeroes every byte of recurrent state a load can write, in the exchange-buffer parity its tick reads: payloads of seeded
    random bytes with valid metas are loaded into slots, then sessions START there, one per tick (both tick parities), at 3 slots
    (weight-stationary full band) and 80 slots (generic full band).  Every session is bit-identical to its lone run."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, _, m = _model("default")
    la = cfg["look_ahead"]
    clips = _clips("default", [9 + i for i in range(len(slots))], 41)
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    d = Driver({"h": st}, la)
    d.run(1)                                    # an all-held tick: the handle serves masks
    state = st.save_slots(slots)
    g = torch.Generator().manual_seed(B)
    state.payload.copy_(torch.randint(0, 256, tuple(state.payload.shape), dtype=torch.uint8, generator=g))
    st.load_slots(slots, state)
    for i, slot in enumerate(slots):
        d.start(i, "h", slot, clips[i])
        d.run(1)
    d.finish()
    st.close()
    for i, slot in enumerate(slots):
        assert _same(d.result(i), _lone_of(m, d, i)), f"session {i} (slot {slot}) differs from its lone run"


def test_neighbours_untouched(built_lib):
    """Every slot that is not loaded into gives, tick by tick, exactly the rows of the same schedule without the save and load calls
    (failed calls included)."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, _, m = _model("laplace")
    la = cfg["look_ahead"]
    a, b, c = _clips("laplace", [16, 18, 14], 5)
    runs = []
    for calls in (False, True):
        st = StreamingFullSubNet(m, batch_size=5, device=DEV)
        d = Driver({"h": st}, la)
        d.start(0, "h", 0, a)
        d.start(1, "h", 1, b)
        d.run(3)
        d.start(2, "h", 2, c)
        d.run(4)
        if calls:
            state = d.save([1])
            d.h["h"].load_slots([4], state)     # a copy of session 1 in slot 4, never stepped
            with pytest.raises(Exception):
                d.h["h"].load_slots([4, 4], d.save([0, 1]))
        d.finish()
        runs.append(d.raw)
        st.close()
    for t, (r0, r1) in enumerate(zip(*runs)):
        assert torch.equal(r0["h"][0][:4], r1["h"][0][:4]) and torch.equal(r0["h"][1][:4], r1["h"][1][:4]), f"tick {t}"


@pytest.mark.parametrize("kind,B", [("laplace", 4), ("default", 3), ("default", 80)])
def test_migrate_same_b_and_host_round_trip(built_lib, kind, B):
    """Sessions moved to a second handle with the same B (one directly, one through pinned host memory and back) continue
    bit-identically; the host round trip returns the payload bytes unchanged."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, _, m = _model(kind)
    la = cfg["look_ahead"]
    a, b = _clips(kind, [18, 21], 17)
    h = {"a": StreamingFullSubNet(m, batch_size=B, device=DEV), "b": StreamingFullSubNet(m, batch_size=B, device=DEV)}
    d = Driver(h, la)
    d.start(0, "a", 0, a)
    d.start(1, "a", 1, b)
    d.run(3)
    d.start(2, "b", 1, a)                       # something else already runs on the destination handle
    d.run(4)
    s0 = d.park(0)
    s1 = d.park(1)
    host = s1.to("cpu")
    assert host.payload.is_pinned() and torch.equal(host.to(DEV).payload, s1.payload)
    d.place([0], s0, "b", [B - 1])
    d.place([1], host, "b", [0])
    d.finish()
    for sid in (0, 1, 2):
        assert _same(d.result(sid), _lone_of(m, d, sid)), f"session {sid}"
    for s in h.values():
        s.close()


@pytest.mark.parametrize("kind", ["laplace", "default"])
def test_migrate_across_b_and_kernels(built_lib, kind):
    """3 -> 80 and 80 -> 3 slots (weight-stationary <-> generic full-band step): masks within 1e-4 rel-L2 of the lone run (small
    geometry) and within the oracle bar; 3 -> 5 and 80 -> 96 (same kernel, another B) are bit-identical."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model(kind)
    la = cfg["look_ahead"]
    clips = _clips(kind, [24, 22, 20, 19], 23)
    pairs = [(3, 80), (80, 3), (3, 5), (80, 96)]
    for (src, dst), x in zip(pairs, clips):
        h = {"s": StreamingFullSubNet(m, batch_size=src, device=DEV), "d": StreamingFullSubNet(m, batch_size=dst, device=DEV)}
        d = Driver(h, la)
        d.start(0, "s", 1, x)
        d.run(9)
        d.place([0], d.park(0), "d", [dst - 1])
        d.finish()
        got, lone = d.result(0), _lone_of(m, d, 0)
        ref = O.fullsubnet_forward(params, cfg, x[None, None])[0]
        e_lone, e_ref = _rel(got, lone), O.rel_l2(got.numpy(), ref)
        print(f"\n[{kind}] {src} -> {dst} slots: vs lone run {e_lone:.2e}  vs oracle {e_ref:.2e}  bit-identical {_same(got, lone)}")
        assert e_ref < MASK_TOL
        if kind != "default":
            assert e_lone < 1e-4
        if (src, dst) in ((3, 5), (80, 96)):
            assert _same(got, lone)
        for s in h.values():
            s.close()


def test_all_slots_in_one_call(built_lib):
    """80 sessions saved in one call and loaded in one call, permuted, into a fresh 80-slot handle all continue bit-identically to the
    source handle, which keeps stepping them."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, _, m = _model("laplace")
    la = cfg["look_ahead"]
    B = 80
    clips = _clips("laplace", [14 + i % 5 for i in range(B)], 3)
    h = {"a": StreamingFullSubNet(m, batch_size=B, device=DEV), "b": StreamingFullSubNet(m, batch_size=B, device=DEV)}
    d = Driver(h, la)
    for i in range(B):
        d.start(i, "a", i, clips[i])
    d.run(2)
    for i in range(B):                          # staggered: sessions at different frame counts when saved
        if i % 3 == 0:
            d.live.discard(i)
    d.run(3)
    d.live |= {i for i in range(B) if i % 3 == 0}
    state = d.save(list(range(B)))
    assert len(state) == B and state[[0, 3]].meta[1].frames == 2 and state[1].meta[0].frames == 5
    perm = np.random.default_rng(1).permutation(B).tolist()
    for i in range(B):
        d.s[B + i] = dict(d.s[i], out=list(d.s[i]["out"]), mask=[])
    d.place([B + i for i in range(B)], state, "b", perm)
    d.finish()
    for i in range(B):
        assert torch.equal(d.result(i), d.result(B + i)), f"session {i}"
    for s in h.values():
        s.close()


def test_lockstep_handle_switches_to_slot_counts(built_lib):
    """A handle that has only used fsn_stream_step keeps giving the same masks after a save (it switches to per-slot counts)."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, _, m = _model("laplace")
    x = _t(np.stack(_clips("laplace", [12] * 3, 8)))
    a, b = StreamingFullSubNet(m, batch_size=3, device=DEV), StreamingFullSubNet(m, batch_size=3, device=DEV)
    for t in range(12):
        ya, yb = a.step(x[:, :, t]), b.step(x[:, :, t])
        if t == 4:
            st = a.save_slots([0, 2])
            assert [st.meta[i].frames for i in range(2)] == [5, 5]
        assert (ya is None) == (yb is None) and (ya is None or torch.equal(ya, yb)), f"frame {t}"
    a.close()
    b.close()


@pytest.mark.parametrize("kind", ["laplace", "layer", "gru"])
def test_audio_park_resume(built_lib, kind):
    """Audio sessions: a fork right after START (tick 1), a park mid-session with another session STARTed in the slot, resumed into a
    different slot, and a fork between FLUSH ticks.  Waveforms and masks bit-identical to the lone runs."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, _, m = _model(kind)
    la = cfg["look_ahead"]
    a, b, c = A._clips(3, [16, 18, 3], 64, seed0=321)
    st = StreamingFullSubNet(m, batch_size=4, device=DEV)
    d = Driver({"h": st}, la, audio=True)
    d.start(0, "h", 0, a)
    d.start(1, "h", 1, b)
    d.run(1)
    d.fork(0, 10, "h", 2)                       # right after START
    d.run(7)
    parked = d.park(1)
    d.start(2, "h", 1, c)
    d.run(3)
    d.place([1], parked, "h", [3])
    while d.s[0]["k"] < d.s[0]["K"] + 2:        # between FLUSH ticks (the first FLUSH is slot tick K)
        d.tick()
    assert 2 not in d.live
    d.fork(0, 11, "h", 1)
    d.finish()
    st.close()
    for sid in (0, 10, 11, 1, 2):
        assert _same(d.result(sid), _lone_of(m, d, sid)), f"session {sid} differs from its lone run"


def test_audio_across_kernels(built_lib):
    """Audio sessions moved 3 -> 80 and 80 -> 3 slots: waveform within the 2e-3 bar of the fp64 pipeline."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("laplace")
    la, F = cfg["look_ahead"], cfg["num_freqs"]
    n_fft = 2 * (F - 1)
    hop = n_fft // 2
    xs = A._clips(2, [20, 22], hop, seed0=55)
    for (src, dst), x in zip([(3, 80), (80, 3)], xs):
        h = {"s": StreamingFullSubNet(m, batch_size=src, device=DEV), "d": StreamingFullSubNet(m, batch_size=dst, device=DEV)}
        d = Driver(h, la, audio=True)
        d.start(0, "s", 0, x)
        d.run(9)
        d.place([0], d.park(0), "d", [dst - 1])
        d.finish()
        wav, mask = d.result(0)
        X = O.stft(x[None].astype(np.float64), n_fft, hop, n_fft)
        crm = O.fullsubnet_forward(params, cfg, np.abs(X)[:, None])
        ref = O.istft(O.enhance(X, crm), n_fft, hop, n_fft, length=len(x))[0]
        e_ref, e_lone = O.rel_l2(wav.numpy(), ref), _rel(d.result(0), _lone_of(m, d, 0))
        print(f"\n[audio] {src} -> {dst} slots: waveform vs fp64 pipeline {e_ref:.2e}  vs lone run {e_lone:.2e}")
        assert e_ref < A.WAVE_TOL
        for s in h.values():
            s.close()


def test_errors_change_nothing(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import SessionState, StreamingFullSubNet
    cfg, params, m = _model("laplace")
    la = cfg["look_ahead"]
    a, b = _clips("laplace", [20, 20], 9)
    h = {"h": StreamingFullSubNet(m, batch_size=4, device=DEV), "ref": StreamingFullSubNet(m, batch_size=4, device=DEV)}
    lib = h["h"].lib
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    err = lambda: lib.fsn_last_error().decode()      # noqa: E731
    fresh = StreamingFullSubNet(m, batch_size=4, device=DEV)
    buf = torch.empty((1, 1 << 20), dtype=torch.uint8, device=DEV)
    meta = (_lib.FsnSlotMeta * 1)()
    assert lib.fsn_stream_save_slots(fresh._st, 1, (C.c_int32 * 1)(0), C.c_void_p(buf.data_ptr()), meta, stream) == -3
    assert lib.fsn_stream_state_bytes(fresh._st) == -3
    d = Driver(h, la)
    for hn in h:
        d.start(hn + "0", hn, 0, a)
        d.start(hn + "1", hn, 2, b)
    d.run(6)
    st = d.h["h"].save_slots([0, 2])

    def load(slots, state=st, meta=None, ptr=None, n=None, handle=None):
        s = (C.c_int32 * len(slots))(*slots)
        return lib.fsn_stream_load_slots((handle or d.h["h"])._st, len(slots) if n is None else n, s,
                                         C.c_void_p(state.payload.data_ptr() if ptr is None else ptr), state.meta if meta is None else meta, stream)

    def tampered(**kw):
        q = (_lib.FsnSlotMeta * 2)(*st.meta)
        for k, v in kw.items():
            if k.startswith("cfg."):
                setattr(q[1].cfg, k[4:], v)
            else:
                setattr(q[1], k, v)
        return q

    c0 = st.meta[0].cfg
    for field, v in (("look_ahead", c0.look_ahead + 1), ("sb_hidden", c0.sb_hidden + 16), ("fb_hidden", c0.fb_hidden * 2),
                     ("rnn_type", 1 - c0.rnn_type), ("fast_math", 1 - c0.fast_math), ("norm_type", 3 if c0.norm_type == 1 else 1)):
        assert load([1, 3], meta=tampered(**{"cfg." + field: v})) == -1 and "h_meta[1]" in err() and f"cfg.{field}" in err(), field
    assert load([1, 3], meta=tampered(version=2)) == -1 and "version" in err()
    assert load([1, 3], meta=tampered(magic=0)) == -1 and "magic" in err()
    assert load([1, 3], meta=tampered(payload_bytes=st.meta[1].payload_bytes + 256)) == -1 and "payload_bytes" in err()
    assert load([1, 3], meta=tampered(weights_id=st.meta[1].weights_id ^ 1)) == -1 and "weights_id" in err()
    assert load([1, 3], meta=tampered(mode=2)) == -3
    assert load([1, 3], meta=tampered(mode=5)) == -1 and "mode 5" in err()
    assert load([1, 1]) == -1 and "h_slots[1]" in err() and "twice" in err()
    assert load([1, 4]) == -1 and "h_slots[1]" in err() and "out of range" in err()
    assert load([1], n=0) == -1
    host = torch.empty(st.payload.shape, dtype=torch.uint8)
    assert load([1, 3], ptr=host.data_ptr()) == -1 and "device memory" in err()
    assert load([1, 3], ptr=st.payload.data_ptr() + 16) == -1 and "256-byte" in err()
    # equal weights: equal weights_id, the load succeeds; one element changed: FSN_EINVAL
    m2 = _fsn(cfg, params, lstm_impl="mma")
    p3 = {k: v.copy() for k, v in params.items()}
    p3["sb_model.fc_output_layer.bias"][1] += 1e-3
    m3 = _fsn(cfg, p3, lstm_impl="mma")
    h2, h3 = StreamingFullSubNet(m2, batch_size=4, device=DEV), StreamingFullSubNet(m3, batch_size=4, device=DEV)
    assert m.weights_id() == m2.weights_id() != 0 and m3.weights_id() != m.weights_id()
    assert m2._cfg.lstm_impl == _lib.LSTM_IMPL["mma"]
    assert load([3, 1], meta=tampered(**{"cfg.lstm_impl": _lib.LSTM_IMPL["auto"]}), handle=h2) == 0   # lstm_impl is not compared
    with pytest.raises(_lib.FsnError, match="weights_id"):
        h3.load_slots([3, 1], st)
    # mode mismatch: an audio session into a mask handle, and into a fresh handle that a mask load has claimed
    au = StreamingFullSubNet(m, batch_size=4, device=DEV)
    au.step_audio(torch.zeros((4, au.hop), device=DEV), [2, 0, 0, 0])
    ast = au.save_slots([0])
    assert ast.meta[0].mode == 2 and ast.meta[0].tick == 1
    assert load([1], state=ast) == -3
    fresh.load_slots([1], SessionState(st.payload[1:], (_lib.FsnSlotMeta * 1)(st.meta[1])))
    assert lib.fsn_stream_state_bytes(fresh._st) == st.meta[0].payload_bytes
    assert load([0], state=ast, handle=fresh) == -3
    for s in (h2, h3, au, fresh):
        s.close()
    # the failed calls changed nothing: the handle continues exactly like the reference handle
    d.finish()
    for sid in ("0", "1"):
        assert torch.equal(d.result("h" + sid), d.result("ref" + sid))
    for s in h.values():
        s.close()
