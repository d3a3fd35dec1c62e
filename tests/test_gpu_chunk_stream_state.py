"""Park, resume and move overlapped-chunk sessions on the device (fsn_chunk_stream_save_slots / _load_slots, ChunkStream.save_slots /
load_slots; DESIGN.md §3.17).

Every session that is parked, resumed, forked or moved -- within one handle, between handles of another B, through host memory, to a
second GPU -- is bit-identical to its uninterrupted lone run on a 1-slot handle.  A session handed over from model to model (other
weights, the sub-band TCN, fullsubnet.Model with an offline norm) equals the fp64 stitch of each model's enhance_audio rows for the
chunks that model enhanced.  Loads leave neighbouring slots alone and never read the payload's padding; every refused call is
followed by a step that must equal a twin handle that never saw it."""
import ctypes as C

import numpy as np
import pytest
import torch

import chunk_stream_ref as R
import sbtcn_oracle as SB
from chunk_stream_ref import P, SLOT_FLUSH, SLOT_HOLD, SLOT_START, SLOT_STEP
from oracle import fsn_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
STITCH_TOL = 1e-6         # a session vs the fp64 stitch of enhance_audio on its chunk rows (DESIGN.md §3.16)
S = 300                   # samples per call row


def _model(kind, seed, dev=DEV):
    """A small FullSubNet+ ("plus"), the same with the sub-band TCN ("tcn") or a small fullsubnet.Model with offline_laplace_norm
    ("fsn"), all at F = 33, on dev."""
    from fsnplus_b200.model import FullSubNet_Plus, Model
    cfg = O.default_plus_config()
    cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    cls = FullSubNet_Plus
    if kind == "plus":
        params = O.make_params_plus(cfg, seed=seed)
    elif kind == "tcn":
        cfg.update(sb_model_hidden_size=32, sequence_model="TCN")
        params = SB.make_params(cfg, seed=seed)
    else:
        cls, cfg = Model, O.default_fsn_config()
        cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48)
        assert cfg["norm_type"] == "offline_laplace_norm"
        params = O.make_params_fsn(cfg, seed=seed)
    m = cls(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(dev).eval()
    with torch.cuda.device(dev):
        m._ensure_handle(torch.device(dev))
    return m


_MODELS = {}


def _cached(kind="plus", seed=3):
    if (kind, seed) not in _MODELS:
        _MODELS[kind, seed] = _model(kind, seed)
    return _MODELS[kind, seed]


def _bank(seed, n=200000):
    return O.synth_clips(2, num_samples=n, seed0=seed).reshape(-1).astype(np.float32)


class Mux:
    """Drives one ChunkStream and keeps, per logical session, its calls (flag, count, samples) and its outputs wherever it runs.
    ``slot[b]``: the session slot b serves (None: free); ``sessions``: every session so far.  Each session draws its counts and
    samples from its own generator, so two Mux with the same seed feed the same sessions the same input whatever else they do."""

    def __init__(self, cs, bank, seed, sessions=None):
        self.cs, self.bank, self.seed = cs, bank, seed
        self.slot = [None] * cs.B
        self.sessions = [] if sessions is None else sessions

    def call(self, plan, Sr=S):
        """plan {slot: (flag, count)}, every other slot HOLDs."""
        B = self.cs.B
        fl, ct = [SLOT_HOLD] * B, [0] * B
        Sr = max([Sr] + [c for _, c in plan.values()])
        x = np.full((B, Sr), np.nan, np.float32)
        for b, (f, c) in plan.items():
            fl[b], ct[b] = f, c
            o = int(self.slot[b]["rng"].integers(0, self.bank.shape[0] - c))
            x[b, :c] = self.bank[o:o + c]
        out, nout = self.cs.step(torch.from_numpy(x).to(self.cs.device), ct, fl)
        out, nout = out.cpu().numpy(), nout.numpy()
        for b in range(B):
            if b not in plan:
                assert nout[b] == 0 and not out[b].any()
        for b, (f, c) in plan.items():
            s = self.slot[b]
            n = int(nout[b])
            s["calls"].append((f, c, x[b, :c].copy()))
            s["ys"].append(out[b, :n].copy())
            s["n"] += c
            assert not out[b, n:].any() and np.isfinite(out[b, :n]).all()
            if f == SLOT_FLUSH:
                s["done"] = True
                self.slot[b] = None
        return out, nout

    def auto(self, force=None, keep=()):
        """One call: every served slot not in `keep` steps a random count (force {slot: count} overrides it), FLUSH once its session's
        input ends."""
        plan = {}
        for b, s in enumerate(self.slot):
            if s is None or b in keep:
                continue
            c = force[b] if force and b in force else int(s["rng"].integers(0, S + 1))
            c = min(c, s["L"] - s["n"])
            plan[b] = (SLOT_FLUSH if s["n"] + c >= s["L"] else SLOT_STEP, c)
        return self.call(plan)

    def start(self, b, L, c):
        s = dict(L=L, n=0, calls=[], ys=[], done=False, rng=np.random.default_rng((self.seed, len(self.sessions))))
        self.sessions.append(s)
        self.slot[b] = s
        return self.call({b: (SLOT_START, c)})

    def put(self, b, s):
        self.slot[b] = s
        if not any(t is s for t in self.sessions):
            self.sessions.append(s)

    def finish(self):
        while any(s is not None for s in self.slot):
            self.auto()


def _fork(s, extra, seed):
    return dict(L=s["L"] + extra, n=s["n"], calls=list(s["calls"]), ys=list(s["ys"]), done=False, rng=np.random.default_rng(seed))


def _y(s):
    return np.concatenate(s["ys"]) if s["ys"] else np.zeros(0, np.float32)


def _alone(m, Cc, s, dev=DEV):
    """The session's calls on a fresh 1-slot handle of model m: its concatenated output."""
    from fsnplus_b200.streaming import ChunkStream
    cs = ChunkStream(m, 1, Cc, dev)
    ys = []
    for f, c, xs in s["calls"]:
        x = np.full((1, max(c, 1)), np.nan, np.float32)
        x[0, :c] = xs
        out, nout = cs.step(torch.from_numpy(x).to(dev), [c], [f])
        ys.append(out.cpu().numpy()[0, :int(nout[0])])
    cs.close()
    return np.concatenate(ys)


def _check_alone(m, Cc, sessions, what):
    for i, s in enumerate(sessions):
        assert s["done"], (what, i)
        y = _y(s)
        assert y.shape[0] == s["n"], (what, i, y.shape, s["n"])
        assert np.array_equal(y, _alone(m, Cc, s)), (what, i, s["n"])
    print(f"\n[{what}] {len(sessions)} sessions bit-identical to their lone runs")


def _to_mid_chunk(s, H, want):
    """The count that takes session s to `want` samples into a half-chunk (0 < want < H)."""
    return (want - s["n"]) % H


@pytest.mark.parametrize("Cc", [512, 514, 640])
def test_fork_park_resume_one_handle(built_lib, Cc):
    """Staggered sessions on 4 slots; one parked mid-chunk while another session uses its slot, then resumed into a different slot;
    one forked into a free slot, both copies stepping on with their own input; one resumed into another slot and flushed at once.
    Every session is bit-identical to its lone run.  C = 514 has 8-byte ring rows and an odd half-chunk; 512 and 640 16-byte rows."""
    from fsnplus_b200.streaming import ChunkStream
    m = _cached()
    H = Cc // 2
    cs = ChunkStream(m, 4, Cc, DEV)
    mx = Mux(cs, _bank(21), seed=Cc)
    mx.start(0, 11 * H + 17, 200)
    mx.auto(force={0: S})
    mx.start(1, 9 * H + 3, 5)
    for _ in range(3):
        mx.auto(force={0: S})
    mx.start(2, 3 * H, 0)
    mx.auto(force={0: _to_mid_chunk(mx.slot[0], H, H // 3)})
    a = mx.slot[0]
    assert a["n"] % H == H // 3 and a["n"] > 2 * H
    parked = cs.save_slots([0])                            # park A mid-chunk; slot 0 serves another session meanwhile
    assert (parked.meta[0].samples, parked.meta[0].chunks) == (a["n"], a["n"] // H - 1)
    mx.slot[0] = None
    mx.start(0, 2 * H + 50, S)
    for _ in range(2):
        mx.auto()
    while mx.slot[2] is not None:                          # end slot 2's session: A resumes there
        mx.auto(keep=(0, 1))
    cs.load_slots([2], parked)
    mx.put(2, a)
    mx.auto()
    b = mx.slot[1]                                         # fork B into slot 3
    assert b is not None and b["n"] > 0 and mx.slot[3] is None
    cs.load_slots([3], cs.save_slots([1]))
    mx.put(3, _fork(b, 3 * H, 99))
    for _ in range(2):
        mx.auto()
    x = mx.slot[0]                                         # end the session that used A's slot meanwhile
    if x is not None:
        mx.call({0: (SLOT_FLUSH, min(S, x["L"] - x["n"]))})
    busy = [i for i, s in enumerate(mx.slot) if s is not None]
    free = [i for i, s in enumerate(mx.slot) if s is None]
    assert busy and free
    st = cs.save_slots([busy[0]])                          # a resume followed at once by FLUSH, in another slot
    s = mx.slot[busy[0]]
    mx.slot[busy[0]] = None
    cs.load_slots([free[0]], st)
    mx.put(free[0], s)
    mx.call({free[0]: (SLOT_FLUSH, min(S, s["L"] - s["n"]))})
    mx.finish()
    assert len(mx.sessions) == 5
    _check_alone(m, Cc, mx.sessions, f"one handle C={Cc}")


def test_move_between_handles_and_through_host(built_lib):
    """3 sessions saved from a 3-slot handle in one call and loaded permuted into an 80-slot handle in one call; there, 5 sessions
    saved in one call and loaded permuted into a 5-slot handle, one of them through .to("cpu") and back (payload bytes unchanged).
    Every session is bit-identical to its lone run."""
    from fsnplus_b200.streaming import ChunkStream
    m = _cached()
    Cc = 512
    H = Cc // 2
    sessions = []
    bank = _bank(22)
    a = Mux(ChunkStream(m, 3, Cc, DEV), bank, 1, sessions)
    for b in range(3):
        a.start(b, 8 * H + 31 * b, 100 + b)
        a.auto()
    st = a.cs.save_slots([0, 1, 2])
    moved = list(a.slot)
    a.cs.close()
    big = Mux(ChunkStream(m, 80, Cc, DEV), bank, 2, sessions)
    dst = [77, 5, 40]
    big.cs.load_slots(dst, st)
    for b, s in zip(dst, moved):
        big.put(b, s)
    big.start(12, 7 * H, 40)
    big.start(79, 9 * H, 250)
    for _ in range(3):
        big.auto(keep=())
    src = [b for b in (77, 5, 40, 12, 79) if big.slot[b] is not None]
    assert len(src) == 5
    st = big.cs.save_slots(src)
    host = st.to("cpu")
    assert host.payload.device.type == "cpu" and host.payload.is_pinned()
    back = host.to(DEV)
    assert torch.equal(back.payload.cpu(), st.payload.cpu())
    assert bytes(back.meta[3]) == bytes(st.meta[3])
    moved = [big.slot[b] for b in src]
    big.cs.close()
    small = Mux(ChunkStream(m, 5, Cc, DEV), bank, 3, sessions)
    perm = [4, 2, 0, 1, 3]
    small.cs.load_slots(perm[:3], st[[0, 1, 2]])
    small.cs.load_slots(perm[3:], host[[3, 4]])            # loaded from host memory: copied to the device first
    for b, s in zip(perm, moved):
        small.put(b, s)
    small.finish()
    small.cs.close()
    assert len(sessions) == 5
    _check_alone(m, Cc, sessions, "moved 3 -> 80 -> 5")


def test_move_to_second_gpu(built_lib):
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    from fsnplus_b200.streaming import ChunkStream
    m0, m1 = _cached(), _model("plus", 3, "cuda:1")
    Cc, H = 512, 256
    sessions = []
    a = Mux(ChunkStream(m0, 2, Cc, DEV), _bank(23), 4, sessions)
    a.start(0, 7 * H + 1, 300)
    a.start(1, 5 * H + 9, 1)
    for _ in range(3):
        a.auto()
    st = a.cs.save_slots([0, 1])
    moved = list(a.slot)
    a.cs.close()
    b = Mux(ChunkStream(m1, 2, Cc, "cuda:1"), _bank(23), 5, sessions)
    b.cs.load_slots([1, 0], st)
    b.put(1, moved[0])
    b.put(0, moved[1])
    b.finish()
    b.cs.close()
    _check_alone(m0, Cc, sessions, "cuda:0 -> cuda:1")


def _stitch_by_model(s, Cc, owners):
    """The fp64 stitch of session s with chunk k enhanced by enhance_audio of owners[k]."""
    x = np.concatenate([c[2] for c in s["calls"]])
    rows = R.chunk_rows(x, Cc)
    assert len(owners) == len(rows)
    enh = np.zeros_like(rows)
    for m in {id(o): o for o in owners}.values():
        idx = [k for k, o in enumerate(owners) if o is m]
        with torch.no_grad():
            enh[idx] = m.enhance_audio(torch.from_numpy(np.ascontiguousarray(rows[idx])).to(DEV)).cpu().numpy()
    return R.stitch(enh, Cc, x.shape[0])


def test_hand_over_between_models(built_lib):
    """Two sessions move through four models at live hand-overs: small FullSubNet+ (TSSE) -> the same configuration with other weights
    -> FullSubNet+ with the sub-band TCN -> fullsubnet.Model with offline_laplace_norm.  Each session equals the fp64 stitch of each
    model's enhance_audio rows for the chunks it enhanced, and what it emitted before a hand-over is what the old model alone gives."""
    from fsnplus_b200.streaming import ChunkStream
    Cc, H = 512, 256
    models = [_cached("plus", 3), _cached("plus", 8), _cached("tcn", 3), _cached("fsn", 3)]
    bank = _bank(24)
    sessions = []
    owners = {}                                            # per session: the model of each chunk enhanced so far
    st = moved = None
    for j, m in enumerate(models):
        mx = Mux(ChunkStream(m, 2, Cc, DEV), bank, 10 + j, sessions)
        if st is None:
            mx.start(0, 14 * H + 77, 211)
            mx.start(1, 12 * H + 5, 3)
        else:
            mx.cs.load_slots([1, 0], st)
            mx.put(1, moved[0])
            mx.put(0, moved[1])
        for _ in range(3):
            mx.auto(force={0: 250, 1: 267})
        if j + 1 < len(models):
            assert all(x is not None for x in mx.slot)
            moved = list(mx.slot)
            st = mx.cs.save_slots([0, 1])
            for i, x in enumerate(moved):
                o = owners.setdefault(id(x), [])
                o.extend([m] * (st.meta[i].chunks - len(o)))
                if j == 0:                                 # emitted before the first hand-over: model 0's own output
                    emitted = _y(x)
                    assert emitted.shape[0] == st.meta[i].chunks * H
                    assert np.array_equal(emitted, _alone(m, Cc, x)[:emitted.shape[0]])
        else:
            mx.finish()
            for x in sessions:
                o = owners[id(x)]
                o.extend([m] * (-(-x["n"] // H) - len(o)))
        mx.cs.close()
    worst = 0.0
    for s in sessions:
        assert s["done"]
        y, want = _y(s), _stitch_by_model(s, Cc, owners[id(s)])
        assert [len([o for o in owners[id(s)] if o is m]) > 0 for m in models] == [True] * 4
        e = O.rel_l2(y, want)
        worst = max(worst, e)
        assert e <= STITCH_TOL, e
    print(f"\n[hand-over] {len(sessions)} sessions over 4 models, worst rel-L2 vs the fp64 stitch {worst:.2e}")


def _nan_padding(state, Cc):
    """A copy of the state's payload with every padding byte (between the ring and the tail, after the tail) set to NaN."""
    from fsnplus_b200 import _lib
    ring = (Cc + P) * 4
    toff = (ring + 15) // 16 * 16
    tend = toff + Cc // 2 * 4
    stride, _ = _lib.chunk_state_layout(Cc)
    assert state.payload.shape[1] == stride
    p = state.payload.clone()
    nan = torch.full((1,), float("nan"), dtype=torch.float32).view(torch.uint8)
    for lo, hi in ((ring, toff), (tend, stride)):
        if hi > lo:
            p[:, lo:hi] = nan.repeat((hi - lo + 3) // 4)[:hi - lo].to(p.device)
    from fsnplus_b200.streaming import SessionState
    return SessionState(p, state.meta), toff - ring, stride - tend


def test_idle_slots_neighbours_and_padding(built_lib):
    """C = 514 (8 bytes between ring and tail).  An idle slot saves as samples = -1 and loads as no session (a STEP is refused, a START
    works).  A session loaded into slot 2 with NaN in every padding byte continues bit-identically to its lone run, and slots 0, 1, 3
    are bit-identical to a twin handle that saw no load."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import ChunkStream
    m = _cached()
    Cc, H = 514, 257
    bank = _bank(25)
    src = Mux(ChunkStream(m, 2, Cc, DEV), bank, 30)
    src.start(0, 9 * H + 100, 280)
    for _ in range(3):
        src.auto()
    idle = src.cs.save_slots([1])
    assert (idle.meta[0].samples, idle.meta[0].chunks) == (-1, 0)
    parked, gap, after = _nan_padding(src.cs.save_slots([0]), Cc)
    assert gap == 8 and after > 0
    s = src.slot[0]
    src.cs.close()

    cs, twin = ChunkStream(m, 4, Cc, DEV), ChunkStream(m, 4, Cc, DEV)
    mx, tw = Mux(cs, bank, 31), Mux(twin, bank, 31)
    for x in (mx, tw):
        x.start(0, 10 * H, 120)
        x.start(1, 9 * H + 7, 300)
        x.start(3, 8 * H + 2, 17)
        x.auto()
    cs.load_slots([2], parked)
    mx.put(2, s)
    for _ in range(6):
        mx.auto()
        tw.auto()
        for b in (0, 1, 3):
            assert (mx.slot[b] is None) == (tw.slot[b] is None)
    mx.finish()
    tw.finish()
    assert len(mx.sessions) == len(tw.sessions) + 1 and mx.sessions[-1] is s
    for a, b in zip(mx.sessions, tw.sessions):
        assert np.array_equal(_y(a), _y(b))
    assert np.array_equal(_y(s), _alone(m, Cc, s))
    cs.load_slots([1], idle)                               # an idle meta ends nothing but leaves the slot without a session
    with pytest.raises(_lib.FsnError, match="slot 1: STEP on a slot without a session"):
        cs.step(torch.zeros((4, 8), device=DEV), [0, 1, 0, 0], [SLOT_HOLD, SLOT_STEP, SLOT_HOLD, SLOT_HOLD])
    mx.start(1, 3 * H, 100)
    mx.start(0, 4 * H, 100)
    st = cs.save_slots([0])
    cs.load_slots([0], cs.save_slots([2]))                 # an idle slot over a live session: slot 0 has none afterwards
    with pytest.raises(_lib.FsnError, match="slot 0: STEP on a slot without a session"):
        cs.step(torch.zeros((4, 8), device=DEV), [1, 0, 0, 0], [SLOT_STEP, SLOT_HOLD, SLOT_HOLD, SLOT_HOLD])
    cs.load_slots([0], st)
    mx.finish()
    for x in mx.sessions[-2:]:
        assert np.array_equal(_y(x), _alone(m, Cc, x))
    cs.close()
    twin.close()


def test_errors_change_nothing(built_lib):
    """Every refusal of save and load names its index or field, and the next step equals a twin handle's that never saw it."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import ChunkStream, SessionState
    lib = _lib.load_library()
    m = _cached()
    Cc, H, B = 512, 256, 3
    bank = _bank(26)
    cs, twin = ChunkStream(m, B, Cc, DEV), ChunkStream(m, B, Cc, DEV)
    mx, tw = Mux(cs, bank, 40), Mux(twin, bank, 40)
    for x in (mx, tw):
        x.start(0, 40 * H, 300)
        x.start(1, 40 * H, 77)
        x.auto()
    good = cs.save_slots([0, 1])
    twin.save_slots([0, 1])
    other = ChunkStream(m, 1, 640, DEV)
    other.step(torch.zeros((1, 700), device=DEV), [700], [SLOT_START])
    wrong_c = other.save_slots([0])
    other.close()
    stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)

    def both():
        mx.auto()
        tw.auto()
        for a, b in zip(mx.sessions, tw.sessions):
            assert np.array_equal(_y(a), _y(b))

    def meta(**kv):
        q = (_lib.FsnChunkSlotMeta * 2)(*good.meta)
        for k, v in kv.items():
            setattr(q[1], k, v)
        return q

    def load(slots, meta_arr, payload=None):
        s = (C.c_int32 * len(slots))(*slots)
        p = good.payload if payload is None else payload
        ptr = p if isinstance(p, C.c_void_p) else C.c_void_p(p.data_ptr())
        return lib.fsn_chunk_stream_load_slots(cs._cs, len(slots), s if slots else None, ptr, meta_arr, stream)

    gp = good.payload
    unaligned = torch.empty(gp.numel() + 256, dtype=torch.uint8, device=DEV)[16:16 + gp.numel()]
    host = torch.empty_like(gp, device="cpu")
    cases = [
        (lambda: load([2, 1], meta(magic=0x534E5346)), "h_meta[1]: bad magic 0x534e5346"),
        (lambda: load([2, 1], meta(version=2)), "h_meta[1]: version 2"),
        (lambda: load([2, 1], meta(chunk_samples=640)), "h_meta[1]: chunk_samples 640"),
        (lambda: load([2, 1], meta(pre_context=128)), "h_meta[1]: pre_context 128"),
        (lambda: load([2, 1], meta(payload_bytes=good.payload.shape[1] + 256)), "h_meta[1]: payload_bytes"),
        (lambda: load([2, 1], meta(samples=-2, chunks=0)), "h_meta[1]: samples -2"),
        (lambda: load([2, 1], meta(chunks=good.meta[1].chunks + 1)), "h_meta[1]: chunks"),
        (lambda: load([2, 1], meta(samples=-1, chunks=1)), "h_meta[1]: chunks 1"),
        (lambda: load([2, 1], meta(samples=3, chunks=1)), "h_meta[1]: chunks 1"),
        (lambda: load([2, 2], meta()), "h_slots[1] = 2: slot 2 is loaded twice"),
        (lambda: load([2, 3], meta()), "h_slots[1] = 3 is out of range"),
        (lambda: load([-1, 2], meta()), "h_slots[0] = -1 is out of range"),
        (lambda: lib.fsn_chunk_stream_load_slots(cs._cs, 0, (C.c_int32 * 1)(2), C.c_void_p(gp.data_ptr()), meta(), stream), "n = 0"),
        (lambda: lib.fsn_chunk_stream_load_slots(cs._cs, 2, None, C.c_void_p(gp.data_ptr()), meta(), stream), "h_slots is null"),
        (lambda: lib.fsn_chunk_stream_load_slots(cs._cs, 2, (C.c_int32 * 2)(2, 1), C.c_void_p(gp.data_ptr()), None, stream),
         "h_meta is null"),
        (lambda: load([2, 1], meta(), C.c_void_p(None)), "d_state is null"),
        (lambda: load([2, 1], meta(), unaligned), "d_state is not 256-byte aligned"),
        (lambda: load([2, 1], meta(), host), "d_state is not device memory"),
        (lambda: lib.fsn_chunk_stream_load_slots(cs._cs, 1, (C.c_int32 * 1)(2), C.c_void_p(wrong_c.payload.data_ptr()), wrong_c.meta,
                                                 stream), "h_meta[0]: chunk_samples 640, this handle's chunks are 512"),
        (lambda: lib.fsn_chunk_stream_save_slots(cs._cs, 0, (C.c_int32 * 1)(0), C.c_void_p(gp.data_ptr()), meta(), stream), "n = 0"),
        (lambda: lib.fsn_chunk_stream_save_slots(cs._cs, 1, None, C.c_void_p(gp.data_ptr()), meta(), stream), "h_slots is null"),
        (lambda: lib.fsn_chunk_stream_save_slots(cs._cs, 1, (C.c_int32 * 1)(3), C.c_void_p(gp.data_ptr()), meta(), stream),
         "h_slots[0] = 3 is out of range"),
        (lambda: lib.fsn_chunk_stream_save_slots(cs._cs, 1, (C.c_int32 * 1)(0), C.c_void_p(gp.data_ptr()), None, stream), "h_meta is null"),
        (lambda: lib.fsn_chunk_stream_save_slots(cs._cs, 1, (C.c_int32 * 1)(0), C.c_void_p(unaligned.data_ptr()), meta(), stream),
         "d_state is not 256-byte aligned"),
        (lambda: lib.fsn_chunk_stream_save_slots(cs._cs, 1, (C.c_int32 * 1)(0), C.c_void_p(host.data_ptr()), meta(), stream),
         "d_state is not device memory"),
        (lambda: lib.fsn_chunk_stream_save_slots(None, 1, (C.c_int32 * 1)(0), C.c_void_p(gp.data_ptr()), meta(), stream), "cs is null"),
    ]
    if torch.cuda.device_count() > 1:
        far = torch.empty_like(gp, device="cuda:1")
        cases.append((lambda: load([2, 1], meta(), far), "d_state is memory of device 1"))
    before = bytes(good.payload.cpu().numpy())
    for fn, msg in cases:
        assert fn() == -1, msg
        err = lib.fsn_last_error().decode()
        assert msg in err, (msg, err)
        both()
    assert bytes(good.payload.cpu().numpy()) == before      # the refused saves wrote nothing
    with pytest.raises(TypeError):
        cs.load_slots([2], SessionState(good.payload[:1], (_lib.FsnSlotMeta * 1)()))
    both()
    mx.finish()
    tw.finish()
    for a, b in zip(mx.sessions, tw.sessions):
        assert np.array_equal(_y(a), _y(b))
    cs.close()
    twin.close()
