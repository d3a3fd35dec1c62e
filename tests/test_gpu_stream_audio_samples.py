"""Sample-granular audio sessions (fsn_stream_step_audio_samples, DESIGN.md §3.19): any number of samples per slot and call, and
sessions of any length.

  * parity: every session's concatenated output against the offline audio call (fsn_model_enhance_audio) of its input, for lengths
    hop + 1 .. 5 hop + 37 and packets of 1 .. 1000 samples, at small geometries (mma / auto, LSTM / GRU, num_freqs 33..513) and at the
    config #4 geometry with 3 slots (weight-stationary full band) and 80 slots; and against the fp64 pipeline fed with the oracle's
    masks;
  * bit identity: fed whole hops, every call's rows and counts are those of the per-hop / K-hop call it stands for, on a mirror handle;
  * many slots: random counts, HOLDs, staggered STARTs, a START of less than a hop, a START over a live partial hop, NaN in every
    unread sample, zero rows past nout, nout summing to L;
  * parking mid-hop, attenuation limits, the mixing rules, every refusal with no state change, and launch counts."""
import numpy as np
import pytest
import torch

from oracle import fsn_oracle as O
from test_gpu_stream_audio_chunks import WAVE_TOL, _meta, _segment
from test_gpu_stream_chunks import _fsn
from test_gpu_stream_sessions import DEV, _small_cfg, _t

pytestmark = pytest.mark.gpu
HOLD, STEP, START, FLUSH = 0, 1, 2, 3


def _model(kind, lstm_impl="mma", F=65):
    if kind == "default":                                   # BASELINE config #4
        cfg = O.default_fsn_config()
        cfg["norm_type"] = "cumulative_laplace_norm"
        params = O.make_params_fsn(cfg, seed=33)
        return cfg, params, _fsn(cfg, params)
    cfg = _small_cfg("cumulative_laplace_norm", kind)
    if F != 65:
        cfg.update(num_freqs=F, look_ahead=1 if F < 65 else 2)
    params = O.make_params_fsn(cfg, seed=13)
    return cfg, params, _fsn(cfg, params, lstm_impl=lstm_impl)


def _clip(L, seed, gain=1.0):
    return (O.synth_clips(1, num_samples=max(L, 16000), seed0=seed)[0, :L] * gain).astype(np.float32)


class Sess:
    def __init__(self, slot, x, start=0, sizes=None, hold=0.0, seed=0):
        self.slot, self.x, self.start, self.hold = slot, np.asarray(x, np.float32), start, hold
        self.sizes, self.rng = sizes, np.random.default_rng(seed)
        self.pos, self.out, self.done, self.flushed = 0, [], False, False

    def packet(self, S):
        if self.sizes is None:
            return int(self.rng.integers(0, S + 1))
        return self.sizes if isinstance(self.sizes, int) else int(self.rng.choice(self.sizes))


def drive(st, sessions, S, check_rows=True, mirror=None, max_calls=100000):
    """Run the sessions (each on its slot, one after another per slot) through sample calls of rows of S samples, NaN wherever the
    call must not read.  Returns each session's output; checks zero rows past nout and, with a mirror handle, the hop calls' bits."""
    B, hop, la = st.B, st.hop, st.look_ahead
    queue = {b: [s for s in sessions if s.slot == b] for b in range(B)}
    c = 0
    while any(queue.values()):
        assert c < max_calls
        flags, counts = np.zeros(B, np.int32), np.zeros(B, np.int32)
        x = np.full((B, S), np.nan, np.float32)
        cur = {}
        for b, q in queue.items():
            if not q or c < q[0].start:
                continue
            s = q[0]
            if s.pos and s.hold and s.rng.random() < s.hold:
                continue
            n = min(s.packet(S), len(s.x) - s.pos)
            last = s.pos + n == len(s.x) and (s.pos + n) > hop
            flags[b] = START if s.pos == 0 and not s.out else FLUSH if last else STEP
            if flags[b] == START and last:
                n = len(s.x) - hop                        # START and FLUSH are two calls
            counts[b] = n
            x[b, :n] = s.x[s.pos:s.pos + n]
            cur[b] = s
        want = _mirror_call(mirror, flags, counts, x, cur) if mirror is not None else None
        out, nout = st.step_audio_samples(_t(x), torch.from_numpy(counts), torch.from_numpy(flags))
        out = out.cpu()
        for b in range(B):
            k = int(nout[b])
            if check_rows:
                assert torch.count_nonzero(out[b, k:]) == 0, f"call {c} slot {b}: output past nout is not zero"
            if want is not None:
                assert k == want[1][b] and torch.equal(out[b, :k], want[0][b][:k]), f"call {c} slot {b}: differs from the hop call"
            if b not in cur:
                assert k == 0
                continue
            s = cur[b]
            s.out.append(out[b, :k].numpy())
            s.pos += int(counts[b])
            s.out.append(np.zeros(0, np.float32))
            if flags[b] == FLUSH:
                queue[b].pop(0)
                s.done = True
                for nxt in queue[b]:
                    nxt.start = max(nxt.start, c + 1)
        c += 1
    res = []
    for s in sessions:
        w = np.concatenate(s.out)
        assert w.size == len(s.x), f"slot {s.slot}: {w.size} output samples for {len(s.x)} input"
        res.append(w)
    return res


def _mirror_call(ref, flags, counts, x, cur):
    """The hop call a sample call of whole hops stands for, run on the mirror handle: (rows, nout in samples)."""
    B, hop, la = ref.B, ref.hop, ref.look_ahead
    n = counts // hop
    assert np.all(counts % hop == 0)
    need = np.where(flags == FLUSH, n + la + 2, np.where(flags == HOLD, 0, n))
    K = int(need.max())
    hf = np.where((flags != FLUSH) & (n == 0), HOLD, flags).astype(np.int32)
    if K <= 1 and not np.any(flags == FLUSH):
        xs = x[:, :hop].copy()
        o, v = ref.step_audio(_t(xs), torch.from_numpy(hf))
        return [r for r in o.cpu()], [hop * int(a) for a in v]
    xs = np.full((B, K * hop), np.nan, np.float32)
    w = min(x.shape[1], K * hop)
    xs[:, :w] = x[:, :w]
    o, nout = ref.step_audio_chunk(_t(xs), torch.from_numpy(hf), torch.from_numpy(n.astype(np.int32)))
    return [r for r in o.cpu()], [hop * int(a) for a in nout]


def _offline(m, x, lim=None):
    with torch.no_grad():
        return m.enhance_audio(_t(x[None]), atten_lim_db=lim)[0].cpu().numpy()


def _check_offline(m, sessions, got, tol=WAVE_TOL, lim=None):
    for s, w in zip(sessions, got):
        e = O.rel_l2(w, _offline(m, s.x, lim))
        assert e < tol, f"slot {s.slot} L={len(s.x)}: {e:.2e} from the offline audio call"


def _lengths(hop, rng):
    return [hop + 1, 2 * hop - 1, 2 * hop, 2 * hop + 1, 5 * hop + 37, int(rng.integers(hop + 1, 9 * hop))]


@pytest.mark.parametrize("kind,impl,F", [("LSTM", "mma", 65), ("LSTM", "auto", 65), ("GRU", "mma", 65), ("LSTM", "mma", 33),
                                         ("LSTM", "auto", 513)])
def test_parity_lengths_and_packets(built_lib, kind, impl, F):
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model(kind, impl, F)
    hop = F - 1
    rng = np.random.default_rng(F)
    Ls = _lengths(hop, rng)
    sizes = [1, 7, 160, 256, 320, 1000, None]
    sessions = []
    for i, size in enumerate(sizes):
        for j, L in enumerate(Ls):
            if size == 1 and L > 3 * hop:
                continue
            sessions.append(Sess(i, _clip(L, 100 * i + j), sizes=size if size else 10 ** 6))
    st = StreamingFullSubNet(m, batch_size=len(sizes), device=DEV)
    got = drive(st, sessions, S=max(1000, max(Ls)))
    st.close()
    _check_offline(m, sessions, got)
    for s, w in list(zip(sessions, got))[:: max(1, len(sessions) // 4)]:   # end to end against the fp64 oracle
        X = O.stft(s.x[None].astype(np.float64), 2 * hop, hop, 2 * hop)
        crm = O.fullsubnet_forward(params, cfg, np.abs(X)[:, None])
        ref = O.istft(O.enhance(X, crm), 2 * hop, hop, 2 * hop, length=len(s.x))[0]
        assert O.rel_l2(w, ref) < WAVE_TOL


@pytest.mark.parametrize("B", [3, 80])
def test_parity_config4(built_lib, B):
    """Config #4 geometry: 3 slots run the weight-stationary full band, 80 the generic one; 10 / 20 ms packets, staggered starts."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("default")
    hop = 256
    rng = np.random.default_rng(B)
    sessions = [Sess(b, _clip(int(rng.integers(hop + 1, 40 * hop)), 500 + b), start=int(rng.integers(0, 6)),
                     sizes=[160, 320][b % 2], hold=0.1, seed=b) for b in range(B)]
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    got = drive(st, sessions, S=320)
    assert st.lib.fsn_stream_fb_ws(st._st) == (1 if B <= 64 else 0)
    st.close()
    _check_offline(m, sessions, got)


@pytest.mark.parametrize("kind", ["LSTM", "GRU"])
def test_whole_hops_match_hop_calls(built_lib, kind):
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model(kind)
    hop = 64
    rng = np.random.default_rng(5)
    sessions = [Sess(b, _clip(hop * int(rng.integers(2, 30)), 40 + b), start=b, sizes=[hop, hop, 2 * hop, 5 * hop], hold=0.2,
                     seed=b) for b in range(4)]
    sessions += [Sess(b, _clip(hop * int(rng.integers(2, 12)), 60 + b), sizes=[hop, 3 * hop], seed=10 + b) for b in range(4)]
    st, ref = StreamingFullSubNet(m, batch_size=4, device=DEV), StreamingFullSubNet(m, batch_size=4, device=DEV)
    drive(st, sessions, S=5 * hop, mirror=ref)
    st.close(); ref.close()


def test_many_slots_random(built_lib):
    """Random counts and HOLDs on 16 slots, sessions reusing slots, a START of less than a hop, a START over a live partial hop."""
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("LSTM")
    hop, B, S = 64, 16, 300
    rng = np.random.default_rng(9)
    sessions = []
    for b in range(B):
        for k in range(2):
            sessions.append(Sess(b, _clip(int(rng.integers(hop + 1, 20 * hop)), 1000 + 2 * b + k), start=int(rng.integers(0, 8)),
                                 sizes=None, hold=0.25, seed=b * 3 + k))
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    # a START of less than a hop, then a START over that live partial hop: the second session is the one that counts
    x0 = _clip(5 * hop + 3, 77)
    flags, counts = np.zeros(B, np.int32), np.zeros(B, np.int32)
    flags[0], counts[0] = START, hop // 2
    xs = np.full((B, S), np.nan, np.float32)
    xs[0, :hop // 2] = 1.0
    out, nout = st.step_audio_samples(_t(xs), torch.from_numpy(counts), torch.from_numpy(flags))
    assert int(nout.sum()) == 0 and torch.count_nonzero(out) == 0
    sessions.insert(0, Sess(0, x0, sizes=[hop // 3], seed=1))
    got = drive(st, sessions, S=S)
    st.close()
    _check_offline(m, sessions, got)


def test_park_mid_hop(built_lib):
    """Park a session with a partial hop (meta.frames = r), resume it in another slot, on a handle of another B and on one with the
    other full-band kernel: the continuation equals the unparked run.  Bad frames values are refused."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("default")
    hop = 256
    x = _clip(30 * hop + 77, 4242)
    cut = 11 * hop + 123

    def feed(st, slot, a, b, first, flush, size=160):
        outs, pos = [], a
        while pos < b:
            n = min(size, b - pos)
            flags, counts = np.zeros(st.B, np.int32), np.zeros(st.B, np.int32)
            flags[slot] = START if first and pos == a else FLUSH if flush and pos + n == b else STEP
            counts[slot] = n
            xs = np.full((st.B, size), np.nan, np.float32)
            xs[slot, :n] = x[pos:pos + n]
            o, k = st.step_audio_samples(_t(xs), torch.from_numpy(counts), torch.from_numpy(flags))
            outs.append(o[slot, :int(k[slot])].cpu().numpy())
            pos += n
        return np.concatenate(outs)

    lone = StreamingFullSubNet(m, batch_size=3, device=DEV)
    whole = feed(lone, 1, 0, len(x), True, True)
    a = StreamingFullSubNet(m, batch_size=3, device=DEV)
    head = feed(a, 1, 0, cut, True, False)
    state = a.save_slots([1])
    assert state.meta[0].frames == cut % hop and state.meta[0].tick == cut // hop
    for B, slot in [(3, 2), (5, 4), (80, 33)]:
        h = a if B == 3 else StreamingFullSubNet(m, batch_size=B, device=DEV)
        h.load_slots([slot], state)
        tail = feed(h, slot, cut, len(x), False, True)
        got = np.concatenate([head, tail])
        if B <= 64:
            assert np.array_equal(got, whole), f"B={B}: the resumed session differs from the unparked run"
        else:
            assert O.rel_l2(got, whole) < 1e-5, f"B={B}: {O.rel_l2(got, whole):.2e}"
    for frames, tick, hops in [(hop, 3, 0), (-1, 3, 0), (5, -1, 0), (5, 40, 30)]:
        bad = state[0]
        bad.meta[0].frames, bad.meta[0].tick, bad.meta[0].hops = frames, tick, hops
        with pytest.raises(_lib.FsnError, match="frames"):
            lone.load_slots([0], bad)


def test_atten_lim(built_lib):
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("LSTM")
    hop = 64
    lims = [6.0, float("inf"), 12.0]
    sessions = [Sess(b, _clip(7 * hop + 13 * (b + 1), 300 + b), sizes=[37, 100], seed=b) for b in range(3)]
    st = StreamingFullSubNet(m, batch_size=3, device=DEV)
    st.set_atten_lim([0, 1, 2], lims)
    got = drive(st, sessions, S=100)
    st.close()
    for s, w, lim in zip(sessions, got, lims):
        e = O.rel_l2(w, _offline(m, s.x, [lim]))
        assert e < WAVE_TOL, f"slot {s.slot}: {e:.2e}"


def _state(st, slots):
    p = st.save_slots(slots)
    torch.cuda.synchronize()
    return _meta(p), [p.payload[:, slice(*_segment(st.model._cfg, i))].cpu().clone() for i in range(9)]


def test_refusals_and_mixing(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("LSTM")
    hop, la, B, S = 64, cfg["look_ahead"], 4, 200
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    x = np.random.default_rng(1).standard_normal((B, S)).astype(np.float32) * 0.1

    def call(flags, counts, S_=S):
        return st.step_audio_samples(_t(x[:, :S_]), torch.tensor(counts, dtype=torch.int32), torch.tensor(flags, dtype=torch.int32))

    call([START, START, START, HOLD], [150, 64, 10, 0])        # slot 0: 2 hops + 22; slot 1: 1 hop; slot 2: 10 pending
    before = _state(st, [0, 1, 2, 3])
    cases = [([5, 0, 0, 0], [0, 0, 0, 0], "flag"), ([STEP, 0, 0, 0], [S + 1, 0, 0, 0], "h_counts"),
             ([STEP, 0, 0, 0], [-1, 0, 0, 0], "h_counts"), ([0, 0, 0, STEP], [0, 0, 0, 5], "without a session"),
             ([0, 0, 0, FLUSH], [0, 0, 0, 0], "without a session"), ([0, 0, FLUSH, 0], [0, 0, 50, 0], "n_fft / 2"),
             ([0, FLUSH, 0, 0], [0, 0, 0, 0], "n_fft / 2")]
    for flags, counts, msg in cases:
        with pytest.raises(_lib.FsnError, match=msg):
            call(flags, counts)
    with pytest.raises(_lib.FsnError, match="S = 0"):
        _lib.check(st.lib.fsn_stream_step_audio_samples(st._st, _t(x).data_ptr(), 0, torch.zeros(B, dtype=torch.int32).data_ptr(),
                                                        torch.zeros(B, dtype=torch.int32).data_ptr(), _t(x).data_ptr(),
                                                        torch.zeros(B, dtype=torch.int32).data_ptr(), None))
    with pytest.raises(_lib.FsnError, match="h_counts is null"):
        _lib.check(st.lib.fsn_stream_step_audio_samples(st._st, _t(x).data_ptr(), S, torch.zeros(B, dtype=torch.int32).data_ptr(),
                                                        None, _t(x).data_ptr(), torch.zeros(B, dtype=torch.int32).data_ptr(), None))
    # a hop call's STEP or FLUSH on a slot holding a partial hop names the slot
    with pytest.raises(_lib.FsnError, match="slot 0: STEP on a session holding a partial hop"):
        st.step_audio(_t(x[:, :hop]), torch.tensor([STEP, HOLD, HOLD, HOLD], dtype=torch.int32))
    with pytest.raises(_lib.FsnError, match="slot 2: FLUSH"):
        st.step_audio_chunk(_t(np.zeros((B, 4 * hop), np.float32)), torch.tensor([HOLD, HOLD, FLUSH, HOLD], dtype=torch.int32),
                            torch.zeros(B, dtype=torch.int32))
    after = _state(st, [0, 1, 2, 3])
    assert before[0] == after[0] and all(torch.equal(p, q) for p, q in zip(before[1], after[1])), "a failed call changed state"
    # slot 1 is hop-aligned: the hop calls continue it and a sample FLUSH of 0 completes what a hop call left mid-flush
    o, v = st.step_audio(_t(x[:, :hop]), torch.tensor([HOLD, STEP, HOLD, HOLD], dtype=torch.int32))
    o, n = st.step_audio_chunk(_t(np.zeros((B, 2 * hop), np.float32)), torch.tensor([HOLD, FLUSH, HOLD, HOLD], dtype=torch.int32),
                               torch.zeros(B, dtype=torch.int32))
    o, n = call([HOLD, FLUSH, HOLD, HOLD], [0, 0, 0, 0])
    assert int(n[1]) > 0
    with pytest.raises(_lib.FsnError, match="STEP after the session's FLUSH"):
        call([HOLD, STEP, HOLD, HOLD], [0, 3, 0, 0])
    with pytest.raises(_lib.FsnError, match="after the session's FLUSH"):
        call([HOLD, FLUSH, HOLD, HOLD], [0, 3, 0, 0])
    o, n = call([HOLD, FLUSH, HOLD, HOLD], [0, 0, 0, 0])     # after the end: a HOLD
    assert int(n[1]) == 0
    # a hop START discards slot 2's partial hop; a mask call is FSN_ESTATE
    st.step_audio(_t(x[:, :hop]), torch.tensor([HOLD, HOLD, START, HOLD], dtype=torch.int32))
    assert st.save_slots([2]).meta[0].frames == 0
    with pytest.raises(_lib.FsnError):
        st.step_slots(_t(np.zeros((B, cfg["num_freqs"]), np.float32)), [HOLD] * B)
    st.close()
    mk = StreamingFullSubNet(m, batch_size=B, device=DEV)
    mk.step_slots(_t(np.zeros((B, cfg["num_freqs"]), np.float32)), [START] + [HOLD] * (B - 1))
    with pytest.raises(_lib.FsnError, match="mask calls"):
        mk.step_audio_samples(_t(x), torch.zeros(B, dtype=torch.int32), torch.zeros(B, dtype=torch.int32))
    mk.close()


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type.name == "CUDA" and "Memcpy" not in e.key and "Memset" not in e.key
               and "memcpy" not in e.key.lower() and "memset" not in e.key.lower())


def test_launch_counts(built_lib):
    from fsnplus_b200.streaming import StreamingFullSubNet
    cfg, params, m = _model("LSTM")
    hop, B, S = 64, 4, 100
    st = StreamingFullSubNet(m, batch_size=B, device=DEV)
    x = _t(np.random.default_rng(0).standard_normal((B, S)).astype(np.float32))
    st.step_audio_samples(x, torch.zeros(B, dtype=torch.int32), torch.tensor([START, START, HOLD, HOLD], dtype=torch.int32))
    res = {}

    def run(counts, flags):
        res["o"] = st.step_audio_samples(x, torch.tensor(counts, dtype=torch.int32), torch.tensor(flags, dtype=torch.int32))
    assert _kernels(lambda: run([10, 20, 0, 0], [STEP, STEP, HOLD, HOLD])) == 1      # no hop completes: the store alone
    assert int(res["o"][1].sum()) == 0 and torch.count_nonzero(res["o"][0]) == 0
    assert _kernels(lambda: run([0, 0, 0, 0], [STEP, HOLD, HOLD, HOLD])) == 0        # nothing consumed
    assert torch.count_nonzero(res["o"][0]) == 0
    assert _kernels(lambda: run([60, 0, 0, 0], [STEP, HOLD, HOLD, HOLD])) == 2       # slot 0's first hop: the START tick, no frame
    assert _kernels(lambda: run([64, 0, 0, 0], [STEP, HOLD, HOLD, HOLD])) > 2        # its second hop: a model step
    st.close()
