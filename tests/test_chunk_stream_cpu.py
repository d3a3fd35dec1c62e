"""Overlapped-chunk sessions on the host (DESIGN.md §3.16): the numpy restatement against the reference's loop
(inferencer.py:191-250), the Hann COLA identity, planted faults, the per-slot schedule, and an fp64 restatement of the two kernels'
indexing (sample ring, pre-context, zero tail, cross-fade across calls) driven by that schedule."""
import numpy as np
import pytest

import chunk_stream_ref as R
from chunk_stream_ref import P, SLOT_FLUSH, SLOT_HOLD, SLOT_START, SLOT_STEP


def _enhancers(seed=0):
    rng = np.random.default_rng(seed)
    h = rng.standard_normal(31) / 4

    def filt(rows):                                        # a random causal FIR filter along each row: it sees the pre-context
        rows = np.atleast_2d(rows)
        return np.stack([np.convolve(r, h)[:r.shape[0]] for r in rows])
    return {"identity": lambda r: np.array(r, np.float64), "gain": lambda r: 0.37 * np.asarray(r, np.float64), "filter": filt}


@pytest.mark.parametrize("C", [512, 600, 1024])
@pytest.mark.parametrize("name", ["identity", "gain", "filter"])
def test_restatement_matches_reference_loop(C, name):
    enh = _enhancers()[name]
    H = C // 2
    rng = np.random.default_rng(C)
    for L in [1, P, H - 1, H, H + 1, 2 * H, 5 * H + 7, 7 * H + 311]:
        x = rng.standard_normal(L)
        got = R.chunk_stream_ref(x, C, enh)
        want = R.reference_loop(x, C, lambda row: enh(row[None])[0])
        assert got.shape == (L,)
        assert np.abs(got - want).max() <= 1e-12, (C, name, L)


@pytest.mark.parametrize("C", [512, 514, 2048])
def test_identity_is_exact(C):
    """The periodic Hann window sums to one across the overlap, and region 0 is unwindowed: y == x."""
    H = C // 2
    rng = np.random.default_rng(1)
    for L in [1, P, H - 1, H, H + 1, 2 * H, 5 * H + 7]:
        x = rng.standard_normal(L)
        y = R.chunk_stream_ref(x, C, _enhancers()["identity"])
        assert y.shape == (L,) and np.abs(y - x).max() <= 1e-12, (C, L)


@pytest.mark.parametrize("fault", ["window_first", "pre_offset", "tail_twice", "drop_last"])
def test_planted_faults_are_caught(fault):
    """Each fault breaks the identity (y == x) or, for the pre-context the identity drops, the agreement with the reference loop under
    the random filter."""
    C, H = 600, 300
    rng = np.random.default_rng(2)
    ident_fails, ref_fails = [], []
    for L in [1, H + 1, 5 * H + 7]:
        x = rng.standard_normal(L)
        y = R.chunk_stream_ref(x, C, _enhancers()["identity"], fault=fault)
        ident_fails.append(not (y.shape == x.shape and np.abs(y - x).max() <= 1e-12))
        f = _enhancers()["filter"]
        y = R.chunk_stream_ref(x, C, f, fault=fault)
        ref = R.reference_loop(x, C, lambda row: f(row[None])[0])
        ref_fails.append(not (y.shape == ref.shape and np.abs(y - ref).max() <= 1e-12))
    assert any(ref_fails if fault == "pre_offset" else ident_fails), fault
    assert ident_fails[-1] or ref_fails[-1], fault                  # the longest session shows every fault


def _random_schedule(rng, B, calls, S, C, p_start=0.15, p_flush=0.1, p_hold=0.2):
    """Per call: (flags [B], counts [B]) with staggered STARTs, HOLDs, counts of 0 / 1 / S / random, and FLUSHes."""
    live = [False] * B
    sched = []
    for _ in range(calls):
        fl, ct = [], []
        for b in range(B):
            u = rng.random()
            c = int(rng.choice([0, 1, S, int(rng.integers(0, S + 1))]))
            if not live[b]:
                f = SLOT_START if u < p_start else SLOT_HOLD
            elif u < p_hold:
                f = SLOT_HOLD
            elif u < p_hold + p_flush:
                f = SLOT_FLUSH
            elif u < p_hold + p_flush + 0.03:
                f = SLOT_START                               # a slot reused mid-session
            else:
                f = SLOT_STEP
            live[b] = f != SLOT_FLUSH and (live[b] or f == SLOT_START)
            fl.append(f)
            ct.append(c)
        sched.append((fl, ct))
    return sched


@pytest.mark.parametrize("S,C", [(1, 512), (160, 512), (700, 512), (1500, 600), (320, 2048)])
def test_schedule_latency_and_flush(S, C):
    """Chunks complete in order, chunk k in the call where the input first reaches k H + C or at FLUSH; emitted = max(0, n / H - 1) H
    (lag min(n, H + n mod H): H to 2H once n >= H); after FLUSH everything through L has come out and the slot has no session."""
    H = C // 2
    rng = np.random.default_rng(S + C)
    B = 6
    slots = [R.ChunkSlotRef(C) for _ in range(B)]
    done, emitted, n = [0] * B, [0] * B, [0] * B
    for fl, ct in _random_schedule(rng, B, 400, S, C):
        for b in range(B):
            if fl[b] == SLOT_START:
                done[b] = emitted[b] = n[b] = 0
            chunks, nout = slots[b].call(fl[b], ct[b], S)
            if fl[b] == SLOT_HOLD:
                assert (chunks, nout) == ([], 0)
                continue
            n[b] += ct[b]
            assert chunks == list(range(done[b], done[b] + len(chunks)))
            done[b] += len(chunks)
            emitted[b] += nout
            assert 0 <= nout <= S + C
            if fl[b] == SLOT_FLUSH:
                assert done[b] == -(-n[b] // H) and emitted[b] == n[b] and slots[b].n is None
            else:
                assert all(k * H + C <= n[b] for k in chunks)
                assert done[b] * H + C > n[b]                # the next chunk is not complete yet
                assert emitted[b] == max(0, n[b] // H - 1) * H
                lag = n[b] - emitted[b]
                assert lag == min(n[b], H + n[b] % H) and lag < 2 * H
                assert lag >= H or n[b] < H


def test_flush_at_every_phase():
    """A session of L samples for every L mod H, flushed with 0, 1 or all of its last samples: ceil(L / H) chunks, L samples out."""
    C, H, S = 512, 256, 100
    for L in range(3 * H, 5 * H + 1):
        for tail in (0, 1, L % S or S):
            slot = R.ChunkSlotRef(C)
            pushed, out, chunks, first = 0, 0, 0, True
            while pushed < L - tail:
                c = min(S, L - tail - pushed)
                k, o = slot.call(SLOT_START if first else SLOT_STEP, c, S)
                first = False
                pushed += c
                out += o
                chunks += len(k)
            k, o = slot.call(SLOT_START if first else SLOT_FLUSH, tail, S)
            if first:                                       # the whole session in its FLUSH call
                k2, o2 = slot.call(SLOT_FLUSH, 0, S)
                k, o = k + k2, o + o2
            assert chunks + len(k) == -(-L // H) and out + o == L, (L, tail)


def test_schedule_errors_change_nothing():
    slot = R.ChunkSlotRef(512)
    for f, c in [(SLOT_STEP, 1), (SLOT_FLUSH, 0), (4, 0), (-1, 0)]:
        with pytest.raises(ValueError):
            slot.call(f, c, 10)
    slot.call(SLOT_START, 10, 10)
    for f, c in [(SLOT_STEP, 11), (SLOT_STEP, -1), (SLOT_FLUSH, 11)]:
        with pytest.raises(ValueError):
            slot.call(f, c, 10)
    assert (slot.n, slot.k) == (10, 0)


class _DeviceSim:
    """fp64 restatement of fsn_chunk_stream_step: chunk_slot_plan's fields, chunk_gather_kernel (ring of C + P samples at
    (phase + r) mod R) and chunk_crossfade_kernel (tail across chunks and calls), around an enhancer of the batch rows."""

    def __init__(self, B, C, enhance):
        self.B, self.C, self.H, self.R = B, C, C // 2, C + P
        self.ring = np.full((B, self.R), np.nan)
        self.tail = np.full((B, self.H), np.nan)
        self.slots = [R.ChunkSlotRef(C) for _ in range(B)]
        self.enhance = enhance
        self.w = R.hann(C)

    def step(self, x, counts, flags):
        B, C, H, Rr, S = self.B, self.C, self.H, self.R, x.shape[1]
        plans, rows = [], []
        for b in range(B):
            s = self.slots[b]
            k0, n0 = (s.k, s.n) if flags[b] in (SLOT_STEP, SLOT_FLUSH) else (0, 0)
            chunks, nout = s.call(flags[b], counts[b], S)
            if flags[b] == SLOT_HOLD:
                plans.append(None)
                continue
            a0 = k0 * H
            p = dict(nc=len(chunks), row0=len(rows), rel0=n0 - a0, rel1=n0 + counts[b] - a0, lo=-P if k0 else 0, ph=a0 % Rr, nout=nout)
            plans.append(p)
            for i in range(p["nc"]):                       # gather
                r = i * H - P + np.arange(P + C)
                v = np.zeros(P + C)
                ok = (r >= p["lo"]) & (r < p["rel1"])
                new = ok & (r >= p["rel0"])
                old = ok & (r < p["rel0"])
                v[new] = x[b, r[new] - p["rel0"]]
                v[old] = self.ring[b, (p["ph"] + r[old] + Rr) % Rr]
                assert not np.isnan(v).any()
                rows.append(v)
            r = np.arange(max(p["rel1"] - Rr, p["rel0"]), p["rel1"])   # append
            self.ring[b, (p["ph"] + r) % Rr] = x[b, r - p["rel0"]]
        enh = self.enhance(np.array(rows)) if rows else None
        out = np.zeros((B, S + C))
        nout = np.zeros(B, np.int64)
        for b, p in enumerate(plans):                      # cross-fade
            if p is None:
                continue
            for i in range(p["nc"]):
                e = enh[p["row0"] + i, P:]
                v = e[:H] if (p["lo"] == 0 and i == 0) else e[:H] * self.w[:H] + self.tail[b]
                o = i * H + np.arange(H)
                keep = o < p["nout"]
                out[b, o[keep]] = v[keep]
                self.tail[b] = e[H:] * self.w[H:]
            assert not np.isnan(out[b, :p["nout"]]).any()
            nout[b] = p["nout"]
        return out, nout


@pytest.mark.parametrize("S,C", [(7, 512), (160, 512), (333, 600), (1300, 512)])
def test_kernel_indexing_matches_restatement(S, C):
    """Staggered sessions through the schedule and the kernels' indexing, NaN in every unread sample: each session's concatenated
    output equals chunk_stream_ref of its input under the random filter."""
    f = _enhancers(3)["filter"]
    rng = np.random.default_rng(S * 7 + C)
    B = 5
    sim = _DeviceSim(B, C, f)
    ins, outs, finished = [None] * B, [None] * B, []
    for fl, ct in _random_schedule(rng, B, 300, S, C):
        x = np.full((B, S), np.nan)
        for b in range(B):
            if fl[b] != SLOT_HOLD:
                x[b, :ct[b]] = rng.standard_normal(ct[b])
        y, nout = sim.step(x, ct, fl)
        for b in range(B):
            if fl[b] == SLOT_HOLD:
                assert nout[b] == 0 and not y[b].any()
                continue
            if fl[b] == SLOT_START:
                ins[b], outs[b] = [], []
            ins[b].append(x[b, :ct[b]])
            outs[b].append(y[b, :nout[b]])
            assert not y[b, nout[b]:].any()
            if fl[b] == SLOT_FLUSH:
                finished.append((np.concatenate(ins[b]), np.concatenate(outs[b])))
    assert len(finished) >= 10
    for xin, yout in finished:
        want = R.chunk_stream_ref(xin, C, f)
        assert yout.shape == want.shape and np.allclose(yout, want, rtol=0, atol=1e-12)
