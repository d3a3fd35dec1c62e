"""fp64 emulation of one slot of the sample-granular audio call (fsn_stream_step_audio_samples, DESIGN.md §3.19), built on the
per-hop slot emulation ``stream_audio_ref.AudioSlotRef``.

Completed hops drive the hop ticks of AudioSlotRef; the r < hop samples of a partial hop wait in the history-ring slot the next hop
takes (t % 3).  A FLUSH that leaves r > 0 samples stores them there, analyses frame K from its r real samples reflected at L - 1
(L = K hop + r) and, after frame K is synthesised, emits its last r samples as tail * inv_last.  The tests show that a session's
concatenated outputs are the offline pipeline ``offline(x, crm)`` for every length and packet schedule, that whole hops give the
per-hop emulation's hops tick for tick, and that every sample becomes final when the latency rule says it does."""
import numpy as np
import pytest

from oracle import fsn_oracle as O
from stream_audio_ref import FLUSH, HOLD, START, STEP, AudioSlotRef, offline


class SampleSlotRef(AudioSlotRef):
    """One slot of the sample call: ``call(flag, samples, mask_of)`` returns the samples that became final, in order."""

    def __init__(self, n_fft, look_ahead):
        super().__init__(n_fft, look_ahead)
        self.pend = np.zeros(0)                       # r < hop samples of the partial hop; held in hist[t % 3] on the device
        self.r_end = 0                                # L - K hop of a session whose FLUSH has come
        self.inv_last = 1.0 / self.w[self.hop:] ** 2

    def _frame(self, j):
        p = np.abs(np.arange(self.hop * (j - 1), self.hop * (j + 1)))
        if self.K:
            L = self.K * self.hop + self.r_end
            p = np.where(p >= L, 2 * (L - 1) - p, p)
        return self.hist[(p // self.hop) % 3, p % self.hop]

    def plan_call(self, flag, count):
        """(hops completed, ticks run) of a call, without changing the state; ValueError for a call the API rejects."""
        if flag == HOLD:
            return 0, 0
        if flag == START:
            return count // self.hop, count // self.hop
        if self.t < 0:
            raise ValueError("no session on this slot")
        if self.K and (flag == STEP or count):
            raise ValueError("the session's input has ended")
        n = (len(self.pend) + count) // self.hop
        if flag == STEP:
            return n, n
        if self.K:
            return 0, max(0, self.K + self.la + 2 - self.t)
        if (self.t + n) * self.hop + (len(self.pend) + count) % self.hop <= self.hop:
            raise ValueError("a session of L <= n_fft / 2 samples")
        return n, n + self.la + 2

    def call(self, flag, samples, mask_of):
        samples = np.asarray(samples, np.float64)
        self.plan_call(flag, len(samples))
        if flag == HOLD:
            return np.zeros(0)
        if flag == START:
            self.t, self.K, self.r_end, self.pend = 0, 0, 0, np.zeros(0)
            self.hist = np.zeros((3, self.hop))
        out = []
        if not self.K:
            pend = np.concatenate([self.pend, samples])
            while len(pend) >= self.hop:
                o = self.tick(START if self.t == 0 else STEP, pend[:self.hop], mask_of)
                pend = pend[self.hop:]
                if o is not None:
                    out.append(o)
            self.pend = pend
            self.hist[self.t % 3, :len(pend)] = pend
        if flag == FLUSH:
            if not self.K:                            # K hops and r_end samples (hop + 1 <= L: K = 1 is a session when r_end > 0)
                self.K, self.r_end, self.pend = self.t, len(self.pend), np.zeros(0)
            while (o := self.tick(FLUSH, None, mask_of)) is not None or self.t <= self.K + self.la + 1:
                if o is not None:
                    out.append(o)
            if self.r_end:                            # once, after frame K
                out.append(self.tail[:self.r_end] * self.inv_last[:self.r_end])
                self.r_end = 0
        return np.concatenate(out) if out else np.zeros(0)


def packets(L, size, rng):
    """Packet sizes summing to L: `size` each (None: all at once, 0: random 0..3 hops' worth, zeros included)."""
    if size is None:
        return [L]
    out, left = [], L
    while left:
        n = min(left, size if size else int(rng.integers(0, 700)))
        out.append(n)
        left -= n
    return out


def run(n_fft, la, x, sizes, crm, holds=0.0, rng=None):
    """A session fed in packets of `sizes` (the last one FLUSHes; with holds, HOLD calls in between).  Returns the concatenated output
    and, per call, (input so far, output so far, the call's packet)."""
    ref = SampleSlotRef(n_fft, la)
    mask_of = lambda m: crm[:, :, m]
    got, log, i = [], [], 0
    for c, n in enumerate(sizes):
        while holds and rng.random() < holds:
            assert ref.call(HOLD, np.zeros(0), mask_of).size == 0
        flag = START if c == 0 else FLUSH if c == len(sizes) - 1 else STEP
        got.append(ref.call(flag, x[i:i + n], mask_of))
        i += n
        log.append((i, sum(len(g) for g in got), n))
    if len(sizes) == 1:                                   # one packet: START, then a FLUSH of nothing
        got.append(ref.call(FLUSH, np.zeros(0), mask_of))
        log.append((i, sum(len(g) for g in got), 0))
    return np.concatenate(got), log


def lengths(hop, rng):
    return [hop + 1, 2 * hop - 1, 2 * hop, 2 * hop + 1, 5 * hop + 37, int(rng.integers(hop + 1, 9 * hop))]


@pytest.mark.parametrize("n_fft", [64, 128, 256, 512, 1024])
@pytest.mark.parametrize("size", [1, 7, 160, 256, 320, 1000, None])
def test_sample_stream_equals_offline(n_fft, size):
    hop, la = n_fft // 2, 2
    rng = np.random.default_rng(n_fft * 7 + (size or 0))
    for L in lengths(hop, rng):
        if size == 1 and L > 3 * hop:
            continue                                      # one sample per call over thousands of calls adds nothing at 5 hops
        x = rng.standard_normal(L)
        crm = rng.standard_normal((2, hop + 1, L // hop + 1)) * 0.5
        got, log = run(n_fft, la, x, packets(L, size, rng), crm)
        want = offline(x, crm, n_fft)
        assert got.shape == (L,), f"L={L}: {got.shape}"
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-10 * max(1.0, np.abs(want).max()), err_msg=f"n_fft={n_fft} L={L}")


@pytest.mark.parametrize("la", [0, 1, 2, 3])
def test_random_schedules_and_latency(la):
    """Random packet sizes (zeros included) and HOLD calls: offline equality, and the emission counts of the latency rule -- after a
    call that is not the FLUSH, exactly the samples of hops q with (q + la + 3) hop <= input are out; after it, all L."""
    n_fft, hop = 128, 64
    rng = np.random.default_rng(31 + la)
    for trial in range(12):
        L = int(rng.integers(hop + 1, 14 * hop))
        x = rng.standard_normal(L)
        crm = rng.standard_normal((2, hop + 1, L // hop + 1)) * 0.5
        got, log = run(n_fft, la, x, packets(L, 0, rng), crm, holds=0.2, rng=rng)
        np.testing.assert_allclose(got, offline(x, crm, n_fft), rtol=0, atol=1e-10 * max(1.0, np.abs(got).max()))
        prev_in, prev_out = 0, 0
        for c, (i, o, n) in enumerate(log):
            if c < len(log) - 1:
                assert o == hop * max(0, i // hop - la - 2), f"L={L} call {c}: input {i}, output {o}"
            else:
                assert o == L
            lag = prev_in - prev_out                      # the header's bound on one call's output
            assert lag <= (la + 2) * hop + prev_in % hop and o - prev_out <= n + (la + 3) * hop
            prev_in, prev_out = i, o


@pytest.mark.parametrize("n_fft", [64, 512])
def test_whole_hops_equal_the_hop_ticks(n_fft):
    """Fed whole hops and ended on a hop boundary, the sample slot runs the per-hop emulation's ticks: the same hop out of each."""
    hop, la = n_fft // 2, 2
    rng = np.random.default_rng(n_fft)
    K = 9
    x = rng.standard_normal(K * hop)
    crm = rng.standard_normal((2, hop + 1, K + 1))
    mask_of = lambda m: crm[:, :, m]
    smp, per = SampleSlotRef(n_fft, la), AudioSlotRef(n_fft, la)
    for q in range(K):
        f = START if q == 0 else STEP
        a = smp.call(f, x[q * hop:(q + 1) * hop], mask_of)
        b = per.tick(f, x[q * hop:(q + 1) * hop], mask_of)
        assert (a.size == 0 and b is None) or np.array_equal(a, b), f"hop {q}"
    a = smp.call(FLUSH, np.zeros(0), mask_of)
    b = []
    while (o := per.tick(FLUSH, None, mask_of)) is not None or per.t <= per.K + la + 1:
        if o is not None:
            b.append(o)
    assert np.array_equal(a, np.concatenate(b))


def test_refusals():
    hop, la = 32, 1
    ref = SampleSlotRef(2 * hop, la)
    mask_of = lambda m: np.zeros((2, hop + 1))
    with pytest.raises(ValueError):
        ref.call(STEP, np.zeros(3), mask_of)                # no session
    ref.call(START, np.zeros(hop - 1), mask_of)
    with pytest.raises(ValueError):
        ref.call(FLUSH, np.zeros(1), mask_of)               # L = hop
    assert ref.t == 0 and len(ref.pend) == hop - 1          # a refused call changes nothing
    ref.call(FLUSH, np.zeros(2), mask_of)                   # L = hop + 1 is the shortest session
    with pytest.raises(ValueError):
        ref.call(STEP, np.zeros(0), mask_of)
    with pytest.raises(ValueError):
        ref.call(FLUSH, np.zeros(1), mask_of)
    assert ref.call(FLUSH, np.zeros(0), mask_of).size == 0  # a FLUSH of nothing after the end is a HOLD


def test_binding_declares_the_call(built_lib):
    from fsnplus_b200 import _lib
    assert "fsn_stream_step_audio_samples" in _lib.SYMBOLS
    assert len(built_lib.fsn_stream_step_audio_samples.argtypes) == 8
