"""CPU checks of parking and resuming overlapped-chunk sessions (fsn_chunk_stream_save_slots / _load_slots; DESIGN.md §3.17).

The payload layout against its formula, the refusals of fsn_chunk_stream_state_layout, and a host restatement of save / load: a
session split at every phase of the half-chunk H, its state (ring, tail, n, k) copied raw into a slot whose buffers hold NaN, and
continued, equals the unsplit session exactly -- also when the session's counters are offset past 2^31."""
import ctypes as C

import numpy as np
import pytest

import chunk_stream_ref as R
from chunk_stream_ref import P, SLOT_FLUSH, SLOT_START, SLOT_STEP


def _layout(Cc):
    ring = (Cc + P) * 4
    tail_off = (ring + 15) // 16 * 16
    return (tail_off + Cc // 2 * 4 + 255) // 256 * 256


@pytest.mark.parametrize("Cc", [512, 514, 640, 16000, 32000])
def test_layout_formula(built_lib, Cc):
    from fsnplus_b200 import _lib
    stride, meta_bytes = _lib.chunk_state_layout(Cc)
    assert stride == _layout(Cc) and stride % 256 == 0
    assert meta_bytes == C.sizeof(_lib.FsnChunkSlotMeta) == 56


@pytest.mark.parametrize("Cc, msg", [(513, "must be even"), (1, "must be even"), (0, "must be even"),
                                     (510, "shorter than the 256-sample pre-context (chunk_samples >= 512)"),
                                     (2 ** 30, "exceeds 2^30 - 1 - 256")])
def test_layout_refusals(built_lib, Cc, msg):
    from fsnplus_b200 import _lib
    with pytest.raises(_lib.FsnError, match=msg.replace("(", r"\(").replace(")", r"\)").replace("^", r"\^")):
        _lib.chunk_state_layout(Cc)


class Slot:
    """One slot of a chunk handle: the ring [C + P] (session sample p at p mod (C + P)), the tail [H] and the host counters n (int64,
    -1 = no session) and k, stepped as chunk_slot_plan, chunk_gather_kernel and chunk_crossfade_kernel do.  Buffers start as NaN: a
    read of anything the session did not write shows."""

    def __init__(self, Cc):
        self.C, self.H, self.R = Cc, Cc // 2, Cc + P
        self.ring = np.full(self.R, np.nan)
        self.tail = np.full(self.H, np.nan)
        self.n, self.k = np.int64(-1), np.int64(0)
        self.w = R.hann(Cc)

    def save(self):
        return self.ring.copy(), self.tail.copy(), self.n, self.k

    def load(self, st):
        self.ring, self.tail, self.n, self.k = st[0].copy(), st[1].copy(), np.int64(st[2]), np.int64(st[3])

    def step(self, flag, x, enhance):
        H, Rr, c = self.H, self.R, x.shape[0]
        assert flag == SLOT_START or self.n >= 0
        n0, k0 = (np.int64(0), np.int64(0)) if flag == SLOT_START else (self.n, self.k)
        a0, n = k0 * H, n0 + c
        kend = (n + H - 1) // H if flag == SLOT_FLUSH else max(k0, n // H - 1)
        nc, rel0, rel1, lo = int(kend - k0), int(n0 - a0), int(n - a0), (-P if k0 else 0)
        phase = int(a0 % Rr)
        for v in (rel0, rel1, phase):                       # the int32 plan fields
            assert -2 ** 31 <= v < 2 ** 31
        nout = int(n - a0) if flag == SLOT_FLUSH else nc * H
        rows = np.zeros((nc, P + self.C))
        for i in range(nc):
            r = i * H - P + np.arange(P + self.C)
            ok = (r >= lo) & (r < rel1)
            cur, old = ok & (r >= rel0), ok & (r < rel0)
            rows[i, cur] = x[r[cur] - rel0]
            rows[i, old] = self.ring[(phase + r[old]) % Rr]
        r = np.arange(max(rel1 - Rr, rel0), rel1)
        self.ring[(phase + r) % Rr] = x[r - rel0]
        enh = enhance(rows) if nc else rows
        out = np.zeros(nc * H)
        tl = self.tail
        for i in range(nc):
            e = enh[i, P:]
            out[i * H:(i + 1) * H] = e[:H] if (lo == 0 and i == 0) else e[:H] * self.w[:H] + tl
            tl = e[H:] * self.w[H:]
        if nc:
            self.tail = tl
        self.n, self.k = (np.int64(-1), np.int64(0)) if flag == SLOT_FLUSH else (n, kend)
        return out[:nout]


def _enhance(rows):
    """A row-wise stand-in for the model: nonlinear and position-dependent, so a wrong row or a wrong offset shows."""
    pos = np.arange(rows.shape[1]) / rows.shape[1]
    return np.tanh(3 * rows) * (1 + pos) + 0.25 * np.roll(rows, 3, axis=1)


def _calls(lo, hi, S, first):
    """Calls consuming samples [lo, hi) in pieces of at most S: (flag, lo, hi); START first when `first`, FLUSH last when hi ends
    the session (flag decided by the caller)."""
    out = []
    p = lo
    while True:
        q = min(hi, p + S)
        out.append([SLOT_START if first and not out else SLOT_STEP, p, q])
        p = q
        if p >= hi:
            return out


def _run(slot, x, calls, end):
    ys = []
    for i, (f, lo, hi) in enumerate(calls):
        if end and i == len(calls) - 1:
            f = SLOT_FLUSH
        ys.append(slot.step(f, x[lo:hi], _enhance))
    return ys


def _session(x, Cc, split, S):
    """Output of x with the calls cut at `split`: saved there and resumed into a fresh slot (None: unsplit).  Returns (y, the state
    saved at the split)."""
    L = x.shape[0]
    if split is None:
        return np.concatenate(_run(Slot(Cc), x, _calls(0, L, S, True), True)), None
    a = Slot(Cc)
    ys = _run(a, x, _calls(0, split, S, True), False)
    st = a.save()
    b = Slot(Cc)
    b.load(st)
    rest = _calls(split, L, S, False) if split < L else [[SLOT_STEP, L, L]]
    ys += _run(b, x, rest, True)
    return np.concatenate(ys), st


@pytest.mark.parametrize("Cc", [512, 514])
def test_split_at_every_phase(Cc):
    """A session of 5 H + 37 samples split after every sample count 0 .. 3 H + 1 and at its end (n = 0, n < H, just before and after
    chunks 0 and 1 complete at 2 H and 3 H, a resume followed at once by FLUSH): each split equals the unsplit session exactly, which
    equals the fp64 stitch of chunk_stream_ref."""
    H = Cc // 2
    L = 5 * H + 37
    x = np.random.default_rng(Cc).standard_normal(L)
    S = 173
    y0, _ = _session(x, Cc, None, S)
    np.testing.assert_allclose(y0, R.chunk_stream_ref(x, Cc, _enhance), rtol=0, atol=1e-12)
    splits = list(range(0, 3 * H + 2)) + [L - 1, L]
    for s in splits:
        y, st = _session(x, Cc, s, S)
        assert st[2] == s and st[3] == max(0, s // H - 1), (s, st[2:])
        assert np.array_equal(y, y0), s
    # the calls right after the resume: the FLUSH of the rest comes at once when it fits one call
    y, _ = _session(x, Cc, L - S + 1, S)
    assert np.array_equal(y, y0)


def test_split_past_2_31():
    """The state of a session at n is moved to n + D (D a multiple of H past 2^31, not a multiple of C + P): ring rolled by D, k + D / H.
    The continuation is the same output: the 64-bit counters and the ring phase carry the session."""
    Cc = 514
    H, Rr = Cc // 2, Cc + P
    L = 7 * H + 11
    x = np.random.default_rng(3).standard_normal(L)
    S = 211
    D = np.int64((2 ** 31 // H + 5) * H)
    assert D > 2 ** 31 and D % Rr
    for s in (2 * H, 2 * H + 5, 3 * H - 1, 4 * H + 100):       # k >= 1: an offset session has no chunk 0
        a = Slot(Cc)
        _run(a, x, _calls(0, s, S, True), False)
        ring, tail, n, k = a.save()
        base, far = Slot(Cc), Slot(Cc)
        base.load((ring, tail, n, k))
        far.load((np.roll(ring, int(D % Rr)), tail, n + D, k + D // H))
        assert far.n > 2 ** 31 and int(far.k * H % Rr) != int(base.k * H % Rr)
        # the offset session reads x[p - D]: feed both the same samples
        rest = _calls(s, L, S, False)
        ya, yb = _run(base, x, rest, True), _run(far, x, rest, True)
        for u, v in zip(ya, yb):
            assert np.array_equal(u, v), s
        assert base.n == far.n == -1
