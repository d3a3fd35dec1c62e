"""CPU: the audio chunk call (fsn_stream_step_audio_chunk, DESIGN.md §3.14) restated in fp64 numpy -- the per-slot plan of its K ticks
(fsn_api.cu, audio_slot_plan), the analysis kernel (hops from the history ring or the caller's row, spectra to the call's scratch),
the model columns and the synthesis kernel (spectra from the scratch or the ring, the tail across calls, the ring rewritten at the end)
-- against stream_audio_ref.AudioSlotRef stepped tick by tick with the expanded flags.  Outputs, masks, emitted-hop counts and the state
left behind must agree.  Also the ctypes signature and the null-handle message.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from stream_audio_ref import FLUSH, HOLD, START, STEP, AudioSlotRef
from oracle import fsn_oracle as O


def expand(flag, n, K):
    """The K per-hop flags a chunk call's (flag, n) stands for."""
    if flag == HOLD:
        return [HOLD] * K
    if flag == START:
        return [START] + [STEP] * (n - 1) + [HOLD] * (K - n)
    if flag == STEP:
        return [STEP] * n + [HOLD] * (K - n)
    return [STEP] * n + [FLUSH] * (K - n)


class ChunkSlotRef(AudioSlotRef):
    """One slot of the chunk call: the host plan, then the two kernels' loops with their index arithmetic."""

    def plan_chunk(self, flag, n, K):
        """(k0, na, start, nstore, hops, nout) as audio_slot_plan computes them; ValueError where it fails."""
        la = self.la
        t, Kh = self.t, (self.K if self.t >= 0 else 0)
        if flag == HOLD:
            return t, 0, 0, 0, Kh, 0
        if not (0 if flag == FLUSH else 1) <= n <= K:
            raise ValueError("h_hops")
        if flag == START:
            k0, na, start, hops = 0, n, 1, 0
        else:
            if t < 0:
                raise ValueError("no session")
            if flag == STEP and Kh:
                raise ValueError("STEP after FLUSH")
            if flag == FLUSH and Kh and n:
                raise ValueError("FLUSH with hops after FLUSH")
            if flag == FLUSH and not Kh and t + n < 2:
                raise ValueError("FLUSH after fewer than 2 hops")
            k0, start = t, 0
            if flag == STEP:
                na, hops = n, 0
            else:
                hops = Kh or (t + n if n < K else 0)        # n = K: no FLUSH tick yet, the end is not known
                na = max(0, min(K, hops + la + 2 - t)) if hops else n
        nout = max(0, k0 + na - max(k0, la + 2))
        return k0, na, start, n, hops, nout

    def chunk(self, flag, n, K, row, mask_of):
        """The call on this slot.  row [K hop]: the caller's samples; mask_of(m) -> [2, F].  Returns (out [K hop], nout, masks
        [2, F, K])."""
        H, F, R, la = self.hop, self.F, self.la + 1, self.la
        k0, na, start, nstore, hops, nout = self.plan_chunk(flag, n, K)
        out, umask = np.zeros(K * H), np.zeros((2, F, K))
        if flag == HOLD:
            return out, 0, umask
        if flag == START:
            self.hist, self.ring, self.tail = np.zeros((3, H)), np.zeros((R, F), complex), None
        kf, j0 = max(0, na - start), k0 + start - 1
        # analysis: active tick i at slot tick k0 + i stores row hop i (i < nstore); model column c = i - start analyses frame j
        sspec, L = np.zeros((K, F), complex), hops * H
        for i in range(na):
            k = k0 + i
            if i < nstore:
                self.hist[k % 3] = row[i * H:(i + 1) * H]
            if i < start:
                continue
            c, j = i - start, k - 1
            if not (hops and j > hops):
                p = np.abs(np.arange(H * (j - 1), H * (j + 1)))
                if L:
                    p = np.where(p >= L, 2 * (L - 1) - p, p)
                sspec[c] = np.fft.rfft(self.hist[(p // H) % 3, p % H] * self.w)
        # the model: column c is the mask of frame j0 + c - la (zero before frame 0)
        cols = [mask_of(j0 + c - la) if j0 + c - la >= 0 else np.zeros((2, F)) for c in range(kf)]
        # synthesis: frame m from the scratch if this call analysed it, else from the ring
        e = 0
        for c in range(kf):
            m = j0 + c - la
            if m < 0:
                continue
            X = sspec[m - j0] if m >= j0 else self.ring[m % R]
            cm = O.decompress_cIRM(np.asarray(cols[c], np.float64))
            E = (cm[0] * X.real - cm[1] * X.imag) + 1j * (cm[1] * X.real + cm[0] * X.imag)
            y = np.fft.irfft(E, n=self.n_fft) * self.w
            if m >= 1:
                out[e * H:(e + 1) * H] = (self.tail + y[:H]) * self.inv_env
                e += 1
            self.tail = y[H:]
        for i in range(start, na):
            umask[..., i] = cols[i - start]
        for c in range(max(0, kf - R), kf):
            self.ring[(j0 + c) % R] = sspec[c]
        assert e == nout
        if flag != HOLD:
            self.t, self.K = k0 + na, hops
        return out, nout, umask


def _masks(F, seed):
    rng = np.random.default_rng(seed)
    cache = {}

    def mask_of(m):
        if m not in cache:
            cache[m] = rng.uniform(-3, 3, (2, F))
        return cache[m]
    return mask_of


def _state_equal(a, b):
    assert a.t == b.t and (a.t < 0 or a.K == b.K)
    if a.t >= 0:
        np.testing.assert_allclose(a.hist, b.hist, rtol=0, atol=0)
        np.testing.assert_allclose(a.ring, b.ring, rtol=1e-12, atol=1e-12)
        if a.tail is None or b.tail is None:
            assert a.tail is None and b.tail is None
        else:
            np.testing.assert_allclose(a.tail, b.tail, rtol=1e-12, atol=1e-12)


def _drive(n_fft, la, calls, seed):
    """calls: [(K, flag, n)] on one slot; the chunk restatement against per-hop ticks, call by call."""
    hop = n_fft // 2
    ref, chk = AudioSlotRef(n_fft, la), ChunkSlotRef(n_fft, la)
    mask_of = _masks(hop + 1, seed)
    rng = np.random.default_rng(seed + 1)
    for K, flag, n in calls:
        nh = n if flag != HOLD else 0
        row = np.full(K * hop, np.nan)
        row[:nh * hop] = rng.standard_normal(nh * hop) * 0.1
        want_out, want_mask = [], np.zeros((2, hop + 1, K))
        for i, f in enumerate(expand(flag, n, K)):
            samples = row[i * hop:(i + 1) * hop] if f in (START, STEP) else None
            p = ref.plan(f)
            o = ref.tick(f, samples, mask_of)
            if o is not None:
                want_out.append(o)
            if p is not None and p[1] >= 0 and p[1] - la >= 0:
                want_mask[..., i] = mask_of(p[1] - la)
        out, nout, umask = chk.chunk(flag, n, K, row, mask_of)
        assert not np.isnan(out).any()
        assert nout == len(want_out)
        want = np.zeros(K * hop)
        if want_out:
            want[:nout * hop] = np.concatenate(want_out)
        np.testing.assert_allclose(out, want, rtol=1e-12, atol=1e-12)
        np.testing.assert_array_equal(umask, want_mask)
        _state_equal(chk, ref)


def _sessions(K, la, rng, n_sessions=3):
    """A single slot's calls: each session STARTs with 1..K hops, STEPs partial and full calls (HOLDs between), FLUSHes with 0..K
    hops, then sends FLUSH calls of 0 hops past its end."""
    calls = []
    for _ in range(n_sessions):
        total = 0
        n = int(rng.integers(1, K + 1))
        calls.append((K, START, n))
        total += n
        for _ in range(int(rng.integers(0, 4))):
            if rng.random() < 0.3:
                calls.append((K, HOLD, 0))
            n = int(rng.integers(1, K + 1))
            calls.append((K, STEP, n))
            total += n
        n = int(rng.integers(0, K + 1))
        if total + n < 2:
            n = 2 - total
        calls.append((K, FLUSH, n))
        calls += [(K, FLUSH, 0)] * int(rng.integers(1, 4 + (la + 2) // K))
    return calls


@pytest.mark.parametrize("n_fft", [64, 512, 1024])
@pytest.mark.parametrize("la", [0, 1, 2, 3])
def test_chunk_restatement_matches_per_hop(n_fft, la):
    rng = np.random.default_rng(n_fft * 10 + la)
    for K in range(1, 10):
        _drive(n_fft, la, _sessions(K, la, rng), seed=K)


@pytest.mark.parametrize("la", [0, 2, 3])
def test_chunk_edges(la):
    """START with n = 1 and n = K, FLUSH with n = 0 and n = K, a FLUSH spilling over into later calls, K varying per call."""
    K = 5
    _drive(64, la, [(K, START, 1), (K, STEP, 1), (K, FLUSH, 0), (K, FLUSH, 0), (K, FLUSH, 0)], 1)
    _drive(64, la, [(K, START, K), (K, FLUSH, K), (K, FLUSH, 0), (K, FLUSH, 0)], 2)
    _drive(64, la, [(3, START, 3), (1, STEP, 1), (9, STEP, 4), (2, FLUSH, 2), (1, FLUSH, 0), (7, FLUSH, 0), (4, FLUSH, 0),
                    (6, START, 2), (8, FLUSH, 8), (2, FLUSH, 0)], 3)
    _drive(512, la, [(1, START, 1), (1, STEP, 1), (37, FLUSH, 0), (3, HOLD, 0), (5, FLUSH, 0)], 4)


def test_plan_rejects():
    s = ChunkSlotRef(64, 1)
    for flag, n in ((STEP, 1), (FLUSH, 0)):
        with pytest.raises(ValueError, match="no session"):
            s.plan_chunk(flag, n, 4)
    for flag, n in ((START, 0), (START, 5), (STEP, 0), (FLUSH, -1), (FLUSH, 5)):
        with pytest.raises(ValueError, match="h_hops"):
            s.plan_chunk(flag, n, 4)
    s.chunk(START, 1, 4, np.zeros(4 * 32), _masks(33, 0))
    with pytest.raises(ValueError, match="fewer than 2"):
        s.plan_chunk(FLUSH, 0, 4)
    s.chunk(FLUSH, 1, 4, np.zeros(4 * 32), _masks(33, 0))
    with pytest.raises(ValueError, match="STEP after FLUSH"):
        s.plan_chunk(STEP, 1, 4)
    with pytest.raises(ValueError, match="hops after FLUSH"):
        s.plan_chunk(FLUSH, 1, 4)


def test_entry_point_signature(built_lib):
    from fsnplus_b200 import _lib
    lib = built_lib
    assert "fsn_stream_step_audio_chunk" in _lib.SYMBOLS
    vp, i32 = C.c_void_p, C.c_int32
    assert lib.fsn_stream_step_audio_chunk.argtypes == [vp, vp, i32, vp, vp, vp, vp, vp, vp]
    assert lib.fsn_stream_step_audio_chunk(None, None, 4, None, None, None, None, None, None) == -1
    assert "st is null" in lib.fsn_last_error().decode()
