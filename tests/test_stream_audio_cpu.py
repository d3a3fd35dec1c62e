"""CPU: the tick schedule of the audio streaming call (DESIGN.md §3.10), emulated in fp64 by stream_audio_ref, reproduces the offline
pipeline O.istft(O.enhance(O.stft(x), crm), length=L) for any masks, emits hop q at slot tick q + look_ahead + 2, and rejects the
calls the C ABI rejects."""
import numpy as np
import pytest

import stream_audio_ref as R


def _session(n_fft, la, K, rng, hold_p=0.3, extra_flush=2):
    """One session of K hops with random masks and random HOLD ticks: returns (streamed waveform, reference, emission ticks)."""
    ref_slot = R.AudioSlotRef(n_fft, la)
    hop, F = n_fft // 2, n_fft // 2 + 1
    x = rng.standard_normal(K * hop)
    crm = rng.uniform(-3, 3, (2, F, K + 1))
    crm[:, :, rng.integers(0, K + 1)] = rng.uniform(-12, 12, (2, F))     # one frame past the +-9.9 clamp
    flags = [R.START] + [R.STEP] * (K - 1) + [R.FLUSH] * (la + 2 + extra_flush)
    out, when, k, q = {}, {}, 0, 0
    for f in flags:
        while rng.random() < hold_p:
            assert ref_slot.tick(R.HOLD) is None
        y = ref_slot.tick(f, x[q * hop:(q + 1) * hop] if f != R.FLUSH else None, lambda m: crm[:, :, m])
        if f != R.FLUSH:
            q += 1
        if y is not None:
            out[len(out)] = y
            when[len(when)] = k
        k += 1
    assert len(out) == K
    return np.concatenate([out[i] for i in range(K)]), R.offline(x, crm, n_fft), [when[i] for i in range(K)]


@pytest.mark.parametrize("n_fft", [64, 128, 512, 1024])
@pytest.mark.parametrize("la", [0, 1, 2, 3])
def test_schedule_reproduces_offline_pipeline(n_fft, la):
    rng = np.random.default_rng(n_fft * 10 + la)
    for K in range(2, 10):
        got, ref, when = _session(n_fft, la, K, rng)
        err = np.abs(got - ref).max()
        assert err <= 1e-12 * max(1.0, np.abs(ref).max()), (K, err)
        assert when == [q + la + 2 for q in range(K)], (K, when)


def test_schedule_table():
    """The per-tick plan (model count, frame analysed, zero frame, frame synthesised) of a 3-hop session at look_ahead 2."""
    s = R.AudioSlotRef(64, 2)
    got = []
    for f in [R.START, R.STEP, R.STEP] + [R.FLUSH] * 5:
        got.append(s.plan(f))
        s.tick(f, np.zeros(32), lambda m: np.zeros((2, 33)))
    assert got == [(0, -1, None, False, None), (1, 0, 0, False, None), (2, 1, 1, False, None), (3, 2, 2, False, 0),
                   (4, 3, 3, False, 1), (5, 4, None, True, 2), (6, 5, None, True, 3), None]


def test_rejected_calls():
    s = R.AudioSlotRef(128, 2)
    with pytest.raises(ValueError):
        s.tick(R.STEP, np.zeros(64))                                    # no session
    with pytest.raises(ValueError):
        s.tick(R.FLUSH)
    s.tick(R.START, np.zeros(64))
    with pytest.raises(ValueError, match="at least 2"):
        s.tick(R.FLUSH)                                                 # K = 1: the reflect padding needs more than n_fft / 2 samples
    s.tick(R.STEP, np.zeros(64))
    s.tick(R.FLUSH, None, lambda m: np.zeros((2, 65)))
    with pytest.raises(ValueError):
        s.tick(R.STEP, np.zeros(64))                                    # STEP after the flush without a START
    with pytest.raises(ValueError):
        s.tick(7)
