"""fp64 emulation of one slot of the audio streaming call (fsn_stream_step_audio_slots, DESIGN.md §3.10).

It keeps the state the device keeps, in the same shape: the last three hops of input, a ring of the last look_ahead + 1 noisy
spectra and the second half of the last synthesised frame.  Each tick follows the schedule table of DESIGN.md §3.10:

    slot tick k | analysis                    | model row            | synthesis
    0 (START)   | store hop 0, no frame       | HOLD                 | -
    1 .. K      | frame k - 1                 | count k - 1          | frame k - 1 - la, if >= 0
    K + 1       | frame K (right reflect)     | count K              | as above
    K + 2 ..    | zero frame                  | count k - 1          | as above; the last tick synthesises frame K
    K + 1 + la  |                             |                      |

K is the number of hops, known at the first FLUSH (tick K).  The masks are taken as given: ``tick`` receives the mask of the frame
the model step produced this tick, so the emulation checks the transforms and the indices, not the model.
"""
import numpy as np

from oracle import fsn_oracle as O

HOLD, STEP, START, FLUSH = 0, 1, 2, 3


class AudioSlotRef:
    def __init__(self, n_fft, look_ahead):
        assert n_fft >= 4 and n_fft & (n_fft - 1) == 0
        self.n_fft, self.hop, self.la = n_fft, n_fft // 2, look_ahead
        self.F = self.hop + 1
        self.w = O.hann_periodic(n_fft)
        self.inv_env = 1.0 / (self.w[:self.hop] ** 2 + self.w[self.hop:] ** 2)
        self.t = -1                                   # ticks of the session so far, HOLD excluded; -1: no session

    def plan(self, flag):
        """What the tick does, without changing the state: None (no tick: HOLD, or a FLUSH after the last hop is out), or
        (k, model count, frame analysed or None, zero frame?, frame synthesised or None).  ValueError for a call the API rejects."""
        if flag == HOLD:
            return None
        if flag == START:
            return 0, -1, None, False, None
        if self.t < 0:
            raise ValueError("no session on this slot")
        k, K = self.t, self.K
        if flag == STEP:
            if K:
                raise ValueError("STEP after FLUSH")
        elif flag == FLUSH:
            if not K:
                if k < 2:
                    raise ValueError(f"FLUSH after {k} hop(s): a session needs at least 2")
                K = k
            if k > K + self.la + 1:
                return None
        else:
            raise ValueError(f"flag {flag}")
        j, m = k - 1, k - 1 - self.la
        real = not K or j <= K
        return k, k - 1, j if real else None, not real, m if m >= 0 else None

    def tick(self, flag, samples=None, mask_of=None):
        """One tick.  samples: the hop (START / STEP); mask_of(m) -> [2, F] cIRM of frame m.  Returns the output hop or None."""
        p = self.plan(flag)
        if p is None:
            return None
        k, _, j, zero, m = p
        if flag == START:
            self.t, self.K = 0, 0
            self.hist, self.ring, self.tail = np.zeros((3, self.hop)), np.zeros((self.la + 1, self.F), complex), None
        if flag == FLUSH and not self.K:
            self.K = k
        if flag in (START, STEP):
            self.hist[k % 3] = np.asarray(samples, np.float64)
        if j is not None:
            self.ring[j % (self.la + 1)] = np.fft.rfft(self._frame(j) * self.w)
        elif zero:
            self.ring[(k - 1) % (self.la + 1)] = 0
        out = None
        if m is not None:
            cm = O.decompress_cIRM(np.asarray(mask_of(m), np.float64))
            X = self.ring[m % (self.la + 1)]
            E = (cm[0] * X.real - cm[1] * X.imag) + 1j * (cm[1] * X.real + cm[0] * X.imag)
            y = np.fft.irfft(E, n=self.n_fft) * self.w
            if m >= 1:
                out = (self.tail + y[:self.hop]) * self.inv_env
            self.tail = y[self.hop:]
        self.t = k + 1
        return out

    def _frame(self, j):
        """Frame j of torch.stft(center=True, reflect): original samples [hop (j - 1), hop (j + 1)), reflected at both ends."""
        p = np.arange(self.hop * (j - 1), self.hop * (j + 1))
        p = np.abs(p)
        if self.K:
            L = self.K * self.hop
            p = np.where(p >= L, 2 * (L - 1) - p, p)
        return self.hist[(p // self.hop) % 3, p % self.hop]


def offline(x, crm, n_fft):
    """The offline pipeline the stream must reproduce: O.istft(O.enhance(O.stft(x), crm), length=L).  x [L], crm [2, F, K + 1]."""
    hop = n_fft // 2
    X = O.stft(np.asarray(x, np.float64)[None], n_fft, hop, n_fft)
    return O.istft(O.enhance(X, np.asarray(crm, np.float64)[None]), n_fft, hop, n_fft, length=len(x))[0]
