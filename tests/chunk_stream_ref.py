"""numpy restatement of the overlapped-chunk sessions (fsn_chunk_stream_*, ChunkStream; DESIGN.md §3.16) and of the reference loop
they follow (fullsubnet_plus/inferencer/inferencer.py:191-250, ``overlapped_chunk``).

C: chunk length (even), H = C / 2, P = 256 samples of pre-context, w = periodic Hann window of C.  Chunk k = 0 .. ceil(L / H) - 1 of
a session x[0, L) is the row x[k H - P, k H + C), zero before 0 and past L; e_k is its enhancement minus the first P samples.  Output
region k = y[k H, (k + 1) H) is e_0[0, H) (k = 0) or e_k[0, H) w[0, H) + e_{k-1}[H, C) w[H, C); the output is y[0, L).

``fault`` plants one of the errors the CPU tests must catch: "window_first" (chunk 0 windowed), "pre_offset" (pre-context taken one
sample early), "tail_twice" (the tail windowed twice), "drop_last" (the last region dropped)."""
import numpy as np

P = 256
SLOT_HOLD, SLOT_STEP, SLOT_START, SLOT_FLUSH = 0, 1, 2, 3


def hann(C):
    """torch.hann_window(C) (periodic) in float64: w[i] + w[i + C / 2] = 1."""
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * np.arange(C) / C)


def num_chunks(L, C, fault=None):
    H = C // 2
    K = -(-L // H)
    return K - 1 if fault == "drop_last" and K else K


def chunk_rows(x, C, fault=None):
    """The input rows [K, P + C] of session x (1-D), zero before 0 and past len(x)."""
    x = np.asarray(x)
    L, H = x.shape[0], C // 2
    K = num_chunks(L, C, fault)
    rows = np.zeros((K, P + C), x.dtype)
    for k in range(K):
        idx = np.arange(k * H - P, k * H + C)
        if fault == "pre_offset" and k:      # only the pre-context comes from the wrong offset
            idx[:P] -= 1
        ok = (idx >= 0) & (idx < L)
        rows[k, ok] = x[idx[ok]]
    return rows


def stitch(enh, C, L, fault=None):
    """y[0, L) in float64 from the enhanced rows enh [K, P + C] (K = ceil(L / H), or fewer with "drop_last")."""
    H = C // 2
    w = hann(C)
    y = np.zeros(max(len(enh), num_chunks(L, C)) * H)
    tail = np.zeros(H)
    for k, row in enumerate(np.asarray(enh, np.float64)):
        e = row[P:]
        first = e[:H] * w[:H] if fault == "window_first" and k == 0 else e[:H] if k == 0 else e[:H] * w[:H] + tail
        y[k * H:(k + 1) * H] = first
        tail = e[H:] * w[H:] * (w[H:] if fault == "tail_twice" else 1.0)
    return y[:L]


def chunk_stream_ref(x, C, enhance, fault=None):
    """The session's output y[0, L): enhance maps rows [K, P + C] to enhanced rows of the same shape."""
    rows = chunk_rows(x, C, fault)
    enh = enhance(rows) if len(rows) else rows
    return stitch(enh, C, len(x), fault)


def reference_loop(noisy, C, model):
    """inferencer.py:191-250 line for line with num_mics = 1 and every chunk full length: the input is zero-padded past its end, so the
    last chunk has C samples too (the reference's is shorter).  model maps one row [P + C] to one enhanced row."""
    noisy = np.asarray(noisy, np.float64)
    L = noisy.shape[-1]
    chunk_length = C
    chunk_hop_length = chunk_length // 2
    num_chunks_ = int(L / chunk_hop_length) + 1
    noisy = np.concatenate([noisy, np.zeros((num_chunks_ + 1) * chunk_hop_length)])
    win = hann(chunk_length)
    prev = None
    enhanced = None
    for chunk_idx in range(num_chunks_):
        if chunk_idx == 0:
            pad = np.zeros(256)
            chunk_start_position = chunk_idx * chunk_hop_length
            chunk_end_position = chunk_start_position + chunk_length
            noisy_chunk = np.concatenate((pad, noisy[chunk_start_position:chunk_end_position]))
            enhanced_chunk = model(noisy_chunk)
            enhanced_chunk = enhanced_chunk[256:]
            cur = enhanced_chunk[:chunk_length // 2]
            prev = enhanced_chunk[chunk_length // 2:] * win[chunk_length // 2:]
        else:
            pad = noisy[(chunk_idx * chunk_hop_length - 256):(chunk_idx * chunk_hop_length)]
            chunk_start_position = chunk_idx * chunk_hop_length
            chunk_end_position = chunk_start_position + chunk_length
            noisy_chunk = np.concatenate((pad, noisy[chunk_start_position:chunk_end_position]))
            enhanced_chunk = model(noisy_chunk)
            enhanced_chunk = enhanced_chunk[256:]
            enhanced_chunk = enhanced_chunk * win[:len(enhanced_chunk)]
            tmp = enhanced_chunk[:chunk_length // 2]
            cur = tmp[:min(len(tmp), len(prev))] + prev[:min(len(tmp), len(prev))]
            prev = enhanced_chunk[chunk_length // 2:]
        enhanced = cur if enhanced is None else np.concatenate((enhanced, cur))
    return enhanced[:L]


class ChunkSlotRef:
    """The host schedule of one slot (chunk_slot_plan in fsn_api.cu): n = samples of the session so far (None: no session), k = its
    chunks enhanced.  ``call`` returns (the chunks this call completes, the samples it emits) and advances the slot; it raises
    ValueError where the library returns FSN_EINVAL, before changing anything."""

    def __init__(self, C):
        self.C, self.H = C, C // 2
        self.n, self.k = None, 0

    def call(self, flag, count, S):
        H = self.H
        if flag not in (SLOT_HOLD, SLOT_STEP, SLOT_START, SLOT_FLUSH):
            raise ValueError(f"flag {flag}")
        if flag == SLOT_HOLD:
            return [], 0
        if not 0 <= count <= S:
            raise ValueError(f"count {count}")
        if flag != SLOT_START and self.n is None:
            raise ValueError("no session")
        n0, k0 = (0, 0) if flag == SLOT_START else (self.n, self.k)
        n = n0 + count
        kend = -(-n // H) if flag == SLOT_FLUSH else max(k0, n // H - 1)
        nout = n - k0 * H if flag == SLOT_FLUSH else (kend - k0) * H
        self.n, self.k = (None, 0) if flag == SLOT_FLUSH else (n, kend)
        return list(range(k0, kend)), nout
