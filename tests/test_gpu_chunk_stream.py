"""Overlapped-chunk sessions on the device (fsn_chunk_stream_*, ChunkStream; DESIGN.md §3.16).

Staggered sessions with holds, per-slot counts that vary per call, slot reuse, L = 1 and L a multiple of H, NaN in every unread
sample: each session's concatenated output equals the stitch (tests/chunk_stream_ref.py, cross-fade in fp64) of enhance_audio on that
session's chunk rows, and is bit-identical to the same session run alone on a 1-slot handle.  End to end against the fp64 pipeline per
chunk for FullSubNet+ (TSSE), FullSubNet+ with the sub-band TCN and fullsubnet.Model with offline_laplace_norm; under a small
workspace cap (sub-batches, same bits); every error, each followed by a call that must match a handle that never saw the bad one."""
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
STITCH_TOL = 1e-6         # a session vs the fp64 stitch of enhance_audio on its chunk rows
WAVE_TOL = 2e-3           # a session vs chunk_stream_ref over the fp64 pipeline (the audio tests' waveform bar)


def _model(cls, cfg, params, monkeypatch=None, cap_gb=None):
    if monkeypatch is not None:
        if cap_gb is None:
            monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
        else:
            monkeypatch.setenv("FSN_WS_CAP_GB", str(cap_gb))
    m = cls(**cfg)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()}, strict=True)
    m = m.to(DEV).eval()
    with torch.cuda.device(DEV):
        m._ensure_handle(torch.device(DEV))
    if monkeypatch is not None:
        monkeypatch.delenv("FSN_WS_CAP_GB", raising=False)
    return m


def _small_plus(**over):
    c = O.default_plus_config()
    c.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)
    c.update(over)
    return c


def _build(kind, seed=3, monkeypatch=None, cap_gb=None):
    """(model, cfg, oracle kind, params) of a small FullSubNet+ ("plus"), the same with the sub-band TCN ("tcn"), a small
    fullsubnet.Model with offline_laplace_norm ("fsn") or the default FullSubNet+ ("default")."""
    from fsnplus_b200.model import FullSubNet_Plus, Model
    cls = FullSubNet_Plus
    if kind == "plus":
        cfg = _small_plus()
        params = O.make_params_plus(cfg, seed=seed)
    elif kind == "tcn":
        cfg = _small_plus(sb_model_hidden_size=32, sequence_model="TCN")
        params = SB.make_params(cfg, seed=seed)
    elif kind == "fsn":
        cls, cfg = Model, O.default_fsn_config()
        cfg.update(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=32, fb_model_hidden_size=48)
        params = O.make_params_fsn(cfg, seed=seed)
    else:
        cfg, kind = O.default_plus_config(), "plus"
        params = O.make_params_plus(cfg, seed=seed)
    return _model(cls, cfg, params, monkeypatch, cap_gb), cfg, kind, params


def _bank(seed, n=200000):
    return O.synth_clips(2, num_samples=n, seed0=seed).reshape(-1).astype(np.float32)


def _schedule(B, H, calls, seed, S_choices, special=(1, 256, 512, 768)):
    """Per call (S, flags, counts, sessions started): each slot runs sessions one after another, some of the special lengths (L = 1,
    multiples of H), the rest random; STARTs staggered, HOLDs mid-session, counts of 0 / 1 / S / random, a session's last samples in its
    FLUSH call (or a FLUSH of 0), and now and then a START that abandons the running session."""
    rng = np.random.default_rng(seed)
    special = list(special)
    rem = [None] * B
    out = []
    for _ in range(calls):
        S = int(rng.choice(S_choices))
        fl, ct = [SLOT_HOLD] * B, [0] * B
        for b in range(B):
            c = int(rng.choice([0, 1, S, int(rng.integers(0, S + 1))]))
            if rem[b] is None or (rng.random() < 0.02 and rem[b] > 0):
                if rng.random() < 0.4:
                    continue
                L = special.pop() if special and rng.random() < 0.5 else int(rng.integers(1, 7 * H))
                c = max(1, min(c, L))
                fl[b], ct[b], rem[b] = SLOT_START, c, L - c
            elif rng.random() < 0.15:
                continue
            elif rem[b] <= c:
                fl[b], ct[b], rem[b] = SLOT_FLUSH, rem[b], None
            else:
                fl[b], ct[b], rem[b] = SLOT_STEP, c, rem[b] - c
        out.append((S, fl, ct))
    for b in range(B):                                     # end every session
        if rem[b] is not None:
            fl = [SLOT_HOLD] * B
            ct = [0] * B
            fl[b], ct[b] = SLOT_FLUSH, rem[b]
            out.append((max(rem[b], 1), fl, ct))
    return out


def _drive(cs, sched, bank, seed):
    """Run the schedule; returns the sessions [(slot, calls [(flag, count, samples)], x, y, flushed)]."""
    rng = np.random.default_rng(seed)
    B, Cc = cs.B, cs.C
    cur = [None] * B
    sessions = []
    for S, fl, ct in sched:
        x = np.full((B, S), np.nan, np.float32)
        for b in range(B):
            if fl[b] != SLOT_HOLD:
                o = int(rng.integers(0, bank.shape[0] - ct[b]))
                x[b, :ct[b]] = bank[o:o + ct[b]]
        out, nout = cs.step(torch.from_numpy(x).to(DEV), ct, fl)
        out = out.cpu().numpy()
        assert out.shape == (B, S + Cc)
        for b in range(B):
            n = int(nout[b])
            if fl[b] == SLOT_HOLD:
                assert n == 0 and not out[b].any()
                continue
            if fl[b] == SLOT_START:
                cur[b] = dict(slot=b, calls=[], x=[], y=[], flushed=False)
                sessions.append(cur[b])
            s = cur[b]
            s["calls"].append((fl[b], ct[b], x[b, :ct[b]].copy()))
            s["x"].append(x[b, :ct[b]])
            s["y"].append(out[b, :n].copy())
            assert not out[b, n:].any() and np.isfinite(out[b, :n]).all()
            if fl[b] == SLOT_FLUSH:
                s["flushed"] = True
                cur[b] = None
    for s in sessions:
        s["x"], s["y"] = np.concatenate(s["x"]), np.concatenate(s["y"])
    return sessions


def _enhance_rows(m):
    def f(rows):
        with torch.no_grad():
            return m.enhance_audio(torch.from_numpy(np.ascontiguousarray(rows, np.float32)).to(DEV)).cpu().numpy()
    return f


def _check_sessions(sessions, C, enhance, tol, what):
    worst = 0.0
    for s in sessions:
        x, y = s["x"], s["y"]
        want = R.chunk_stream_ref(x, C, enhance)
        if s["flushed"]:
            assert y.shape == x.shape, (what, s["slot"], y.shape, x.shape)
        else:                                              # abandoned by a START: y[0, k H) of what it consumed
            assert y.shape[0] == max(0, x.shape[0] // (C // 2) - 1) * (C // 2)
            want = want[:y.shape[0]]
        if y.size:
            e = O.rel_l2(y, want) if np.abs(want).max() > 0 else float(np.abs(y).max())
            worst = max(worst, e)
            assert e <= tol, (what, s["slot"], x.shape[0], e)
    print(f"\n[{what}] {len(sessions)} sessions, worst rel-L2 {worst:.2e}")
    return worst


def _alone(m, C, s):
    from fsnplus_b200.streaming import ChunkStream
    cs = ChunkStream(m, 1, C, DEV)
    ys = []
    for f, c, xs in s["calls"]:
        S = max(c, 1)
        x = np.full((1, S), np.nan, np.float32)
        x[0, :c] = xs
        out, nout = cs.step(torch.from_numpy(x).to(DEV), [c], [f])
        ys.append(out.cpu().numpy()[0, :int(nout[0])])
    cs.close()
    return np.concatenate(ys)


@pytest.mark.parametrize("C", [512, 640])
def test_stitched_sessions_and_batch_independence(built_lib, C):
    """80 slots at F = 33: every session equals the stitch of enhance_audio on its rows, and its lone run bit for bit."""
    from fsnplus_b200.streaming import ChunkStream
    m, cfg, _, _ = _build("plus")
    H = C // 2
    sched = _schedule(80, H, 40, seed=C, S_choices=[1, 37, 160, 320, 700, 1500], special=(1, 1, H, 2 * H, 3 * H, 4 * H))
    cs = ChunkStream(m, 80, C, DEV)
    sessions = _drive(cs, sched, _bank(5), seed=C + 1)
    cs.close()
    assert len(sessions) >= 120 and sum(s["flushed"] for s in sessions) >= 100
    lengths = {s["x"].shape[0] for s in sessions if s["flushed"]}
    assert 1 in lengths and any(n and n % H == 0 for n in lengths)
    _check_sessions(sessions, C, _enhance_rows(m), STITCH_TOL, f"stitch C={C}")
    same = 0
    for s in sessions:
        alone = _alone(m, C, s)
        assert np.array_equal(alone, s["y"]), (s["slot"], s["x"].shape[0])
        same += 1
    print(f"[alone C={C}] {same} sessions bit-identical to their lone runs")


def test_default_geometry(built_lib):
    """The default FullSubNet+ (F = 257, hop 256) with 1 s chunks at 16 kHz, 6 slots."""
    from fsnplus_b200.streaming import ChunkStream
    m, cfg, _, _ = _build("default")
    C = 16000
    sched = _schedule(6, C // 2, 30, seed=9, S_choices=[320, 4000, 9000], special=(1, 8000, 24000))
    cs = ChunkStream(m, 6, C, DEV)
    sessions = _drive(cs, sched, _bank(6, 400000), seed=10)
    cs.close()
    assert sum(s["flushed"] for s in sessions) >= 6
    _check_sessions(sessions, C, _enhance_rows(m), STITCH_TOL, "stitch default")


def _fp64_rows(m, cfg, kind, params):
    F = cfg["num_freqs"]
    n_fft, hop = 2 * (F - 1), F - 1

    def f(rows):
        out = []
        for row in np.asarray(rows, np.float64):
            X = O.stft(row[None], n_fft, hop, n_fft)
            mag, real, imag = np.abs(X)[:, None], X.real[:, None], X.imag[:, None]
            if kind == "fsn":
                crm = O.fullsubnet_forward(params, cfg, mag)
            elif kind == "tcn":
                crm = SB.forward(params, cfg, mag, real, imag)
            else:
                crm = O.fullsubnet_plus_forward(params, cfg, mag, real, imag)
            out.append(O.istft(O.enhance(X, crm), n_fft, hop, n_fft, length=row.shape[0])[0])
        return np.stack(out)
    return f


@pytest.mark.parametrize("kind", ["plus", "tcn", "fsn"])
def test_end_to_end_against_fp64(built_lib, kind):
    from fsnplus_b200.streaming import ChunkStream
    m, cfg, kind, params = _build(kind, seed=7)
    C = 512
    sched = _schedule(4, C // 2, 12, seed=11, S_choices=[100, 333, 900], special=(1, 768))
    cs = ChunkStream(m, 4, C, DEV)
    sessions = _drive(cs, sched, _bank(12), seed=13)
    cs.close()
    _check_sessions(sessions, C, _fp64_rows(m, cfg, kind, params), WAVE_TOL, f"fp64 {kind}")


def test_capped_handle_is_bit_identical(built_lib, monkeypatch):
    """A model whose cap fits 8 chunk rows per sub-batch: the same outputs bit for bit, and the burst call ran in sub-batches."""
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import ChunkStream
    C, B = 512, 40
    m, cfg, _, _ = _build("plus", seed=4)
    cap = _lib.plan_audio(m._cfg, 8, P + C, cap_bytes=1e12)[3] * 1.02 / 1e9
    mc, _, _, _ = _build("plus", seed=4, monkeypatch=monkeypatch, cap_gb=cap)
    sched = [(C, [SLOT_START] * B, [C] * B), (C, [SLOT_STEP] * B, [C] * B), (300, [SLOT_FLUSH] * B, list(range(0, 300, 300 // B))[:B])]
    res = []
    for model in (m, mc):
        cs = ChunkStream(model, B, C, DEV)
        res.append(_drive(cs, sched, _bank(14), seed=15))
        cs.close()
    # the last call's batch: slot b's chunks 3 .. ceil((2 C + count) / H) - 1, all at its FLUSH
    n = sum(-(-(2 * C + c) // (C // 2)) - 3 for c in sched[-1][2])
    bs, tw, fc = mc.last_plan_bins()
    assert bs < n and (bs, tw, fc) == tuple(_lib.plan_audio(mc._cfg, n, P + C, cap_bytes=cap * 1e9)[:3]), (n, bs, tw, fc)
    assert mc.last_plan()[0] == bs
    for a, b in zip(*res):
        assert np.array_equal(a["y"], b["y"])
    print(f"\n[cap] {n} rows in the last call, in sub-batches of {bs}")


def test_errors_change_nothing(built_lib):
    from fsnplus_b200 import _lib
    from fsnplus_b200.streaming import ChunkStream
    lib = _lib.load_library()
    m, cfg, _, _ = _build("plus", seed=5)
    h = C.c_void_p()
    for Cc, B, msg in [(513, 2, "even"), (510, 2, "pre-context"), (512, 0, "B = 0")]:
        assert lib.fsn_chunk_stream_create(m._handle, B, Cc, C.byref(h)) == -1
        assert msg in lib.fsn_last_error().decode()
    assert lib.fsn_chunk_stream_create(None, 2, 512, C.byref(h)) == -1
    assert lib.fsn_chunk_stream_create(m._handle, 2, 512, None) == -1
    md, _, _, _ = _build("default", seed=5)                   # rows of 256 + 512 samples are too short for the TSSE kernels
    assert lib.fsn_chunk_stream_create(md._handle, 2, 512, C.byref(h)) == -1
    err = lib.fsn_last_error().decode()
    assert "chunk_samples = 512" in err and "TSSE kernel size" in err, err
    raw = C.c_void_p()                                     # a model that has not been finalized
    _lib.check(lib.fsn_model_create(C.byref(m._cfg), C.byref(raw)))
    assert lib.fsn_chunk_stream_create(raw, 2, 512, C.byref(h)) == -3
    lib.fsn_model_destroy(raw)

    Cc, B, S = 512, 3, 400
    cs, twin = ChunkStream(m, B, Cc, DEV), ChunkStream(m, B, Cc, DEV)
    bank = _bank(16)
    rng = np.random.default_rng(17)

    def rows():
        x = np.full((B, S), np.nan, np.float32)
        x[:, :S] = bank[rng.integers(0, 100000):][:B * S].reshape(B, S)
        return torch.from_numpy(x).to(DEV)

    def both(x, counts, flags):
        a, na = cs.step(x, counts, flags)
        b, nb = twin.step(x, counts, flags)
        assert np.array_equal(a.cpu().numpy(), b.cpu().numpy()) and np.array_equal(na.numpy(), nb.numpy())

    x = rows()
    bad = [([SLOT_STEP, SLOT_HOLD, SLOT_HOLD], [1, 0, 0], "slot 0: STEP on a slot without a session"),
           ([SLOT_HOLD, SLOT_FLUSH, SLOT_HOLD], [0, 0, 0], "slot 1: FLUSH on a slot without a session")]
    for fl, ct, msg in bad:
        with pytest.raises(_lib.FsnError, match=msg):
            cs.step(x, ct, fl)
    both(x, [S, 5, 0], [SLOT_START, SLOT_START, SLOT_HOLD])
    bad = [([SLOT_STEP, 4, SLOT_HOLD], [1, 1, 0], "slot 1: flag 4"),
           ([SLOT_STEP, SLOT_STEP, SLOT_HOLD], [1, S + 1, 0], "slot 1: h_counts = 401"),
           ([SLOT_STEP, SLOT_STEP, SLOT_HOLD], [-1, 1, 0], "slot 0: h_counts = -1"),
           ([SLOT_STEP, SLOT_STEP, SLOT_STEP], [1, 1, 1], "slot 2: STEP on a slot without a session")]
    for _ in range(2):
        x = rows()
        for fl, ct, msg in bad:
            with pytest.raises(_lib.FsnError, match=msg):
                cs.step(x, ct, fl)
        both(x, [S, 7, -5], [SLOT_STEP, SLOT_STEP, SLOT_HOLD])    # a HOLD ignores its count
    stream = C.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    fl, ct, no = (C.c_int32 * B)(1, 1, 0), (C.c_int32 * B)(1, 1, 0), (C.c_int32 * B)()
    out = torch.empty((B, S + Cc), device=DEV)
    xp, op = C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr())
    for args, msg in [((None, S, fl, ct, op, no), "d_samples is null"), ((xp, S, None, ct, op, no), "h_flags is null"),
                      ((xp, S, fl, None, op, no), "h_counts is null"), ((xp, S, fl, ct, None, no), "d_out is null"),
                      ((xp, S, fl, ct, op, None), "h_nout is null"), ((xp, 0, fl, ct, op, no), "S = 0")]:
        assert lib.fsn_chunk_stream_step(cs._cs, *args, stream) == -1
        assert msg in lib.fsn_last_error().decode()
    for _ in range(3):
        both(rows(), [S, S, 0], [SLOT_STEP, SLOT_STEP, SLOT_HOLD])
    both(rows(), [3, 0, 0], [SLOT_FLUSH, SLOT_FLUSH, SLOT_HOLD])
    with pytest.raises(_lib.FsnError, match="slot 0: STEP on a slot without a session"):
        cs.step(rows(), [1, 0, 0], [SLOT_STEP, SLOT_HOLD, SLOT_HOLD])
    both(rows(), [9, 0, 0], [SLOT_START, SLOT_HOLD, SLOT_HOLD])
    cs.close()
    twin.close()
