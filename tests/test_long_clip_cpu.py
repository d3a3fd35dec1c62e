"""CPU: the forward plan for long clips (fsn_plan_forward, DESIGN.md §3.7), the FSN_SB_WINDOW knob, and the command line's
``--max_batch_seconds`` and lone windowed batches.  The plan is a host function of the configuration, so no GPU is needed."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import fsn_oracle as O

HOP = 256


def _frames(seconds):
    return int(seconds * 16000) // HOP + 1


def _cfg(kind="plus", **over):
    from fsnplus_b200.model import FullSubNet_Plus, Model
    if kind == "plus":
        c = O.default_plus_config()
        c.update(over)
        return FullSubNet_Plus(**c)._cfg
    c = O.default_fsn_config()
    c.update(over)
    return Model(**c)._cfg


def _plan(cfg, B, T, cap, force=0):
    from fsnplus_b200 import _lib
    return _lib.plan_forward(cfg, B, T, cap, force)


def _bytes(cfg, B, T, Tw):
    """Exact workspace of (B, T, Tw): a forced window under an unlimited cap keeps the whole batch."""
    bs, tw, n = _plan(cfg, B, T, 1e18, Tw)
    assert (bs, tw) == (B, Tw)
    return n


def _per_sample_split(cfg, B, T, cap):
    """The sub-batch of the per-sample estimate (ws_bytes_per_sample), the only split before windows existed: default config."""
    F, Tp, H, L = 257.0, T + 2, 384, 2
    Cp = (257 + 31) // 32 * 32
    per = 3 * F * Tp * 4 * 2 + 3 * Tp * (4.0 * Cp + 512) * 4 + F * Tp * 128 + F * L * H * 4 + F * Tp * (4.0 * H + H) * 2
    bmax = max(1, int(cap / per))
    if B <= bmax:
        return B
    n = -(-B // bmax)
    return -(-B // n)


@pytest.mark.parametrize("B,seconds", [(1, 3), (2, 3), (64, 3), (256, 3), (1, 60), (1, 180)])
def test_fits_unwindowed_keeps_todays_split(built_lib, B, seconds):
    cfg = _cfg()
    bs, tw, n = _plan(cfg, B, _frames(seconds), 24e9)
    assert tw == 0 and bs == _per_sample_split(cfg, B, _frames(seconds), 24e9) and n <= 24e9


@pytest.mark.parametrize("kind", ["plus", "fsn"])
@pytest.mark.parametrize("B,seconds,cap", [(1, 240, 24e9), (1, 600, 24e9), (1, 3600, 24e9), (1, 7200, 24e9), (4, 1800, 24e9),
                                           (64, 3600, 24e9), (1, 90, 2e9), (3, 60, 2e9), (3, 60, 0.4e9)])
def test_windowed_plan_honours_cap_and_is_maximal(built_lib, kind, B, seconds, cap):
    cfg = _cfg(kind)
    T = _frames(seconds)
    Tp = T + 2
    bs, tw, n = _plan(cfg, B, T, cap)
    assert tw > 0 and tw % 32 == 0 and n <= cap and n == _bytes(cfg, bs, T, tw)
    if cap >= 2e9:
        assert tw >= 256
    # Bs maximal: the next larger equal split does not fit even with the smallest window tried at this level
    if bs < B:
        nxt = next(-(-B // k) for k in range(-(-B // bs) - 1, 0, -1) if -(-B // k) > bs)
        assert _bytes(cfg, nxt, T, min(256 if tw >= 256 else 32, (Tp + 31) // 32 * 32)) > cap
    # Tw maximal: one window fewer (evened out) does not fit
    nwin = -(-Tp // tw)
    if nwin > 1:
        longer = (-(-Tp // (nwin - 1)) + 31) // 32 * 32
        assert _bytes(cfg, bs, T, longer) > cap


def test_two_hour_clip_fits_default_cap(built_lib):
    for kind in ("plus", "fsn"):
        bs, tw, n = _plan(_cfg(kind), 1, 450000, 24e9)
        assert bs == 1 and tw >= 256 and n <= 24e9, kind


def test_nothing_fits_runs_one_clip_with_a_small_window(built_lib):
    bs, tw, n = _plan(_cfg(), 4, _frames(600), 1e8)
    assert (bs, tw) == (1, 256) and n > 1e8


def test_forced_window_and_paths_without_windows(built_lib):
    T = _frames(10)
    assert _plan(_cfg(), 2, T, 24e9, 96)[:2] == (2, 96)
    assert _plan(_cfg(lstm_impl="mma"), 2, _frames(3600), 24e9, 96)[1] == 0
    assert _plan(_cfg(sequence_model="TCN"), 1, T, 24e9, 96)[1] == 0
    from fsnplus_b200 import _lib
    bs, tw = C.c_int32(), C.c_int32()
    for bad in (-32, 33, 1):
        assert built_lib.fsn_plan_forward(C.byref(_cfg()), 1, T, 24e9, bad, C.byref(bs), C.byref(tw), None) == -1
    with pytest.raises(_lib.FsnError):
        _lib.plan_forward(_cfg(), 0, T, 24e9)


@pytest.mark.parametrize("value", ["0", "33", "-64", "abc", "64x", "100"])
def test_sb_window_knob_is_validated_at_create(built_lib, monkeypatch, value):
    monkeypatch.setenv("FSN_SB_WINDOW", value)
    h = C.c_void_p()
    assert built_lib.fsn_model_create(C.byref(_cfg()), C.byref(h)) == -1
    assert b"FSN_SB_WINDOW" in built_lib.fsn_last_error()


def test_sb_window_knob_accepts_multiples_of_32(built_lib, monkeypatch):
    monkeypatch.setenv("FSN_SB_WINDOW", "2048")
    h = C.c_void_p()
    rc = built_lib.fsn_model_create(C.byref(_cfg()), C.byref(h))
    assert rc in (0, -2)                                        # -2: no CUDA device on this machine
    if rc == 0:
        built_lib.fsn_model_destroy(h)


def test_cut_by_total_seconds():
    from fsnplus_b200.tools import inference as T
    lengths = [100, 100, 100, 100, 100]
    assert T.bucket_by_length(lengths, 4) == [[0, 1, 2, 3], [4]]
    assert T.bucket_by_length(lengths, 4, max_samples=250) == [[0, 1], [2, 3], [4]]
    assert T.batch_by_sorted_length([50, 400, 30, 60, 20], 8, max_samples=100) == [[4, 2, 0], [3], [1]]
    assert T.batch_by_sorted_length([50, 400, 30, 60, 20], 2) == [[4, 2], [0, 3], [1]]


def _write_dir(tmp_path, lens):
    from scipy.io import wavfile
    from fsnplus_b200.tools import inference as T
    rng = np.random.default_rng(5)
    noisy = tmp_path / "noisy"
    noisy.mkdir()
    for i, n in enumerate(lens):
        wavfile.write(noisy / f"f{i}.wav", 16000, (rng.standard_normal(n) * 0.05).astype(np.float32))
    cfg = T.load_toml(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inference_reference.toml"))
    cfg["dataset"]["args"]["dataset_dir_list"] = [str(noisy)]
    return cfg


def _local_mask(mag, real=None, imag=None, frames=None):
    import torch
    m = torch.stack([torch.tanh(3.0 * mag[:, 0]) * 4.0, torch.sin(7.0 * mag[:, 0]) * 2.0], 1)
    if frames is not None:
        for b, n in enumerate(frames):
            m[b, :, :, int(n):] = 0.0
    return m


@pytest.mark.parametrize("ragged", [False, True])
def test_max_batch_seconds_writes_the_same_files(tmp_path, ragged):
    from fsnplus_b200.tools import inference as T
    lens = [8000, 8000, 8000, 8000, 30000, 4000, 8000]
    cfg = _write_dir(tmp_path, lens)
    quiet = lambda *a: None
    # 1.2 s = 19200 samples: at most two 8000-sample clips, so --batch_size 2 without the flag makes the same batches here (a batched
    # iSTFT of equal-length clips may round differently from a lone one, so the reference run must batch alike)
    T.run(cfg, tmp_path / "x.tar", tmp_path / "plain", batch_size=2, device="cpu", log=quiet, model_and_epoch=(_local_mask, 1), ragged=ragged)
    logs = []
    T.run(cfg, tmp_path / "x.tar", tmp_path / "cut", batch_size=8, device="cpu", log=logs.append, model_and_epoch=(_local_mask, 1),
          ragged=ragged, max_batch_seconds=1.2)
    a, b = tmp_path / "plain" / "enhanced_0001", tmp_path / "cut" / "enhanced_0001"
    for i in range(len(lens)):
        assert (a / f"f{i}.wav").read_bytes() == (b / f"f{i}.wav").read_bytes(), i
    sizes = [int(line.split(": ")[1].split(" x ")[0]) for line in logs if " done" in line]
    assert max(sizes) == 2 and sum(sizes) == len(lens)


class _Replica:
    """A CPU stand-in replica with the model's planning and release hooks: clips longer than 60 frames plan windowed, and a forward
    "holds" a workspace (24 units when windowed, 5 otherwise) until release_workspace()."""

    def __init__(self, rid, events, held):
        self.rid, self.events, self.held = rid, events, held

    def plan(self, B, T):
        return (B, 64 if T > 60 else 0, 0)

    def release_workspace(self):
        self.held[self.rid] = 0
        self.events.append(("release", self.rid))

    def __call__(self, mag, real=None, imag=None, frames=None):
        windowed = self.plan(mag.shape[0], mag.shape[-1])[1] > 0
        others = sum(v for r, v in self.held.items() if r != self.rid)
        self.held[self.rid] = max(self.held.get(self.rid, 0), 24 if windowed else 5)
        self.events.append(("call", self.rid, mag.shape[-1], others))
        return _local_mask(mag, real, imag, frames)


def test_windowed_batches_run_alone_on_one_replica(tmp_path):
    """Four replicas, two long files among short ones: each windowed batch starts only after every earlier batch finished and every
    replica released its workspaces, runs on the first replica, and that replica releases its workspaces before the next batch starts;
    the other batches keep up to four in flight on all replicas."""
    from fsnplus_b200.tools import inference as T
    lens = [4000, 4000, 20000, 6000, 6000, 21000, 9000, 9000]
    cfg = _write_dir(tmp_path, lens)
    events, held = [], {}
    reps = [_Replica(r, events, held) for r in range(4)]
    T.run(cfg, tmp_path / "x.tar", tmp_path / "o", batch_size=1, device="cpu", log=lambda s: events.append(("log", s)),
          model_and_epoch=(reps[0], 1), streams=4, replicas=reps[1:])
    calls = [i for i, e in enumerate(events) if e[0] == "call"]
    long_calls = [i for i in calls if events[i][2] > 60]
    assert len(long_calls) == 2
    done = lambda j: sum(1 for e in events[:j] if e[0] == "log" and " done" in e[1])
    for i in long_calls:
        assert events[i][1] == 0 and events[i][3] == 0                 # replica 0; no other replica holds a workspace
        assert sum(1 for j in calls if j < i) == done(i)                 # everything in flight was finished first
        nxt = next((j for j in calls if j > i), len(events))
        assert ("release", 0) in events[i:nxt] and done(nxt) == done(i) + 1
    assert {events[i][1] for i in calls if i not in long_calls} == {0, 1, 2, 3}
    assert max(sum(1 for j in calls if j < k) - done(k) for k in range(len(events))) > 1   # short batches overlap
    a = sorted(p.name for p in (tmp_path / "o" / "enhanced_0001").iterdir())
    assert a == [f"f{i}.wav" for i in range(len(lens))]


def test_stand_in_without_replicas_runs_one_batch_at_a_time(tmp_path):
    from fsnplus_b200.tools import inference as T
    cfg = _write_dir(tmp_path, [4000, 6000, 9000])
    logs = []
    T.run(cfg, tmp_path / "x.tar", tmp_path / "o", batch_size=1, device="cpu", log=logs.append, model_and_epoch=(_local_mask, 1), streams=4)
    assert any("1 stream(s)" in line for line in logs)


def test_length_limits_are_checked(built_lib):
    """T + look_ahead <= 65535 x 256 (the TCN convolution grid), num_freqs x (T + look_ahead) < 2^31 (a clip's plane index), and the
    planner keeps 3 x Bs x (T + look_ahead) + 128 below 2^31 (the full-band TCN's rows)."""
    from fsnplus_b200 import _lib
    big = _cfg()                                                    # num_freqs 257: the plane limit binds first
    _plan(big, 1, 2147483647 // 257 - 2, 1e18)
    with pytest.raises(_lib.FsnError, match="plane index"):
        _plan(big, 1, 2147483647 // 257 - 1, 1e18)
    small = _cfg(num_freqs=33, sb_num_neighbors=3, sb_model_hidden_size=64)   # the grid limit binds first
    _plan(small, 1, 65535 * 256 - 2, 1e18)
    with pytest.raises(_lib.FsnError, match="65535 x 256"):
        _plan(small, 1, 65535 * 256 - 1, 1e18)
    for T in (10**6, 3 * 10**6):
        bs, tw, n = _plan(small, 1000, T, 1e18)
        assert 3 * bs * (T + 2) + 128 <= 2**31 - 1 and bs < 1000
