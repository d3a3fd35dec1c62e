"""CPU: the forward plan of the sub-band TCN in bin chunks (fsn_plan_forward_bins, DESIGN.md §3.8), the FSN_SB_CHUNK knob, and the
command line's lone chunked batches.  The plan is a host function of the configuration, so no GPU is needed."""
import ctypes as C

import pytest

from oracle import fsn_oracle as O

from test_long_clip_cpu import _Replica, _frames, _local_mask, _write_dir

F = 257
ROW_LIMIT = 2**31 - 1 - 128


def _cfg(kind="plus", **over):
    from fsnplus_b200.model import FullSubNet_Plus, Model
    c = O.default_plus_config() if kind == "plus" else O.default_fsn_config()
    c.update(over)
    return (FullSubNet_Plus if kind == "plus" else Model)(**c)._cfg


def _tcn():
    return _cfg(sequence_model="TCN")


def _bins(cfg, B, T, cap, force_window=0, force_bins=0):
    from fsnplus_b200 import _lib
    return _lib.plan_forward_bins(cfg, B, T, cap, force_window, force_bins)


def _exact(cfg, bs, T, fc):
    """Exact workspace of (bs, fc): forced chunks under an unlimited cap keep the whole batch."""
    got = _bins(cfg, bs, T, 1e18, 0, fc if fc else F)
    assert got[:3] == (bs, 0, fc)
    return got[3]


@pytest.mark.parametrize("B,seconds", [(1, 3), (64, 3), (256, 3), (1, 60), (1, 480)])
def test_tcn_plans_that_fit_stay_unchunked(built_lib, B, seconds):
    from fsnplus_b200 import _lib
    cfg, T = _tcn(), _frames(seconds)
    bs, tw, fc, n = _bins(cfg, B, T, 24e9)
    assert fc == 0 and (bs, tw, n) == _lib.plan_forward(cfg, B, T, 24e9)


@pytest.mark.parametrize("kind", ["plus", "fsn"])
@pytest.mark.parametrize("B,seconds,cap,force", [(1, 3, 24e9, 0), (2, 3, 24e9, 0), (64, 3, 24e9, 0), (256, 3, 24e9, 0), (1, 60, 24e9, 0),
                                                 (1, 180, 24e9, 0), (1, 240, 24e9, 0), (1, 600, 24e9, 0), (1, 3600, 24e9, 0),
                                                 (1, 7200, 24e9, 0), (4, 1800, 24e9, 0), (64, 3600, 24e9, 0), (1, 90, 2e9, 0),
                                                 (3, 60, 2e9, 0), (3, 60, 0.4e9, 0), (2, 10, 24e9, 96), (4, 600, 1e8, 0)])
def test_recurrent_plans_are_unchanged(built_lib, kind, B, seconds, cap, force):
    """Every case of the LSTM planner's tests, forced windows included, and GRU: never chunked, the same plan and bytes."""
    from fsnplus_b200 import _lib
    T = _frames(seconds)
    for cfg in ((_cfg(kind), _cfg(kind, sequence_model="GRU")) if kind == "plus" else (_cfg(kind),)):
        bs, tw, fc, n = _bins(cfg, B, T, cap, force, 7)             # FSN_SB_CHUNK is ignored by LSTM / GRU models
        assert fc == 0 and (bs, tw, n) == _lib.plan_forward(cfg, B, T, cap, force)


def _runs(B, bs, fc):
    return -(-B // bs) * -(-F // (fc or F))


@pytest.mark.parametrize("B,seconds,cap", [(1, 600, 24e9), (1, 1800, 24e9), (1, 3600, 24e9), (1, 7200, 24e9), (4, 1800, 24e9),
                                           (1, 90, 2e9), (3, 60, 0.4e9)])
def test_chunked_plan_honours_cap_and_is_minimal(built_lib, B, seconds, cap):
    cfg, T = _tcn(), _frames(seconds)
    bs, tw, fc, n = _bins(cfg, B, T, cap)
    print(f"\n[{B} x {seconds} s, cap {cap / 1e9:g} GB] Bs={bs} Fc={fc} chunks={-(-F // fc)} {n / 1e9:.2f} GB")
    assert tw == 0 and 0 < fc < F and n <= cap and bs * fc * (T + 2) <= ROW_LIMIT
    assert n == _exact(cfg, bs, T, fc)
    nch = -(-F // fc)
    assert fc == -(-F // nch)                                       # evened out
    if nch > 1:                                                     # one chunk fewer, evened out, does not fit
        wider = -(-F // (nch - 1))
        assert _exact(cfg, bs, T, wider if wider < F else 0) > cap
    # brute force over every equal split and every chunk width: nothing fits with fewer chunk runs
    best = _runs(B, bs, fc)
    for k in range(1, B + 1):
        s = -(-B // k)
        for w in range(1, F + 1):
            if _runs(B, s, w) < best and s * w * (T + 2) <= ROW_LIMIT:
                assert _exact(cfg, s, T, w if w < F else 0) > cap, (s, w)


def test_plan_table_of_the_issue(built_lib):
    """The default config's chunk widths for one clip of 1 h / 2 h and for 4 x 30 min at 24 GB."""
    cfg = _tcn()
    assert _bins(cfg, 1, _frames(3600), 24e9)[:3] == (1, 0, 26)
    assert _bins(cfg, 1, _frames(7200), 24e9)[:3] == (1, 0, 9)
    assert _bins(cfg, 4, _frames(1800), 24e9)[:3] == (1, 0, 65)


def test_nothing_fits_runs_one_clip_in_one_bin_chunks(built_lib):
    bs, tw, fc, n = _bins(_tcn(), 4, _frames(600), 1e8)
    assert (bs, tw, fc) == (1, 0, 1) and n > 1e8


def test_force_bins_is_honoured(built_lib):
    cfg, T = _tcn(), _frames(20)
    for fb in (1, 7, 16, 64, 100, 256):
        bs, tw, fc, n = _bins(cfg, 3, T, 24e9, 0, fb)
        assert (bs, tw, fc) == (3, 0, fb) and n == _exact(cfg, 3, T, fb)
    assert _bins(cfg, 3, T, 24e9, 0, 257)[2] == 0 and _bins(cfg, 3, T, 24e9, 0, 300)[2] == 0
    bs, _, fc, n = _bins(cfg, 4, _frames(60), 2e9, 0, 64)           # the largest equal split that fits with 64 bins
    print(f"\n[4 x 60 s, cap 2 GB, 64 bins] Bs={bs} {n / 1e9:.2f} GB")
    assert fc == 64 and n <= 2e9 and 1 < bs < 4 and _exact(cfg, -(-4 // (-(-4 // bs) - 1)), _frames(60), 64) > 2e9
    out = [C.c_int32() for _ in range(3)]
    assert built_lib.fsn_plan_forward_bins(C.byref(cfg), 1, T, 24e9, 0, -1, *(C.byref(o) for o in out), None) == -1


@pytest.mark.parametrize("value", ["0", "-3", "abc", "8x"])
def test_sb_chunk_knob_is_validated_at_create(built_lib, monkeypatch, value):
    monkeypatch.setenv("FSN_SB_CHUNK", value)
    h = C.c_void_p()
    assert built_lib.fsn_model_create(C.byref(_tcn()), C.byref(h)) == -1
    assert b"FSN_SB_CHUNK" in built_lib.fsn_last_error()


@pytest.mark.parametrize("value", ["1", "7", "300"])
def test_sb_chunk_knob_accepts_positive_bins(built_lib, monkeypatch, value):
    monkeypatch.setenv("FSN_SB_CHUNK", value)
    h = C.c_void_p()
    rc = built_lib.fsn_model_create(C.byref(_tcn()), C.byref(h))
    assert rc in (0, -2)                                        # -2: no CUDA device on this machine
    if rc == 0:
        bs, tw, fc, n = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int64()
        assert built_lib.fsn_model_plan_bins(h, 2, 100, C.byref(bs), C.byref(tw), C.byref(fc), C.byref(n)) == 0
        assert fc.value == (0 if int(value) >= F else int(value))
        built_lib.fsn_model_destroy(h)


class _ChunkReplica(_Replica):
    """The stand-in replica of the windowed-batch test, planning bin chunks instead of windows (plan_bins) for clips over 60 frames."""

    def plan(self, B, T):
        return (B, 0, 0)

    def plan_bins(self, B, T):
        return (B, 0, 26 if T > 60 else 0, 0)

    def __call__(self, mag, real=None, imag=None, frames=None):
        chunked = self.plan_bins(mag.shape[0], mag.shape[-1])[2] > 0
        others = sum(v for r, v in self.held.items() if r != self.rid)
        self.held[self.rid] = max(self.held.get(self.rid, 0), 24 if chunked else 5)
        self.events.append(("call", self.rid, mag.shape[-1], others))
        return _local_mask(mag, real, imag, frames)


def test_chunked_batches_run_alone_on_one_replica(tmp_path):
    """As for windowed batches: each chunked batch starts after every earlier batch finished and every replica released its
    workspaces, runs on the first replica, and that replica releases its workspaces before the next batch starts."""
    from fsnplus_b200.tools import inference as T
    lens = [4000, 4000, 20000, 6000, 6000, 21000, 9000, 9000]
    cfg = _write_dir(tmp_path, lens)
    events, held = [], {}
    reps = [_ChunkReplica(r, events, held) for r in range(4)]
    T.run(cfg, tmp_path / "x.tar", tmp_path / "o", batch_size=1, device="cpu", log=lambda s: events.append(("log", s)),
          model_and_epoch=(reps[0], 1), streams=4, replicas=reps[1:])
    calls = [i for i, e in enumerate(events) if e[0] == "call"]
    long_calls = [i for i in calls if events[i][2] > 60]
    assert len(long_calls) == 2
    done = lambda j: sum(1 for e in events[:j] if e[0] == "log" and " done" in e[1])
    for i in long_calls:
        assert events[i][1] == 0 and events[i][3] == 0
        assert sum(1 for j in calls if j < i) == done(i)
        nxt = next((j for j in calls if j > i), len(events))
        assert ("release", 0) in events[i:nxt] and done(nxt) == done(i) + 1
    assert {events[i][1] for i in calls if i not in long_calls} == {0, 1, 2, 3}


def test_plan_is_windowed_asks_plan_bins_first():
    from fsnplus_b200.tools import inference as T

    class OnlyPlan:
        def plan(self, B, T):
            return (B, 0, 0)

    class Chunked(OnlyPlan):
        def plan_bins(self, B, T):
            return (B, 0, 9, 0)

    assert not T.plan_is_windowed(OnlyPlan(), 1, 10**6)
    assert T.plan_is_windowed(Chunked(), 1, 10**6)
    assert not T.plan_is_windowed(_local_mask, 1, 10**6)
