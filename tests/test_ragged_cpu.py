"""CPU: host logic of ragged batches -- enhance_ragged (per-clip STFT, scatter into one zero-padded batch, one model call with
``frames``, per-clip iSTFT) and the command line's ``--ragged`` path (length-sorted batches, rank sharding, same files as the
default path).  The model is a frame-local stand-in, so every clip's result must equal its own enhance_batch exactly."""
import os

import numpy as np
import pytest
import torch


def _local_mask(mag, real=None, imag=None, frames=None):
    """A frame-local compressed cIRM: a pointwise function of mag, zero past each clip's end when ``frames`` is given (as the
    library's ragged forward does)."""
    m = torch.stack([torch.tanh(3.0 * mag[:, 0]) * 4.0, torch.sin(7.0 * mag[:, 0]) * 2.0], 1)
    if frames is not None:
        for b, n in enumerate(frames):
            m[b, :, :, int(n):] = 0.0
    return m


def _clips(lengths, seed=0):
    from fsnplus_b200.synth import synth_clips
    return [synth_clips(1, num_samples=n, seed=seed + i)[0] for i, n in enumerate(lengths)]


@pytest.mark.parametrize("complex_inputs", [True, False])
def test_enhance_ragged_equals_per_clip(complex_inputs):
    """Lengths that share a frame count but not a sample count, equal lengths (one STFT group), and a clip of a few frames."""
    from fsnplus_b200 import inference as H
    lengths = [16000, 5000, 16000, 16100, 300, 16255, 9999]
    clips = _clips(lengths)
    model = _local_mask if complex_inputs else (lambda mag, frames=None: _local_mask(mag, frames=frames))
    got = H.enhance_ragged(model, clips, 512, 256, 512, complex_inputs=complex_inputs)
    assert len(got) == len(clips)
    for c, y in zip(clips, got):
        want = H.enhance_batch(model, c[None], 512, 256, 512, complex_inputs=complex_inputs)[0]
        assert y.shape == c.shape and torch.equal(y, want)
    assert H.enhance_ragged(model, [], 512, 256, 512) == []


def test_enhance_ragged_passes_own_frame_counts():
    """The model sees one [B, 1, F, T_max] batch, zero past every clip's centred-STFT frame count 1 + L // hop, and those counts."""
    from fsnplus_b200 import inference as H
    lengths = [4000, 12000, 700]
    seen = {}

    def spy(mag, real, imag, frames=None):
        seen.update(mag=mag.clone(), frames=list(frames))
        return _local_mask(mag, frames=frames)

    H.enhance_ragged(spy, _clips(lengths), 512, 256, 512)
    want = [1 + n // 256 for n in lengths]
    assert seen["frames"] == want and tuple(seen["mag"].shape) == (3, 1, 257, max(want))
    for b, n in enumerate(want):
        assert (seen["mag"][b, :, :, n:] == 0).all() and (seen["mag"][b, :, :, :n] != 0).any()


def test_batch_by_sorted_length():
    from fsnplus_b200.tools import inference as T
    assert T.batch_by_sorted_length([30, 10, 20, 10, 50, 40, 20], 3) == [[1, 3, 2], [6, 0, 5], [4]]
    assert T.batch_by_sorted_length([], 4) == []


def test_run_ragged_writes_the_same_files(tmp_path, monkeypatch):
    """run(ragged=True) on a directory of mixed lengths writes byte-identical files to the default exact-length path, also when
    the length-sorted batches are sharded over two ranks.  The default path runs with batch_size=1 here: enhance_ragged makes one
    iSTFT per clip, and a batched iSTFT of equal-length clips may round differently in the last bit."""
    from scipy.io import wavfile
    from fsnplus_b200.tools import inference as T
    rng = np.random.default_rng(5)
    noisy = tmp_path / "noisy"
    noisy.mkdir()
    lens = [4096, 9000, 6000, 4096, 12001, 700, 6000, 3333]
    for i, n in enumerate(lens):
        wavfile.write(noisy / f"f{i}.wav", 16000, (rng.standard_normal(n) * 0.05).astype(np.float32))
    cfg = T.load_toml(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "inference_reference.toml"))
    cfg["dataset"]["args"]["dataset_dir_list"] = [str(noisy)]
    quiet = lambda *a: None

    T.run(cfg, tmp_path / "unused.tar", tmp_path / "plain", batch_size=1, device="cpu", log=quiet, model_and_epoch=(_local_mask, 3))
    seen = {}
    for rank in (0, 1):
        monkeypatch.setenv("RANK", str(rank)); monkeypatch.setenv("WORLD_SIZE", "2"); monkeypatch.setenv("LOCAL_RANK", str(rank))
        seen[rank] = T.run(cfg, tmp_path / "unused.tar", tmp_path / "ragged", batch_size=3, device="cpu", log=quiet,
                           model_and_epoch=(_local_mask, 3), ragged=True)
    # sorted by length: [5 f700, 7 f3333, 0 f4096] [3 f4096, 2 f6000, 6 f6000] [1 f9000, 4 f12001]; rank 0 takes batches 0 and 2
    assert sorted(seen[0]) == ["f0", "f1", "f4", "f5", "f7"] and sorted(seen[1]) == ["f2", "f3", "f6"]
    a, b = tmp_path / "plain" / "enhanced_0003", tmp_path / "ragged" / "enhanced_0003"
    assert sorted(p.name for p in b.iterdir()) == sorted(p.name for p in a.iterdir()) == [f"f{i}.wav" for i in range(len(lens))]
    for i in range(len(lens)):
        assert (a / f"f{i}.wav").read_bytes() == (b / f"f{i}.wav").read_bytes(), i


def test_frames_argument_checks():
    """frames is converted to int32 per sample; a wrong length, a float or CUDA tensor, and pipelined=True are refused before
    any device work."""
    from fsnplus_b200.model import FullSubNet_Plus
    arr = FullSubNet_Plus._frames_arg(torch.tensor([3, 5], dtype=torch.int64), 2)
    assert list(arr) == [3, 5]
    assert list(FullSubNet_Plus._frames_arg((7, 1, 2), 3)) == [7, 1, 2]
    with pytest.raises(ValueError):
        FullSubNet_Plus._frames_arg([3], 2)
    with pytest.raises(ValueError):
        FullSubNet_Plus._frames_arg(torch.tensor([3.0, 5.0]), 2)
    m = FullSubNet_Plus(num_freqs=33, look_ahead=2, sequence_model="LSTM", fb_num_neighbors=0, sb_num_neighbors=3,
                        fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=32,
                        sb_model_hidden_size=32).eval()
    x = torch.zeros(2, 1, 33, 8)
    with pytest.raises(ValueError):
        m.enhance_spectrum(x, x, x, pipelined=True, frames=[8, 4])
