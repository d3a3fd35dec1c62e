"""Directory-to-directory enhancement with the reference's command line and TOML.

    python -m fsnplus_b200.tools.inference -C config/inference.toml -M ckpt.tar -I noisy_dir[,dir2] -O out_dir
    torchrun --nproc-per-node 8 -m fsnplus_b200.tools.inference ...          # one process per GPU, files sharded

Same flags, configuration keys, checkpoint format and output convention as the reference's
``speech_enhance/tools/inference.py:22-39`` + ``audio_zen/inferencer/base_inferencer.py:21-160``: the model named by
``[model].path`` / ``[model].args`` is built (reference dotted paths are mapped to this package), ``ckpt["model"]`` is loaded
strictly, every audio file under the dataset directories is enhanced with the ``[inferencer].type`` method and written as
``<out>/enhanced_<epoch:04d>/<name>.wav`` in int16 after the reference's ``0.8 * 32767 * y / max|y|`` scaling
(base_inferencer.py:151-152,160).

What differs, by design: clips are enhanced in BATCHES.  The reference is hard-wired to batch 1
(base_inferencer.py:65-69); here files are grouped by exact sample count (the forward is per-utterance -- offline norm,
time pooling in the attention -- so padding a clip would change its result) and each group runs ``--batch_size`` clips per
launch.  With ``--ragged`` files are instead sorted by sample count and cut into batches of ``--batch_size`` clips of different
lengths, each enhanced by one ragged model call (every clip is masked at its own end, so its result is unchanged).  ``librosa`` / ``soundfile`` are not dependencies: WAV (PCM 8/16/24/32, float32/64) is read with scipy and written
with the standard library; other containers are rejected with a clear error.
"""
import argparse
import os
import time
import wave
from pathlib import Path

import numpy as np
import torch

from .. import inference as H

AUDIO_EXT = (".wav",)
#: librosa.util.find_files also matches these; they are reported instead of silently skipped
UNSUPPORTED_EXT = (".aac", ".au", ".flac", ".m4a", ".mp3", ".ogg")

MODEL_PATHS = {                                                           # config/inference.toml:27-28
    "fullsubnet_plus.model.fullsubnet_plus.FullSubNet_Plus": "FullSubNet_Plus",
    "fsnplus_b200.model.FullSubNet_Plus": "FullSubNet_Plus",
    "fullsubnet.model.fullsubnet.Model": "Model",
    "fsnplus_b200.model.Model": "Model",
}
INFERENCE_TYPES = {"mag_complex_full_band_crm_mask": True,                # fullsubnet_plus/inferencer/inferencer.py:140-165
                   "full_band_crm_mask": False}                           # :116-137


def load_toml(path):
    try:
        import tomllib
        with open(path, "rb") as f:
            return tomllib.load(f)
    except ModuleNotFoundError:                                           # pragma: no cover (python < 3.11)
        import toml
        return toml.load(path)


def find_files(dirs):
    """Sorted recursive listing per directory, like librosa.util.find_files (dataset_inference.py:23-26)."""
    files = []
    for d in dirs:
        d = Path(d).expanduser().absolute()
        if not d.is_dir():
            raise FileNotFoundError(f"dataset directory {d} does not exist")
        found = sorted(p for p in d.rglob("*") if p.is_file() and p.suffix.lower() in AUDIO_EXT + UNSUPPORTED_EXT)
        bad = [p for p in found if p.suffix.lower() in UNSUPPORTED_EXT]
        if bad:
            raise NotImplementedError(f"only WAV input is supported without librosa/soundfile; found {bad[0]} (+{len(bad) - 1} more)")
        files += found
    return files


def read_wav(path, sr):
    """float32 mono in [-1, 1) like librosa.load(path, sr=sr)[0] (dataset_inference.py:36-37): integer PCM is divided by
    its full scale, channels are averaged; a different sample rate is converted with a polyphase resampler."""
    from scipy.io import wavfile
    rate, x = wavfile.read(str(path))
    if x.dtype == np.uint8:
        y = (x.astype(np.float32) - 128.0) / 128.0
    elif np.issubdtype(x.dtype, np.integer):
        y = x.astype(np.float32) / float(2 ** (8 * x.dtype.itemsize - 1))
    else:
        y = x.astype(np.float32)
    if y.ndim == 2:
        y = y.mean(axis=1)
    if rate != sr:
        from math import gcd
        from scipy.signal import resample_poly
        g = gcd(int(rate), int(sr))
        y = resample_poly(y, sr // g, rate // g).astype(np.float32)
    return np.ascontiguousarray(y, dtype=np.float32)


def wav_length(path, sr):
    """Number of samples read_wav(path, sr) will return, from the header only (the data stay on disk: memory-mapped)."""
    from scipy.io import wavfile
    rate, x = wavfile.read(str(path), mmap=True)
    n = int(x.shape[0])
    if rate != sr:
        from math import gcd
        g = gcd(int(rate), int(sr))
        up, down = sr // g, rate // g
        n = -(-n * up // down)                                            # scipy.signal.resample_poly: ceil(n * up / down)
    return n


def to_int16(enhanced):
    """base_inferencer.py:151-152."""
    amp = np.iinfo(np.int16).max
    return np.int16(0.8 * amp * enhanced / np.max(np.abs(enhanced)))


def write_wav_int16(path, pcm, sr):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(int(sr))
        w.writeframes(np.ascontiguousarray(pcm, dtype="<i2").tobytes())


def _cut(idx, lengths, batch_size, max_samples):
    """Runs of at most batch_size indices; with max_samples, a run is also cut before its total length would exceed
    max_samples (a clip longer than that is a run of its own)."""
    if max_samples is None:
        return [idx[i:i + batch_size] for i in range(0, len(idx), batch_size)]
    runs, cur, tot = [], [], 0
    for i in idx:
        n = int(lengths[i])
        if cur and (len(cur) == batch_size or tot + n > max_samples):
            runs.append(cur)
            cur, tot = [], 0
        cur.append(i)
        tot += n
    if cur:
        runs.append(cur)
    return runs


def bucket_by_length(lengths, batch_size, max_samples=None):
    """Indices grouped by identical length, each group cut into runs of at most batch_size (and, with max_samples, at most
    max_samples samples of audio); groups in order of first appearance so the output order stays close to the directory order."""
    groups = {}
    for i, n in enumerate(lengths):
        groups.setdefault(int(n), []).append(i)
    batches = []
    for idx in groups.values():
        batches += _cut(idx, lengths, batch_size, max_samples)
    return batches


def batch_by_sorted_length(lengths, batch_size, max_samples=None):
    """Indices sorted by length (stable: ties keep the directory order), cut into runs of at most batch_size (and, with
    max_samples, at most max_samples samples of audio): neighbouring clips have similar lengths, which keeps the padding of a
    ragged batch small."""
    order = sorted(range(len(lengths)), key=lambda i: int(lengths[i]))
    return _cut(order, lengths, batch_size, max_samples)


def plan_is_windowed(model, batch, frames):
    """True when the model's plain forward of `batch` clips of `frames` STFT frames will run its sub-band stage in time windows or, for
    the sub-band TCN, in bin chunks (model.plan_bins / model.plan, the C ABI's fsn_plan_forward_bins): such a forward takes the model's
    whole workspace cap.  Stand-in models without a plan are never windowed."""
    plan_bins = getattr(model, "plan_bins", None)
    if plan_bins is not None:
        _, tw, fc, _ = plan_bins(batch, frames)
        return tw > 0 or fc > 0
    plan = getattr(model, "plan", None)
    return plan is not None and plan(batch, frames)[1] > 0


def build_model(model_config, checkpoint_path, device, trust_checkpoint=False):
    """base_inferencer.py:97-110 (_load_model).  The checkpoint is read with ``weights_only=True`` (tensors and plain containers
    only: the reference's ``{"model": state_dict, "epoch": int}`` loads); ``trust_checkpoint=True`` opts into full unpickling."""
    from .. import model as M
    path = model_config["path"]
    if path not in MODEL_PATHS:
        raise NotImplementedError(f"[model].path = {path!r} is not one of {sorted(MODEL_PATHS)}")
    net = getattr(M, MODEL_PATHS[path])(**model_config["args"])
    ckpt = torch.load(str(checkpoint_path), map_location="cpu", weights_only=not trust_checkpoint)
    net.load_state_dict(ckpt["model"])
    return net.to(device).eval(), ckpt["epoch"]


def _rank_world():
    return int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))


@torch.no_grad()
def run(config, checkpoint_path, output_dir, batch_size=64, device=None, log=print, model_and_epoch=None, trust_checkpoint=False, streams=4,
        ragged=False, max_batch_seconds=None, replicas=None):
    """Enhance every file of config["dataset"]["args"]["dataset_dir_list"].  Under torchrun each rank takes every
    world-size-th batch (files are independent: no collective).  Returns {name: path} of the files this rank wrote.
    ``model_and_epoch`` (tests of the host logic) replaces the checkpoint load with a ready ``(callable, epoch)``.
    ``ragged=True``: batches of clips of different lengths (length-sorted, ``batch_size`` clips each) through ``enhance_ragged``.
    ``max_batch_seconds``: a batch is also cut before its total audio exceeds that many seconds (a longer clip goes alone).
    A batch whose forward the model plans in time windows or bin chunks (a long clip: it uses the model's whole workspace cap) runs alone on the
    first replica: every batch in flight is finished and every replica's workspaces are released first, and the first replica's
    after it, so only one capped workspace exists at a time.
    ``replicas`` (tests of the host logic, with ``model_and_epoch``): ready models for the replicas after the first."""
    rank, world, local_rank = _rank_world()
    if device is None:
        device = f"cuda:{local_rank}"
    ac = config["acoustics"]
    sr, n_fft, hop, win = ac["sr"], ac["n_fft"], ac["hop_length"], ac["win_length"]
    itype = config["inferencer"]["type"]
    if itype not in INFERENCE_TYPES:
        raise NotImplementedError(f"Not implemented Inferencer type: {itype}")       # base_inferencer.py:135
    files = find_files(config["dataset"]["args"]["dataset_dir_list"])
    ds_sr = config["dataset"]["args"].get("sr", sr)
    model, epoch = model_and_epoch or build_model(config["model"], Path(checkpoint_path).expanduser().absolute(), device, trust_checkpoint)
    on_gpu = torch.device(device).type == "cuda"
    enhanced_dir = Path(output_dir).expanduser().absolute() / f"enhanced_{str(epoch).zfill(4)}"
    enhanced_dir.mkdir(parents=True, exist_ok=True)

    # bucket on the lengths from the WAV headers; a rank decodes only the files of ITS batches, one batch at a time (host memory
    # and start-up time scale with the batch, not with the dataset -- the reference streams one clip at a time)
    lengths = [wav_length(p, ds_sr) for p in files]
    max_samples = None if max_batch_seconds is None else max(1, int(max_batch_seconds * ds_sr))
    batches = (batch_by_sorted_length(lengths, batch_size, max_samples=max_samples) if ragged
               else bucket_by_length(lengths, batch_size, max_samples=max_samples))
    mine = [(bi, idx) for bi, idx in enumerate(batches) if bi % world == rank]
    # Ragged real recordings make many small batches (a lone clip fills a small fraction of the SMs): up to `streams`
    # batches are in flight at once, each on its own CUDA stream and its own model replica (own C handle and workspaces).
    if replicas is not None:
        nstream = max(1, min(streams, len(mine), 1 + len(replicas)))
        models = [model] + list(replicas[:nstream - 1])
    else:
        nstream = max(1, min(streams, len(mine))) if (on_gpu and model_and_epoch is None) else 1
        models = [model] + [build_model(config["model"], Path(checkpoint_path).expanduser().absolute(), device, trust_checkpoint)[0]
                            for _ in range(nstream - 1)]
    cuda_streams = [torch.cuda.Stream(device) for _ in range(nstream)] if on_gpu else [None] * nstream

    def release_all(ms):
        for m in ms:
            if hasattr(m, "release_workspace"):
                m.release_workspace()
    written, audio_s, inflight = {}, 0.0, []
    t_start = time.time()

    def finish(item):
        bi, idx, host, ev, n_samples = item
        if ev is not None:
            ev.synchronize()
        enhanced = host.numpy() if torch.is_tensor(host) else [h.numpy() for h in host]
        log(f"[rank {rank}] batch {bi}: {len(idx)} x {n_samples} samples done")
        for j, i in enumerate(idx):
            y = enhanced[j]
            if (np.abs(y) > 1).any():
                log(f"Warning: enhanced is not in the range [-1, 1], {files[i].stem}")      # base_inferencer.py:148-149
            out = enhanced_dir / f"{files[i].stem}.wav"
            write_wav_int16(out, to_int16(y), sr)
            written[files[i].stem] = out

    for n, (bi, idx) in enumerate(mine):
        alone = plan_is_windowed(models[0], len(idx), max(int(lengths[i]) for i in idx) // hop + 1)   # centred STFT frames
        k = 0 if alone else n % nstream
        while inflight and (alone or len(inflight) >= nstream):
            finish(inflight.pop(0))                                        # the batch that used this stream / replica last
        if alone:
            release_all(models)                                            # the windowed / chunked forward may take the whole cap
        if ragged:
            clips = [torch.from_numpy(read_wav(files[i], ds_sr)) for i in idx]
            audio_s += sum(c.numel() for c in clips) / sr
            desc = f"{min(c.numel() for c in clips)}..{max(c.numel() for c in clips)}"
            if on_gpu:
                with torch.cuda.stream(cuda_streams[k]):
                    enh = H.enhance_ragged(models[k], [c.pin_memory().to(device, non_blocking=True) for c in clips], n_fft, hop, win,
                                           complex_inputs=INFERENCE_TYPES[itype])
                    host = [torch.empty(tuple(e.shape), dtype=e.dtype).pin_memory() for e in enh]
                    for h, e in zip(host, enh):
                        h.copy_(e, non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(cuda_streams[k])
                inflight.append((bi, idx, host, ev, desc))
            else:
                enh = H.enhance_ragged(models[k], clips, n_fft, hop, win, complex_inputs=INFERENCE_TYPES[itype])
                inflight.append((bi, idx, [e.cpu() for e in enh], None, desc))
            if alone:
                finish(inflight.pop(0))
                release_all(models[:1])
            continue
        noisy = torch.from_numpy(np.stack([read_wav(files[i], ds_sr) for i in idx]))
        audio_s += len(idx) * noisy.size(1) / sr
        if on_gpu:
            with torch.cuda.stream(cuda_streams[k]):
                dev_noisy = noisy.pin_memory().to(device, non_blocking=True)
                enh = H.enhance_batch(models[k], dev_noisy, n_fft, hop, win, complex_inputs=INFERENCE_TYPES[itype])
                host = torch.empty(tuple(enh.shape), dtype=enh.dtype).pin_memory()
                host.copy_(enh, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(cuda_streams[k])
            inflight.append((bi, idx, host, ev, noisy.size(1)))
        else:
            inflight.append((bi, idx, H.enhance_batch(models[k], noisy, n_fft, hop, win, complex_inputs=INFERENCE_TYPES[itype]).cpu(), None, noisy.size(1)))
        if alone:
            finish(inflight.pop(0))                                        # nothing starts while the windowed batch holds its workspace
            release_all(models[:1])
    while inflight:
        finish(inflight.pop(0))
    if audio_s > 0:
        log(f"[rank {rank}] {len(written)} files, {audio_s:.1f} s of audio, {nstream} stream(s), overall rtf: {(time.time() - t_start) / audio_s:.3e}")
    return written


def main(argv=None):
    parser = argparse.ArgumentParser("Inference")                          # same flags as the reference tools/inference.py:22-29
    parser.add_argument("-C", "--configuration", type=str, required=True, help="Config file.")
    parser.add_argument("-M", "--model_checkpoint_path", type=str, required=True, help="The path of the model's checkpoint.")
    parser.add_argument("-I", "--dataset_dir_list", help="delimited list input", default=[],
                        type=lambda s: [item.strip() for item in s.split(",")])
    parser.add_argument("-O", "--output_dir", type=str, required=True, help="The path for saving enhanced speeches.")
    parser.add_argument("--batch_size", type=int, default=64, help="clips of equal length per launch (additive)")
    parser.add_argument("--trust_checkpoint", action="store_true", help="unpickle arbitrary objects from the checkpoint (default: tensors only)")
    parser.add_argument("--streams", type=int, default=4, help="batches in flight at once, each on its own CUDA stream and model replica (additive)")
    parser.add_argument("--ragged", action="store_true",
                        help="batch clips of different lengths (sorted by length, --batch_size per batch) in one ragged model call (additive)")
    parser.add_argument("--max_batch_seconds", type=float, default=None,
                        help="also cut a batch before its total audio exceeds this many seconds; a longer clip goes alone (additive)")
    args = parser.parse_args(argv)
    configuration = load_toml(args.configuration)
    if len(args.dataset_dir_list) > 0:
        print(f"use specified dataset_dir_list: {args.dataset_dir_list}, instead of in config")
        configuration["dataset"]["args"]["dataset_dir_list"] = args.dataset_dir_list
    run(configuration, args.model_checkpoint_path, args.output_dir, batch_size=args.batch_size, trust_checkpoint=args.trust_checkpoint, streams=args.streams,
        ragged=args.ragged, max_batch_seconds=args.max_batch_seconds)


if __name__ == "__main__":
    main()
