"""Score a folder of enhanced speech against its clean references on the GPU, with the reference's command line and output.

    python -m fsnplus_b200.tools.calculate_metrics -R clean_dir -E enhanced_dir -M SI_SDR,STOI -S DNS_1 -D out/

Same flags, pairing and printed lines as the reference's ``speech_enhance/tools/calculate_metrics.py``: ``-R`` / ``-E`` are
directories (sorted recursive WAV listings) or files of one path per line (scp); the lists are aligned by basename, or by the
DNS Challenge renaming rules with ``-S DNS_1`` / ``DNS_2``; the reference is read mono and the estimate's first channel is used, the
reference truncated to the estimate's length.  Printed: ``=== E === R ===``, then per metric ``M: [(name, value), ...]`` and
``M: mean``; ``-D`` writes ``<D><M>.txt`` ranked by value, descending.  ``--limit`` / ``--offset`` are accepted and ignored, as there.

What differs, by design: SI_SDR and STOI are computed by this package's CUDA kernels (fsnplus_b200.metrics, DESIGN.md §3.20), in
batches of clips sorted by length; PESQ, MOSNET and mir_eval's SDR are not available and are refused before any file is read; a file
at another sample rate is resampled with scipy's resample_poly, not librosa's resampler; a clip that leaves no frame after STOI's
silent-frame removal scores 1e-5 instead of raising; an estimate longer than its reference is an error naming the pair.
"""
import argparse
import os
from pathlib import Path

import numpy as np

from .inference import batch_by_sorted_length, find_files, read_wav, wav_length

SUPPORTED = ("SI_SDR", "STOI")
NOT_AVAILABLE = ("WB_PESQ", "NB_PESQ", "MOSNET", "SDR")


def check_metrics(names):
    """Refuse any metric this package does not compute, before any file is read."""
    for m in names:
        if m not in SUPPORTED:
            what = "is not available here" if m in NOT_AVAILABLE else "is not a metric"
            raise NotImplementedError(f"metric {m!r} {what}; supported: {', '.join(SUPPORTED)}")


def basename(path):
    return os.path.splitext(os.path.basename(str(path)))[0]


def load_list(path):
    """A directory's sorted recursive WAV listing, or the paths of an scp file (one per line, made absolute)."""
    p = Path(path).expanduser().absolute()
    if p.is_dir():
        return [str(f) for f in find_files([p])]
    with open(p) as f:
        return [os.path.abspath(os.path.expanduser(line.rstrip("\n"))) for line in f if line.strip()]


DATASET_KEYS = {                                   # the clean basename an estimate's basename names (calculate_metrics.py:81-97)
    "dns_1": lambda est: "clean_" + "_".join(est.split("_")[-2:]),
    "dns_2": lambda est: f"synthetic_clean_fileid_{est.split('_')[-1]}",
}


def align(refs, ests, specific_dataset=""):
    """(refs, ests) paired row by row: by equal basenames, or by a dataset's renaming rule (each reference must match exactly one
    estimate)."""
    sd = specific_dataset.lower()
    if not sd:
        if len(refs) != len(ests):
            raise ValueError(f"{len(refs)} references and {len(ests)} estimates")
        for z, (r, e) in enumerate(zip(refs, ests), start=1):
            if basename(r) != basename(e):
                raise ValueError(f"the lists differ in file name at row {z}:\n\t{r}\n\t{e}")
        return list(refs), list(ests)
    if sd not in DATASET_KEYS:
        raise NotImplementedError(f"Not supported specific dataset {specific_dataset}.")
    by_key = {}
    for e in ests:
        by_key.setdefault(DATASET_KEYS[sd](basename(e)), []).append(e)
    paired = []
    for r in refs:
        found = by_key.get(basename(r), [])
        if len(found) != 1:
            raise ValueError(f"{specific_dataset}: reference {r} matches {len(found)} estimates {found[:3]}, not one")
        paired.append(found[0])
    return list(refs), paired


def load_pair(ref_path, est_path, sr, log=print):
    """(name, reference, estimate): the reference mono, the estimate's first channel, the reference cut to the estimate's length."""
    ref = read_wav(ref_path, sr)
    est = read_wav(est_path, sr, first_channel=True)
    if est.size > ref.size:
        raise ValueError(f"estimate {est_path} has {est.size} samples, more than its reference {ref_path} ({ref.size})")
    if ref.size != est.size:
        log(f"[Warning] ref {ref.size} and est {est.size} are not in the same length")
    return basename(ref_path), ref[:est.size], est


def score_batch(metric, refs, ests, sr, device):
    """One batch's scores (lists of equal-length float32 arrays) on the GPU, as Python floats."""
    import torch
    from .. import metrics
    r = [torch.from_numpy(x).to(device) for x in refs]
    e = [torch.from_numpy(x).to(device) for x in ests]
    out = metrics.si_sdr(r, e) if metric == "SI_SDR" else metrics.stoi(r, e, sr=sr)
    return out.cpu().tolist()


def write_ranked(path, results):
    """``name: value`` lines, highest value first (ties keep their order), to ``path``."""
    ranked = sorted(results, key=lambda nv: nv[1], reverse=True)
    d = os.path.dirname(path)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(path, "w+") as f:
        for name, value in ranked:
            f.write(name + ": " + str(value) + "\n")


def run(reference, estimated, metric_types, sr=16000, export_dir="", specific_dataset="", batch_size=256, max_batch_seconds=600.0,
        device="cuda", log=print):
    """Score every pair; returns {metric: [(name, value), ...]} in pair order and prints / exports as the reference does."""
    names = metric_types.split(",")
    check_metrics(names)
    refs, ests = align(load_list(reference), load_list(estimated), specific_dataset)
    lengths = [wav_length(e, sr) for e in ests]
    results = {m: [None] * len(refs) for m in names}
    cap = max(1, int(max_batch_seconds * sr))
    log(f"=== {estimated} === {reference} ===")
    for idx in batch_by_sorted_length(lengths, batch_size, max_samples=cap):
        pairs = [load_pair(refs[i], ests[i], sr, log) for i in idx]
        for m in dict.fromkeys(names):
            scores = score_batch(m, [p[1] for p in pairs], [p[2] for p in pairs], sr, device)
            for i, p, v in zip(idx, pairs, scores):
                results[m][i] = (p[0], float(v))
    for m in names:
        log(f"{m}: {results[m]}")
        log(f"{m}: {np.mean([v for _, v in results[m]])}")
        if export_dir:
            write_ranked(export_dir + str(m) + ".txt", results[m])
    return results


def main(argv=None):
    parser = argparse.ArgumentParser(description="Mean objective scores of estimated speech against references (SI_SDR, STOI)",
                                     epilog="python -m fsnplus_b200.tools.calculate_metrics -E est_dir -R ref_dir -M SI_SDR,STOI")
    parser.add_argument("-R", "--reference", required=True, type=str, help="reference directory or scp file")
    parser.add_argument("-E", "--estimated", required=True, type=str, help="estimate directory or scp file")
    parser.add_argument("-M", "--metric_types", required=True, type=str, help="comma-separated metrics: SI_SDR, STOI")
    parser.add_argument("--sr", type=int, default=16000, help="sample rate the files are read at")
    parser.add_argument("-D", "--export_dir", type=str, default="", help="prefix of the <prefix><metric>.txt rankings")
    parser.add_argument("--limit", type=int, default=None, help="accepted and ignored, as in the reference")
    parser.add_argument("--offset", type=int, default=0, help="accepted and ignored, as in the reference")
    parser.add_argument("-S", "--specific_dataset", type=str, default="", help="DNS_1 or DNS_2 name alignment (any case)")
    parser.add_argument("--batch_size", type=int, default=256, help="clips per device call (additive)")
    parser.add_argument("--max_batch_seconds", type=float, default=600.0, help="most seconds of audio per device call (additive)")
    parser.add_argument("--device", type=str, default="cuda", help="CUDA device (additive)")
    args = parser.parse_args(argv)
    run(args.reference, args.estimated, args.metric_types, sr=args.sr, export_dir=args.export_dir, specific_dataset=args.specific_dataset,
        batch_size=args.batch_size, max_batch_seconds=args.max_batch_seconds, device=args.device)


if __name__ == "__main__":
    main()
