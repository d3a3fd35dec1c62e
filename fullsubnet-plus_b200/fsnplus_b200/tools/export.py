"""Export a reference checkpoint to one model file that a C or C++ program loads with ``fsn_model_load`` (include/fsnplus_b200.h).

    python -m fsnplus_b200.tools.export -C config/inference.toml -M ckpt.tar -O model.fsn [--trust_checkpoint]

The model is built from ``[model]`` of the TOML and ``ckpt["model"]`` is loaded strictly, exactly as ``fsnplus_b200.tools.inference``
does (the checkpoint is read with ``weights_only=True`` unless ``--trust_checkpoint``).  Runs on the host: no GPU is needed.
"""
import argparse
import os

from .inference import build_model, load_toml


def main(argv=None):
    parser = argparse.ArgumentParser("Export")
    parser.add_argument("-C", "--configuration", type=str, required=True, help="Config file (the inference TOML).")
    parser.add_argument("-M", "--model_checkpoint_path", type=str, required=True, help="The path of the model's checkpoint.")
    parser.add_argument("-O", "--output", type=str, required=True, help="The model file to write.")
    parser.add_argument("--trust_checkpoint", action="store_true", help="unpickle arbitrary objects from the checkpoint (default: tensors only)")
    args = parser.parse_args(argv)
    configuration = load_toml(args.configuration)
    model, epoch = build_model(configuration["model"], args.model_checkpoint_path, device="cpu", trust_checkpoint=args.trust_checkpoint)
    model.save_model_file(args.output)
    print(f"wrote {args.output}: {os.path.getsize(args.output)} bytes, {len(model.state_dict())} parameters (epoch {epoch})")


if __name__ == "__main__":
    main()
