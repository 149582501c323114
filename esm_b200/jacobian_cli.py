"""`python -m esm_b200.jacobian_cli MODEL seqs.fasta out_dir [--max-tokens N] [--precision fp16|fp32x3] [--cpu-offload]
[--save-jacobian]`: the categorical Jacobian contact map (esm_b200.jacobian) of every protein in a FASTA file.

Writes one `<label>.pt` per record holding {"label", "contacts" [L, L] fp32} and, with --save-jacobian, "jacobian"
[L, 20, L, 20] fp32 (1,600 L^2 bytes), on the host. MODEL is loaded as extract_cli loads it (an ESM-2, ESM-1b or
ESM-1v name or a local .pt file), and a random-init model is refused. A record of fewer than 2 residues is reported
and skipped.
"""
from __future__ import annotations

import argparse
import pathlib
import sys

import torch

from . import jacobian, pretrained
from .data import FastaBatchedDataset
from .variants import DEFAULT_MAX_TOKENS


def create_parser():
    p = argparse.ArgumentParser(description="Categorical Jacobian contact maps of the proteins in a FASTA file")
    p.add_argument("model_location", type=str,
                   help="ESM-2, ESM-1b or ESM-1v model name (esm2_t33_650M_UR50D, esm1b_t33_650M_UR50S, "
                        "esm1v_t33_650M_UR90S_1, ...) or a local .pt file")
    p.add_argument("fasta_file", type=pathlib.Path)
    p.add_argument("output_dir", type=pathlib.Path)
    p.add_argument("--max-tokens", type=int, default=DEFAULT_MAX_TOKENS,
                   help="tokens per stack call (substitution copies per chunk times L + 2); the results do not "
                        "depend on it")
    p.add_argument("--precision", choices=["fp16", "fp32x3"], default="fp16",
                   help="fp16: fp16 MMA operands (default); fp32x3: hi+lo operand pairs, fp32-grade logits (~3x slower)")
    p.add_argument("--cpu-offload", action="store_true",
                   help="keep the transformer layers' weights in pinned host memory and stream them to the GPU layer "
                        "by layer (ESM-2 15B on one GPU); same outputs")
    p.add_argument("--save-jacobian", action="store_true",
                   help="also write the Jacobian [L, 20, L, 20] fp32 (1,600 L^2 bytes per protein)")
    return p


def run(args) -> int:
    """Returns the number of files written."""
    model, alphabet = pretrained.load_model_and_alphabet(args.model_location)
    if getattr(model, "random_init", False):
        raise RuntimeError("refusing to write contacts of a random-init model: give model_location a checkpoint")
    dev = torch.device("cuda", torch.cuda.current_device())
    model = model.eval()
    if args.precision != "fp16":
        model.set_precision(args.precision)
    model = model.cpu_offload(dev) if args.cpu_offload else model.to(dev)
    dataset = FastaBatchedDataset.from_file(args.fasta_file)
    to_tokens = alphabet.get_batch_converter()
    args.output_dir.mkdir(parents=True, exist_ok=True)
    written = 0
    for label, seq in zip(dataset.sequence_labels, dataset.sequence_strs):
        _, _, tokens = to_tokens([(label, seq)])
        L = tokens.shape[1] - 2
        if L < 2:
            print(f"skipping {label!r}: {L} residue(s), the categorical Jacobian needs at least 2", file=sys.stderr)
            continue
        out = jacobian.categorical_jacobian(model, tokens, max_tokens=args.max_tokens,
                                            return_jacobian=args.save_jacobian)
        result = {"label": label, "contacts": out["contacts"].cpu()}
        if args.save_jacobian:
            result["jacobian"] = out["jacobian"].cpu()
        path = args.output_dir / f"{label}.pt"
        path.parent.mkdir(parents=True, exist_ok=True)  # labels may contain '/', as in extract_cli
        torch.save(result, path)
        written += 1
    return written


def main():
    run(create_parser().parse_args())


if __name__ == "__main__":
    main()
