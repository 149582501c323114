"""`python -m esm_b200.sample_msa_cli MODEL --msa in.a3m [--msa-samples N] [--rows 1-3] [--columns 5-40,52]
[--append-rows K] [--chains C] [--sweeps W] [--block K] [--temperature T] [--seed S] [--no-gaps] [--max-tokens N]
[--precision fp16|fp32x3] --out DIR`: sample alignments from the MSA Transformer by Gibbs sampling
(esm_b200.sampling.msa_gibbs).

The alignment is the first --msa-samples records of the a3m file (default all), insertions removed as read_msa removes
them. --append-rows adds K rows of <mask> below it, which the sampler fills with new family members. Designable
entries: with neither --rows nor --columns, every entry, or only the appended rows when there are any. --rows and
--columns (1-based numbers and inclusive ranges; rows count the input rows first, then the appended ones; columns
count alignment columns, not <cls>) make the entries in those rows and columns designable, each defaulting to all;
appended rows stay designable in full. MODEL is an MSA Transformer name or .pt file, loaded as predict_cli loads it,
and a random-init model is refused. --msa-select max / min reads the whole file and keeps --msa-samples rows picked by
esm_b200.msa_select.greedy_select; it needs --msa-samples.

Writes DIR/sample_{c}.a3m per chain (the input descriptions, then generated_{i} for the appended rows, 0-based) and
DIR/samples.tsv with the columns chain, seed and logp, the summed log q of the chain's last sweep.
"""
from __future__ import annotations

import argparse
import pathlib

import torch

from . import sampling
from .predict_cli import MSA_SELECT, load_model, read_alignment
from .sample_cli import _positive, parse_positions
from .variants import DEFAULT_MAX_TOKENS


def _nonnegative(text: str) -> int:
    v = int(text)
    if v < 0:
        raise argparse.ArgumentTypeError(f"must be >= 0, got {v}")
    return v


def create_parser():
    p = argparse.ArgumentParser(description="Sample alignments from the MSA Transformer (Gibbs sampling)")
    p.add_argument("model_location", type=str,
                   help="MSA Transformer model name (esm_msa1b_t12_100M_UR50S, ...) or a local .pt file")
    p.add_argument("--msa", type=pathlib.Path, required=True, help="a3m alignment to start every chain from")
    p.add_argument("--msa-samples", type=_positive, default=None,
                   help="how many alignment rows to read, from the top (default: all)")
    p.add_argument("--msa-select", choices=MSA_SELECT, default="first",
                   help="which --msa-samples rows to keep: first (default) or max / min, picked from the whole file "
                        "for the largest / smallest mean Hamming distance, as the contact notebook's greedy_select")
    p.add_argument("--rows", type=parse_positions, default=None,
                   help="designable rows, 1-based numbers and inclusive ranges such as 1-3 (default: see above)")
    p.add_argument("--columns", type=parse_positions, default=None,
                   help="designable alignment columns, 1-based numbers and inclusive ranges such as 5-40,52")
    p.add_argument("--append-rows", type=_nonnegative, default=0, help="add this many all-<mask> rows to generate")
    p.add_argument("--chains", type=_positive, default=1, help="independent chains, one a3m file each")
    p.add_argument("--sweeps", type=_positive, default=1, help="passes over the designable entries")
    p.add_argument("--block", type=_positive, default=1, help="entries resampled together per step")
    p.add_argument("--temperature", type=float, default=1.0, help="divides the logits (finite, > 0)")
    p.add_argument("--seed", type=int, default=0, help="random stream key in [0, 2^64)")
    p.add_argument("--no-gaps", dest="gaps", action="store_false",
                   help="draw the 20 amino acids only, never the gap '-'")
    p.add_argument("--max-tokens", type=int, default=DEFAULT_MAX_TOKENS,
                   help="tokens per stack call (chains per chunk times R * C); the samples do not depend on it")
    p.add_argument("--precision", choices=["fp16", "fp32x3"], default="fp16",
                   help="fp16: fp16 MMA operands (default); fp32x3: fp32-grade logits")
    p.add_argument("--out", type=pathlib.Path, required=True, help="directory to write the samples to")
    return p


def designable_mask(R: int, W: int, appended: int, rows, columns) -> torch.Tensor:
    """bool [R + appended, W] of the designable entries by the rules in the module docstring; rows and columns are
    0-based lists or None. Raises ValueError for a row or column outside the alignment."""
    total = R + appended
    for name, sel, size in (("row", rows, total), ("column", columns, W)):
        if sel is not None and max(sel) >= size:
            raise ValueError(f"{name} {max(sel) + 1} is outside the alignment's {size} {name}s")
    if rows is None and columns is None:
        mask = torch.zeros((total, W), dtype=torch.bool)
        mask[R if appended else 0:] = True
        return mask
    r = torch.zeros(total, dtype=torch.bool)
    r[list(range(total)) if rows is None else rows] = True
    c = torch.zeros(W, dtype=torch.bool)
    c[list(range(W)) if columns is None else columns] = True
    mask = r[:, None] & c[None, :]
    mask[R:] = True
    return mask


def run(args) -> int:
    """Returns the number of chains written."""
    if args.msa_select != "first" and args.msa_samples is None:
        raise ValueError(f"--msa-select {args.msa_select} picks --msa-samples rows from the file: give --msa-samples")
    msa = read_alignment(args.msa, args.msa_samples, args.msa_select)
    if not msa:
        raise ValueError(f"{args.msa} holds no alignment records")
    model, alphabet, _ = load_model(args.model_location)
    if getattr(model, "random_init", False):
        raise RuntimeError("refusing to sample from a random-init model: give model_location a checkpoint")
    tokens = alphabet.get_batch_converter()(msa)[2]
    R, C = tokens.shape[1:]
    if args.append_rows:
        new = torch.full((1, args.append_rows, C), alphabet.mask_idx, dtype=torch.int64)
        new[:, :, 0] = alphabet.cls_idx
        tokens = torch.cat([tokens, new], 1)
    designable = designable_mask(R, C - 1, args.append_rows, args.rows, args.columns)
    dev = torch.device("cuda", torch.cuda.current_device())
    model = model.eval()
    if args.precision != "fp16":
        model.set_precision(args.precision)
    model = model.to(dev)
    out = sampling.msa_gibbs(model, tokens, designable=designable, chains=args.chains, sweeps=args.sweeps,
                             block=args.block, temperature=args.temperature, seed=args.seed, gaps=args.gaps,
                             max_tokens=args.max_tokens)
    per_sweep = out["logp"].shape[1] // args.sweeps
    last = out["logp"][:, -per_sweep:].double().sum(1).tolist()
    names = [desc for desc, _ in msa] + [f"generated_{i}" for i in range(args.append_rows)]
    args.out.mkdir(parents=True, exist_ok=True)
    for c, aln in enumerate(out["tokens"][:, :, 1:].tolist()):
        with open(args.out / f"sample_{c}.a3m", "w") as f:
            for name, row in zip(names, aln):
                f.write(f">{name}\n{''.join(alphabet.get_tok(t) for t in row)}\n")
    with open(args.out / "samples.tsv", "w") as f:
        f.write("chain\tseed\tlogp\n")
        for c, lp in enumerate(last):
            f.write(f"{c}\t{args.seed}\t{lp:.4f}\n")
    return len(last)


def main():
    run(create_parser().parse_args())


if __name__ == "__main__":
    main()
