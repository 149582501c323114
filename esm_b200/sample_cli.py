"""`python -m esm_b200.sample_cli MODEL (--sequence SEQ | --length N) [--positions 1-10,25] [--chains C] [--sweeps W]
[--block K] [--temperature T] [--seed S] [--max-tokens N] [--precision fp16|fp32x3|fp8] [--cpu-offload]
--out samples.fasta`: sample protein sequences by Gibbs sampling (esm_b200.sampling).

--sequence starts every chain from that protein; --length N starts from N masked residues (de novo generation, every
position designable). --positions lists the designable residues as 1-based numbers and inclusive ranges (default:
all). MODEL is loaded as extract_cli loads it (an ESM-2, ESM-1b or ESM-1v name or a local .pt file), and a random-init
model is refused. Writes one FASTA record per chain, `>sample_{c} seed={seed} logp={logp}`, where logp is the summed
log q of the chain's last sweep.
"""
from __future__ import annotations

import argparse
import pathlib

import torch

from . import pretrained, sampling
from .variants import DEFAULT_MAX_TOKENS


def parse_positions(text: str):
    """"1-10,25" -> 0-based residue indices [0, ..., 9, 24]; ranges are inclusive, numbers 1-based."""
    out = []
    for part in text.split(","):
        part = part.strip()
        lo, sep, hi = part.partition("-")
        try:
            a = int(lo)
            b = int(hi) if sep else a
        except ValueError:
            raise argparse.ArgumentTypeError(f"bad position or range {part!r}: use 1-based numbers like 1-10,25")
        if a < 1 or b < a:
            raise argparse.ArgumentTypeError(f"bad position or range {part!r}: numbers start at 1, ranges ascend")
        out.extend(range(a - 1, b))
    return out


def _positive(text: str) -> int:
    v = int(text)
    if v < 1:
        raise argparse.ArgumentTypeError(f"must be >= 1, got {v}")
    return v


def create_parser():
    p = argparse.ArgumentParser(description="Sample protein sequences from a masked language model (Gibbs sampling)")
    p.add_argument("model_location", type=str,
                   help="ESM-2, ESM-1b or ESM-1v model name (esm2_t33_650M_UR50D, esm1b_t33_650M_UR50S, "
                        "esm1v_t33_650M_UR90S_1, ...) or a local .pt file")
    start = p.add_mutually_exclusive_group(required=True)
    start.add_argument("--sequence", type=str, help="start every chain from this protein")
    start.add_argument("--length", type=_positive, help="start from this many masked residues (de novo)")
    p.add_argument("--positions", type=parse_positions, default=None,
                   help="designable residues, 1-based numbers and inclusive ranges such as 1-10,25 (default: all)")
    p.add_argument("--chains", type=_positive, default=1, help="independent chains, one FASTA record each")
    p.add_argument("--sweeps", type=_positive, default=1, help="passes over the designable positions")
    p.add_argument("--block", type=_positive, default=1, help="positions resampled together per step")
    p.add_argument("--temperature", type=float, default=1.0, help="divides the logits (finite, > 0)")
    p.add_argument("--seed", type=int, default=0, help="random stream key in [0, 2^64)")
    p.add_argument("--max-tokens", type=int, default=DEFAULT_MAX_TOKENS,
                   help="tokens per stack call (chains per chunk times L + 2); the samples do not depend on it")
    p.add_argument("--precision", choices=["fp16", "fp32x3", "fp8"], default="fp16",
                   help="fp16: fp16 MMA operands (default); fp32x3: fp32-grade logits (~3x slower); fp8: e4m3 "
                        "projections")
    p.add_argument("--cpu-offload", action="store_true",
                   help="keep the transformer layers' weights in pinned host memory and stream them to the GPU layer "
                        "by layer (ESM-2 15B on one GPU); same samples")
    p.add_argument("--out", type=pathlib.Path, required=True, help="FASTA file to write")
    return p


def run(args) -> int:
    """Returns the number of records written."""
    model, alphabet = pretrained.load_model_and_alphabet(args.model_location)
    if getattr(model, "random_init", False):
        raise RuntimeError("refusing to sample from a random-init model: give model_location a checkpoint")
    dev = torch.device("cuda", torch.cuda.current_device())
    model = model.eval()
    if args.precision != "fp16":
        model.set_precision(args.precision)
    model = model.cpu_offload(dev) if args.cpu_offload else model.to(dev)
    if args.sequence is not None:
        tokens = alphabet.get_batch_converter()([("start", args.sequence)])[2]
    else:
        tokens = torch.tensor([[alphabet.cls_idx] + [alphabet.mask_idx] * args.length + [alphabet.eos_idx]])
    out = sampling.gibbs(model, tokens, positions=args.positions, chains=args.chains, sweeps=args.sweeps,
                         block=args.block, temperature=args.temperature, seed=args.seed, max_tokens=args.max_tokens)
    per_sweep = out["logp"].shape[1] // args.sweeps
    last = out["logp"][:, -per_sweep:].double().sum(1).tolist()
    toks = out["tokens"][:, 1:-1].tolist()
    args.out.parent.mkdir(parents=True, exist_ok=True)
    with open(args.out, "w") as f:
        for c, (row, lp) in enumerate(zip(toks, last)):
            f.write(f">sample_{c} seed={args.seed} logp={lp:.4f}\n{''.join(alphabet.get_tok(t) for t in row)}\n")
    return len(toks)


def main():
    run(create_parser().parse_args())


if __name__ == "__main__":
    main()
