"""`python -m esm_b200.predict_cli --model-location M [M ...] --sequence S --dms-input in.csv --dms-output out.csv ...`:
the command line of the reference's examples/variant-prediction/predict.py (same flags, defaults and choices,
predict.py:45-104, plus --max-tokens) on the library's batched scorers (esm_b200.variants).

  * models: ESM-2 and ESM-1b / ESM-1v names or .pt files load through pretrained.load_model_and_alphabet; MSA
    Transformer names, and .pt files whose args.arch is "msa_transformer", through load_msa_model_and_alphabet
    (predict.py loads all of them through one loader). Each model is freed before the next one is loaded.
  * output: predict.py's table (df.to_csv): a leading unnamed index column, the input columns as read, then one
    column per --model-location named by the location string. It is written with the csv module: the input cells are
    copied unchanged, the scores written with repr. Neither pandas nor Biopython is needed.
  * --precision fp32x3 runs every model (sequence models and the MSA Transformer) with fp16 hi + lo operand pairs.
  * --window N scores proteins longer than N residues (ESM-1b / ESM-1v cannot take more than 1022) through overlapping
    windows of N residues (esm_b200.windows), with every strategy; sequence models only.
  * --msa-select max / min reads the whole a3m file and keeps --msa-samples rows picked by the greedy Hamming
    selection of the reference's contact notebook (esm_b200.msa_select.greedy_select) instead of the first ones.
  * there is no CPU path: --nogpu raises.
"""
from __future__ import annotations

import argparse
import csv
import gc
import pathlib
from typing import Dict, List

import torch

from . import msa_select, pretrained, variants

STRATEGIES = ["wt-marginals", "pseudo-ppl", "masked-marginals"]
PRECISIONS = ["fp16", "fp32x3"]
MSA_SELECT = ["first", "max", "min"]
MSA_ONLY_MASKED = "MSA Transformer only supports masked marginal strategy"  # predict.py:163-165
MSA_NO_WINDOW = "--window applies to ESM-2, ESM-1b and ESM-1v models; MSA Transformer alignments are not windowed"


def create_parser():
    """The flags, defaults and choices of predict.py:45-104, plus --max-tokens and --precision."""
    p = argparse.ArgumentParser(description="Score the single mutants of a deep mutational scan with one or more ESM "
                                            "models on the GPU and write the table back with one score column per "
                                            "model")
    p.add_argument("--model-location", type=str, nargs="+",
                   help="one or more models: ESM-2, ESM-1b, ESM-1v or MSA Transformer names, or local .pt files")
    p.add_argument("--sequence", type=str, help="wild-type protein sequence the mutations refer to")
    p.add_argument("--dms-input", type=pathlib.Path, help="input CSV table with one mutation per row")
    p.add_argument("--mutation-col", type=str, default="mutant",
                   help="name of the input column holding the mutations, written wild type, position, mutant (e.g. A24G)")
    p.add_argument("--dms-output", type=pathlib.Path, help="output CSV: the input table plus one score column per model")
    p.add_argument("--offset-idx", type=int, default=0,
                   help="number subtracted from each mutation position to get its 0-based index in --sequence")
    p.add_argument("--scoring-strategy", type=str, default="wt-marginals", choices=STRATEGIES,
                   help="wt-marginals: one pass over the wild type; masked-marginals: each position masked in turn; "
                        "pseudo-ppl: pseudo-log-likelihood of each mutated sequence")
    p.add_argument("--msa-path", type=pathlib.Path, help="a3m alignment whose first row is --sequence (MSA Transformer)")
    p.add_argument("--msa-samples", type=int, default=400, help="how many alignment rows to read, from the top")
    p.add_argument("--msa-select", choices=MSA_SELECT, default="first",
                   help="which --msa-samples rows to keep: first: the first ones in the file; max / min: the whole file "
                        "is read and rows are picked greedily for the largest / smallest mean Hamming distance to "
                        "those already picked, starting from the query (the contact notebook's greedy_select)")
    p.add_argument("--nogpu", action="store_true", help="accepted for compatibility; raises, as there is no CPU path")
    p.add_argument("--max-tokens", type=int, default=variants.DEFAULT_MAX_TOKENS,
                   help="tokens per batched forward of masked copies (at least one copy per forward)")
    p.add_argument("--precision", choices=PRECISIONS, default="fp16",
                   help="fp16: fp16 MMA operands (default, fastest); fp32x3: hi+lo operand pairs, fp32-grade scores "
                        "(slower); applies to every model location")
    p.add_argument("--cpu-offload", action="store_true",
                   help="keep the transformer layers' weights of ESM-2 / ESM-1b / ESM-1v models in pinned host memory "
                        "and stream them to the GPU layer by layer (ESM-2 15B on one GPU); same scores. The MSA "
                        "Transformer stays resident")
    p.add_argument("--window", type=int, default=None,
                   help="score through overlapping windows of this many residues, merged with tapered weights, so "
                        "that proteins longer than the model's window (1022 residues for ESM-1b / ESM-1v) can be "
                        "scored; sequence models only")
    return p


def is_msa_location(location: str) -> bool:
    """Whether a --model-location names an MSA Transformer: a name in pretrained.MSA_ARCH, or a .pt file whose
    args.arch is "msa_transformer" (read through a memory map, so the weights are not loaded twice)."""
    if location.endswith(".pt"):
        try:
            data = torch.load(location, map_location="cpu", weights_only=False, mmap=True)
        except RuntimeError:  # files in the legacy (non-zip) format cannot be memory-mapped
            data = torch.load(location, map_location="cpu", weights_only=False)
        return getattr(data.get("args"), "arch", None) == "msa_transformer"
    return location in pretrained.MSA_ARCH


def load_model(location: str):
    """(model, alphabet, is_msa) for a --model-location."""
    if is_msa_location(location):
        model, alphabet = pretrained.load_msa_model_and_alphabet(location)
        return model, alphabet, True
    model, alphabet = pretrained.load_model_and_alphabet(location)
    return model, alphabet, False


def read_table(path) -> (List[str], List[List[str]]):
    """(header, rows) of a CSV file, cells as written. Blank lines are skipped, as pandas.read_csv skips them."""
    with open(path, newline="") as f:
        rows = [r for r in csv.reader(f) if r and not (len(r) == 1 and not r[0].strip())]
    return rows[0], rows[1:]


def write_table(path, header: List[str], rows: List[List[str]], scores: Dict[str, List[float]]) -> None:
    """df.to_csv(path) of predict.py:235: index column, input columns, one score column per model location (a location
    equal to an input column's name replaces that column, as the DataFrame assignment does)."""
    header = list(header)
    rows = [list(r) for r in rows]
    for loc, col in scores.items():
        cells = [repr(v) for v in col]
        if loc in header:
            j = header.index(loc)
            for r, c in zip(rows, cells):
                r[j] = c
        else:
            header.append(loc)
            for r, c in zip(rows, cells):
                r.append(c)
    with open(path, "w", newline="") as f:
        w = csv.writer(f, lineterminator="\n")
        w.writerow([""] + header)
        for i, r in enumerate(rows):
            w.writerow([str(i)] + r)


def read_alignment(path, samples, select: str = "first"):
    """The alignment rows to run: the first `samples` records of the a3m file (all for None), or with select "max" /
    "min" `samples` rows of the whole file picked by msa_select.greedy_select."""
    if select == "first":
        return variants.read_msa(path, samples)
    return msa_select.greedy_select(variants.read_msa(path, None), samples, select)


def score_model(model, alphabet, is_msa: bool, args, mutations: List[str]) -> List[float]:
    """predict.py:159-233 for one model on the library."""
    window = getattr(args, "window", None)
    if is_msa:
        if window is not None:
            raise ValueError(MSA_NO_WINDOW)
        data = [read_alignment(args.msa_path, args.msa_samples, getattr(args, "msa_select", "first"))]
        assert args.scoring_strategy == "masked-marginals", MSA_ONLY_MASKED
        _, _, tokens = alphabet.get_batch_converter()(data)
        lp = variants.masked_marginals(model, tokens, max_tokens=args.max_tokens)
        return variants.label_scores(lp, alphabet, args.sequence, mutations, args.offset_idx)
    _, _, tokens = alphabet.get_batch_converter()([("protein1", args.sequence)])
    if args.scoring_strategy == "wt-marginals":
        lp = variants.wt_marginals(model, tokens, window=window)
    elif args.scoring_strategy == "masked-marginals":
        lp = variants.masked_marginals(model, tokens, max_tokens=args.max_tokens, window=window)
    else:
        return variants.pseudo_ppl(model, alphabet, args.sequence, mutations, args.offset_idx, args.max_tokens,
                                   window=window)
    return variants.label_scores(lp, alphabet, args.sequence, mutations, args.offset_idx)


def run(args) -> None:
    if args.nogpu:
        raise RuntimeError("--nogpu: esm_b200 runs on CUDA (sm_90a) only and has no CPU path; run without --nogpu "
                           "on a machine with an H100")
    if getattr(args, "window", None) is not None:
        if args.window < 2:
            raise ValueError(f"--window must be at least 2 residues, got {args.window}")
        if any(is_msa_location(loc) for loc in args.model_location):
            raise ValueError(MSA_NO_WINDOW)
    header, rows = read_table(args.dms_input)
    col = header.index(args.mutation_col)
    mutations = [r[col] for r in rows]
    scores: Dict[str, List[float]] = {}
    for location in args.model_location:
        model, alphabet, is_msa = load_model(location)
        if getattr(model, "random_init", False):
            raise RuntimeError("refusing to score variants with a random-init model: give --model-location a checkpoint")
        model = model.eval()
        if getattr(args, "precision", "fp16") != "fp16":
            model.set_precision(args.precision)
        model = model.cpu_offload() if getattr(args, "cpu_offload", False) and not is_msa else model.cuda()
        scores[location] = score_model(model, alphabet, is_msa, args, mutations)
        del model
        gc.collect()
        torch.cuda.empty_cache()
    write_table(args.dms_output, header, rows, scores)


def main():
    run(create_parser().parse_args())


if __name__ == "__main__":
    main()
