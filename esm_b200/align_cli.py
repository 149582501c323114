"""Align search hits residue by residue (esm_b200.align):

    python -m esm_b200.align_cli HITS.tsv --queries QDIR --targets TDIR --layer 33 \\
        [--mode local|global] [--gap-open O] [--gap-extend E] [--no-zscore] [--max-cells N] \\
        --out alignments.tsv [--fasta SEQS.fasta --a3m OUT_DIR]

HITS.tsv is search_cli query output (query, rank, target, score). QDIR and TDIR are extract_cli output directories
written with --include per_tok --repr_layers LAYER (for search_cli query --all, both are the index's directory).
Each <label>.pt named in the hits is read once. alignments.tsv has one line per hit: query, rank, target, the search
score, the alignment score, the query and target spans (0-based, end exclusive) and the CIGAR-like op string.
With --fasta (the sequences the embeddings were extracted from) and --a3m, one <query>.a3m per query is written:
the query first, then its hits in rank order, ready for predict_cli --msa-path or msa_select.
"""
from __future__ import annotations

import argparse
import pathlib
import sys
from typing import Dict, List, Tuple

import torch

from . import align
from .data import FastaBatchedDataset


def create_parser():
    p = argparse.ArgumentParser(description="Align search_cli hits by their per-residue embeddings")
    p.add_argument("hits", type=pathlib.Path, help="search_cli query output")
    p.add_argument("--queries", type=pathlib.Path, required=True, help="extract_cli directory of the queries")
    p.add_argument("--targets", type=pathlib.Path, required=True, help="extract_cli directory of the targets")
    p.add_argument("--layer", type=int, required=True, help="the representation layer to align")
    p.add_argument("--mode", choices=list(align.MODES), default="local")
    p.add_argument("--gap-open", type=float, default=align.GAP_OPEN, help="gap open penalty (default untuned)")
    p.add_argument("--gap-extend", type=float, default=align.GAP_EXTEND, help="gap extend penalty (default untuned)")
    p.add_argument("--no-zscore", action="store_true", help="align on the raw cosine similarities")
    p.add_argument("--max-cells", type=int, default=None, help="similarity cells per GPU chunk")
    p.add_argument("--out", type=pathlib.Path, required=True)
    p.add_argument("--fasta", type=pathlib.Path, help="the sequences the embeddings were extracted from")
    p.add_argument("--a3m", type=pathlib.Path, help="directory for one <query>.a3m per query (needs --fasta)")
    return p


def read_hits(path) -> List[Tuple[str, int, str, str]]:
    """(query, rank, target, score text) per line of a search_cli hits file."""
    with open(path) as f:
        header = f.readline().rstrip("\n").split("\t")
        if header[:4] != ["query", "rank", "target", "score"]:
            raise ValueError(f"{path} is not search_cli query output (header {header})")
        out = []
        for n, line in enumerate(f, 2):
            parts = line.rstrip("\n").split("\t")
            if len(parts) < 4:
                raise ValueError(f"{path}:{n}: expected 4 tab-separated fields")
            out.append((parts[0], int(parts[1]), parts[2], parts[3]))
    return out


def load_embeddings(root: pathlib.Path, labels, layer: int) -> Dict[str, torch.Tensor]:
    """representations[layer] of <root>/<label>.pt for each label, each file read once."""
    out = {}
    for label in sorted(set(labels)):
        path = root / f"{label}.pt"
        if not path.exists():
            raise ValueError(f"{path} not found: the hits name {label!r}")
        obj = torch.load(path, map_location="cpu", weights_only=True)
        reps = obj.get("representations", {}) if isinstance(obj, dict) else {}
        if layer not in reps:
            raise ValueError(f"{path} has no representations[{layer}] (extract_cli --include per_tok "
                             f"--repr_layers {layer})")
        out[label] = reps[layer]
    return out


def check_lengths(emb: Dict[str, torch.Tensor], seqs: Dict[str, str]) -> None:
    for label, x in emb.items():
        if label not in seqs:
            raise ValueError(f"{label!r} is not in the FASTA file")
        if x.shape[0] != len(seqs[label]):
            raise ValueError(f"{label!r} has {x.shape[0]} embedding rows but {len(seqs[label])} residues: its "
                             f"extraction was truncated (rerun extract_cli with --truncation_seq_length "
                             f"{len(seqs[label])} or --window)")


def run(args) -> int:
    """Returns the number of alignment lines written."""
    if args.a3m is not None and args.fasta is None:
        raise ValueError("--a3m needs --fasta: an a3m row holds residues, not embeddings")
    hits = read_hits(args.hits)
    qemb = load_embeddings(args.queries, [h[0] for h in hits], args.layer)
    temb = load_embeddings(args.targets, [h[2] for h in hits], args.layer)
    seqs = None
    if args.fasta is not None:
        ds = FastaBatchedDataset.from_file(args.fasta)
        seqs = dict(zip(ds.sequence_labels, ds.sequence_strs))
        check_lengths(qemb, seqs)
        check_lengths(temb, seqs)
    res = align.align_pairs([qemb[h[0]] for h in hits], [temb[h[2]] for h in hits], args.mode, args.gap_open,
                            args.gap_extend, zscore=not args.no_zscore, max_cells=args.max_cells)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    with open(args.out, "w") as f:
        f.write("query\trank\ttarget\tsearch_score\tscore\tq_start\tq_end\tt_start\tt_end\tcigar\n")
        for (q, rank, t, s), a in zip(hits, res):
            f.write(f"{q}\t{rank}\t{t}\t{s}\t{a.score:.6g}\t{a.query_span[0]}\t{a.query_span[1]}\t"
                    f"{a.target_span[0]}\t{a.target_span[1]}\t{a.cigar()}\n")
    if args.a3m is not None:
        per_query: Dict[str, list] = {}
        for (q, rank, t, _), a in zip(hits, res):
            per_query.setdefault(q, []).append((rank, t, a))
        for q, items in per_query.items():
            items.sort(key=lambda x: x[0])
            path = args.a3m / f"{q}.a3m"
            path.parent.mkdir(parents=True, exist_ok=True)
            path.write_text(align.to_a3m(seqs[q], [(t, seqs[t], a) for _, t, a in items], q))
    return len(hits)


def main():
    args = create_parser().parse_args()
    n = run(args)
    print(f"wrote {n} alignments to {args.out}", file=sys.stderr)


if __name__ == "__main__":
    main()
