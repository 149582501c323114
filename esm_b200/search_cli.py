"""Nearest-neighbour search over extract_cli embeddings (esm_b200.search):

    python -m esm_b200.search_cli build EXTRACT_DIR --layer 33 [--metric cosine|l2] --out db.pt
    python -m esm_b200.search_cli build EXTRACT_DIR --layer 33 [--metric cosine|l2] --out db/ [--append]
    python -m esm_b200.search_cli build EXTRACT_DIR --layer 33 [--metric cosine|l2] --out ivf.pt --nlist 4096
                                        [--train-rows N] [--iters 20] [--seed 0]
    python -m esm_b200.search_cli query db.pt|db/|ivf.pt (--queries EXTRACT_DIR | --all) --k 10 [--nprobe P]
                                        --out hits.tsv
    python -m esm_b200.search_cli range db.pt|db/ (--queries EXTRACT_DIR | --all)
                                        (--min-score S | --max-distance R) [--max-hits M] --out hits.tsv

`build` reads the mean representation at --layer of every `<label>.pt` under EXTRACT_DIR (extract_cli --include mean)
and saves an index: one file (EmbeddingIndex) when --out ends in .pt, else a sharded index directory (IndexWriter),
written one shard at a time so that memory stays bounded; --append adds EXTRACT_DIR's proteins to an existing
directory index as new shards. Both formats hold the rows in label order, so they give the same hits. `query`
searches an index with the mean representations of a second extract_cli directory, which must hold the index's layer
at the index's width, or with every indexed protein against the others (--all); a directory index is streamed through
the GPU (ShardedIndex), so it may be larger than the device's memory. hits.tsv has one line per hit: query, rank
(1-based), target, score (cosine similarity, or Euclidean distance for l2). Embedding the queries stays in
extract_cli, with its model loading and checkpoint checks.

`build --nlist` trains an inverted-file index (IVFIndex: k-means lists on the GPU) and saves it to a .pt file; it
cannot go to a directory or be appended to. `query` reads the index type from the file, and --nprobe (default
min(8, nlist); nlist scans every list and gives the exact hits) sets how many lists each query scans. An IVF query
can find fewer than k hits when its lists hold fewer rows; hits.tsv then has fewer lines for it. --nprobe on an exact
or sharded index is refused.

`range` finds every indexed protein within a threshold instead of the top k: --min-score for a cosine index (every
hit with similarity >= S), --max-distance for an l2 index (distance <= R); --max-hits keeps each query's best M. It
writes the same hits.tsv as `query`, ranks in the same order, so align_cli reads it unchanged. A threshold flag that
does not match the index's metric, NaN, or an IVF index (its range over the probed lists is not defined) is refused.
"""
from __future__ import annotations

import argparse
import pathlib
import sys

import torch

from . import search


def create_parser():
    p = argparse.ArgumentParser(description="Exact k-nearest-neighbour search over extract_cli embeddings")
    sub = p.add_subparsers(dest="command", required=True)
    b = sub.add_parser("build", help="build an index from an extract_cli output directory")
    b.add_argument("extract_dir", type=pathlib.Path)
    b.add_argument("--layer", type=int, required=True, help="the representation layer to index")
    b.add_argument("--metric", choices=list(search.METRICS), default="cosine")
    b.add_argument("--out", type=pathlib.Path, required=True,
                   help="db.pt: one file; any other path: a sharded index directory")
    b.add_argument("--append", action="store_true", help="add shards to an existing directory index")
    b.add_argument("--shard-rows", type=int, default=search.SHARD_ROWS, help="rows per shard of a directory index")
    b.add_argument("--nlist", type=int, help="train an inverted-file index of this many k-means lists (.pt only)")
    b.add_argument("--train-rows", type=int, help="k-means training sample (default min(N, 256 nlist))")
    b.add_argument("--iters", type=int, default=20, help="k-means iterations")
    b.add_argument("--seed", type=int, default=0, help="k-means training sample seed")
    q = sub.add_parser("query", help="search an index")
    q.add_argument("index", type=pathlib.Path)
    src = q.add_mutually_exclusive_group(required=True)
    src.add_argument("--queries", type=pathlib.Path, help="an extract_cli output directory of query proteins")
    src.add_argument("--all", action="store_true", help="every indexed protein against the others")
    q.add_argument("--k", type=int, default=10, help=f"hits per query, 1 to {search.MAX_K}")
    q.add_argument("--nprobe", type=int, help="lists scanned per query (IVF index only)")
    q.add_argument("--out", type=pathlib.Path, required=True)
    r = sub.add_parser("range", help="every indexed protein within a threshold of each query")
    r.add_argument("index", type=pathlib.Path)
    src = r.add_mutually_exclusive_group(required=True)
    src.add_argument("--queries", type=pathlib.Path, help="an extract_cli output directory of query proteins")
    src.add_argument("--all", action="store_true", help="every indexed protein against the others")
    thr = r.add_mutually_exclusive_group(required=True)
    thr.add_argument("--min-score", type=float, help="cosine index: hits with similarity >= this")
    thr.add_argument("--max-distance", type=float, help="l2 index: hits at Euclidean distance <= this")
    r.add_argument("--max-hits", type=int, help="keep each query's best M hits")
    r.add_argument("--out", type=pathlib.Path, required=True)
    return p


def csr_rows(lims: torch.Tensor, values: torch.Tensor) -> list:
    """A CSR array (lims [Q + 1]) as one Python list per query."""
    lims, values = lims.cpu().tolist(), values.cpu().tolist()
    return [values[lims[i]:lims[i + 1]] for i in range(len(lims) - 1)]


def write_hits(path, query_labels, target_labels, scores, idx) -> int:
    """hits.tsv from [Q, k] tensors or per-query lists; returns the number of hit lines."""
    if isinstance(scores, torch.Tensor):
        scores, idx = scores.cpu().tolist(), idx.cpu().tolist()
    n = 0
    with open(path, "w") as f:
        f.write("query\trank\ttarget\tscore\n")
        for q, row_s, row_i in zip(query_labels, scores, idx):
            for r, (s, i) in enumerate(zip(row_s, row_i)):
                if i < 0:  # an IVF query with fewer hits than k
                    continue
                f.write(f"{q}\t{r + 1}\t{target_labels[i]}\t{s:.6g}\n")
                n += 1
    return n


BUILD_BATCH = 4096  # extract_cli files read per IndexWriter.add


def _is_file_index(path: pathlib.Path) -> bool:
    return path.suffix == ".pt"


def build_shards(extract_dir, layer: int, metric: str, out, append: bool, shard_rows: int = search.SHARD_ROWS) -> int:
    """A sharded index of extract_dir's mean representations in label order, or new shards after an existing index's
    (append). Files are read twice, once for the labels and once in label order, so memory holds one batch and one
    shard. Returns the rows added."""
    out = pathlib.Path(out)
    exists = (out / search.MANIFEST).exists()
    if exists and not append:
        raise ValueError(f"{out} already holds an index: pass --append to add to it")
    if append and not exists:
        raise ValueError(f"--append needs an existing directory index at {out}")
    search._check_metric(metric)
    items = search._scan_extract_dir(extract_dir, layer, keep_vectors=False)
    dim = torch.load(items[0][1], map_location="cpu", weights_only=True)["mean_representations"][layer].numel()
    writer = search.IndexWriter(out, dim, metric, layer, shard_rows)
    for b0 in range(0, len(items), BUILD_BATCH):
        batch = items[b0:b0 + BUILD_BATCH]
        vecs = [torch.load(f, map_location="cpu", weights_only=True)["mean_representations"][layer].reshape(-1).float()
                for _, f in batch]
        writer.add(torch.stack(vecs), [l for l, _ in batch])
    writer.close()
    return len(items)


def run(args) -> int:
    """Returns the number of rows indexed (build) or hit lines written (query)."""
    if args.command == "build":
        if args.nlist is not None and not _is_file_index(args.out):
            raise ValueError("--nlist builds an IVF index into one .pt file, not a directory")
        if args.nlist is not None and args.append:
            raise ValueError("--nlist builds a new IVF index: it cannot --append")
        if args.nlist is None and (args.train_rows is not None or args.iters != 20 or args.seed != 0):
            raise ValueError("--train-rows, --iters and --seed train an IVF index: pass --nlist")
        if not _is_file_index(args.out):
            return build_shards(args.extract_dir, args.layer, args.metric, args.out, args.append, args.shard_rows)
        if args.append:
            raise ValueError("--append adds shards to a directory index, not to a .pt file")
        if args.nlist is not None:
            index = search.IVFIndex.from_extract_dir(args.extract_dir, args.layer, args.metric, nlist=args.nlist,
                                                     train_rows=args.train_rows, iters=args.iters, seed=args.seed)
        else:
            index = search.EmbeddingIndex.from_extract_dir(args.extract_dir, args.layer, args.metric)
        args.out.parent.mkdir(parents=True, exist_ok=True)
        index.save(args.out)
        return len(index)
    if args.command == "range":
        return run_range(args)
    sharded = args.index.is_dir()
    if sharded and args.nprobe is not None:
        raise ValueError("--nprobe applies to an IVF index; a directory index is searched exactly")
    index = search.ShardedIndex.open(args.index) if sharded else search.load_file_index(args.index, device="cpu")
    ivf = isinstance(index, search.IVFIndex)
    if args.nprobe is not None and not ivf:
        raise ValueError(f"--nprobe applies to an IVF index; {args.index} is an exact index")
    if ivf:
        index.check_nprobe(args.nprobe)
    candidates = len(index) - 1 if args.all else len(index)
    search._check_k(args.k, candidates)
    qlabels, queries = _queries(args, index)
    if not sharded:
        index = index.to(torch.device("cuda", torch.cuda.current_device()))
    extra = {"nprobe": args.nprobe} if ivf else {}
    scores, idx = index.search_all(args.k, **extra) if args.all else index.search(queries, args.k, **extra)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    return write_hits(args.out, qlabels, index.labels, scores, idx)


def _queries(args, index):
    """(query labels, fp32 queries or None for --all) of a query or range command, checked against the index."""
    if args.all:
        return index.labels, None
    if index.layer is None:
        raise ValueError(f"{args.index} records no layer: query it through esm_b200.search")
    qlabels, queries = search._read_extract_dir(args.queries, index.layer)
    if queries.shape[1] != index.dim:
        raise ValueError(f"the queries have width {queries.shape[1]}, the index {index.dim}")
    search.prepare_rows(queries, index.metric, "queries")
    return qlabels, queries


def run_range(args) -> int:
    sharded = args.index.is_dir()
    index = search.ShardedIndex.open(args.index) if sharded else search.load_file_index(args.index, device="cpu")
    if isinstance(index, search.IVFIndex):
        raise ValueError(f"{args.index} is an IVF index: a range search over its probed lists is not defined; "
                         f"range-search the exact index it was built from")
    thr = {"min_score": args.min_score, "max_distance": args.max_distance, "max_hits": args.max_hits}
    search.check_range_args(index.metric, **thr)
    qlabels, queries = _queries(args, index)
    if not sharded:
        index = index.to(torch.device("cuda", torch.cuda.current_device()))
    lims, scores, idx = index.range_search_all(**thr) if args.all else index.range_search(queries, **thr)
    args.out.parent.mkdir(parents=True, exist_ok=True)
    return write_hits(args.out, qlabels, index.labels, csr_rows(lims, scores), csr_rows(lims, idx))


def main():
    args = create_parser().parse_args()
    n = run(args)
    print(f"indexed {n} rows" if args.command == "build" else f"wrote {n} hits to {args.out}", file=sys.stderr)


if __name__ == "__main__":
    main()
