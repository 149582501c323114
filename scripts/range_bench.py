"""Developer tool (GPU box): range search (esm_b200.search range_search) against top-k search and a plain-PyTorch path.

The data is scripts/ivf_bench.py's synthetic mixture: seeded clusters on the unit sphere, E = 1280, fp16 cosine rows;
the queries come from the same mixture. For each N (resident: 1 M and 10 M rows; streamed: a sharded copy of the first
size, in a temporary directory), Q in {1, 1,024, 8,192} and a min_score picked for about 10, 1,000 and 100,000 hits a
query (the median over 8 queries of the score at that rank), it reports:
  * call_ms: one range_search call, host clock around synchronised work (median of --repeats after a warm-up);
  * kernel_ms: the range kernel alone (esmb200_knn_range on one query batch, CUDA events), and its TFLOP/s
    (2 Q N E operations) against the 989 TFLOP/s dense fp16 figure of the H100 SXM data sheet;
  * hits and hits/s over the call;
  * topk_ms: search(k = 128) at the same Q and N;
  * torch_ms: chunked torch.mm + mask + nonzero + sort (N = 1 M, Q <= 1,024), and whether its hits equal the range
    search's outside a 1e-3 band around the threshold (the two accumulate in different orders).
Cases with more than --max-total hits are skipped (the results alone would take 12 bytes a hit). Prints one JSON line
per case and a last line with the card name and power limit (a read-only nvidia-smi query), and writes them to --out.

    python scripts/range_bench.py [--repeats 3] [--sizes 1000000,10000000] [--out results.jsonl]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from esm_b200 import search  # noqa: E402
from ivf_bench import E, mixture, query_gpu  # noqa: E402

QS = (1, 1024, 8192)
TARGETS = (10, 1000, 100_000)
PEAK_TFLOPS = 989.0


def host_timed(fn, repeats):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return sorted(times)[len(times) // 2], out


def kernel_ms(index, q16, tau, nnz, repeats):
    hits = search._HitBuffer(q16.shape[0], max(nnz, 1), index.device)

    def launch():
        hits.counts.zero_()
        hits.total.zero_()
        search.knn_range(q16, index.rows, 0, tau, *hits.tensors())
    launch()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        hits.counts.zero_()
        hits.total.zero_()
        a.record()
        search.knn_range(q16, index.rows, 0, tau, *hits.tensors())
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def torch_path(rows, q16, t):
    """Every (query, row) with fp32 score >= t by chunked torch.mm, sorted by (query, score desc, row)."""
    qs, js, ss = [], [], []
    for r0 in range(0, rows.shape[0], 1 << 20):
        s = torch.mm(q16.float(), rows[r0:r0 + (1 << 20)].float().T)
        i, j = (s >= t).nonzero(as_tuple=True)
        qs.append(i)
        js.append(j + r0)
        ss.append(s[i, j])
    q, j, s = torch.cat(qs), torch.cat(js), torch.cat(ss)
    order = torch.sort(-s, stable=True).indices
    order = order[torch.sort(q[order], stable=True).indices]
    return q[order], j[order], s[order]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sizes", type=str, default="1000000,10000000")
    ap.add_argument("--centres", type=int, default=20000)
    ap.add_argument("--spread", type=float, default=1.0)
    ap.add_argument("--max-total", type=float, default=2e8)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("range_bench needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(0)
    centres = torch.nn.functional.normalize(torch.randn((args.centres, E), generator=g, device="cuda"), dim=1)
    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    sizes = [int(s) for s in args.sizes.split(",")]
    for N in sizes:
        rows = mixture(N, centres, args.spread, seed=1)
        index = search.EmbeddingIndex._from_rows(rows, E, None, "cosine", None)
        probe = mixture(8, centres, args.spread, seed=99)
        sc = torch.mm(probe.float(), rows.float().T)
        thresholds = {h: float(torch.topk(sc, h, dim=1).values[:, -1].median()) for h in TARGETS}
        del sc
        for Q in QS:
            q = mixture(Q, centres, args.spread, seed=2 + Q).float()
            q16 = search.prepare_rows(q, "cosine")
            topk_ms, _ = host_timed(lambda: index.search(q, 128), args.repeats)
            for h, t in thresholds.items():
                rec = {"case": "resident", "N": N, "Q": Q, "target_hits": h, "min_score": t, "topk128_ms": topk_ms}
                if Q * h > args.max_total:
                    emit({**rec, "skipped": f"about {Q * h:.0e} hits"})
                    continue
                call, (lims, s, i) = host_timed(lambda: index.range_search(q, min_score=t), args.repeats)
                nnz = int(lims[-1])
                tau = search.range_thresholds("cosine", None, Q, t, None, index.device)
                kms = kernel_ms(index, q16[:search.QUERY_BATCH], tau[:search.QUERY_BATCH],
                                int(lims[min(Q, search.QUERY_BATCH)]), args.repeats)
                qb = min(Q, search.QUERY_BATCH)
                rec.update(call_ms=call, kernel_ms=kms, hits=nnz, hits_per_query=nnz / Q, hits_per_s=nnz / call * 1e3,
                           kernel_tflops=2 * qb * N * E / kms / 1e9,
                           kernel_share_of_989=2 * qb * N * E / kms / 1e9 / PEAK_TFLOPS)
                if N == sizes[0] and Q <= 1024:
                    tms, (tq, tj, ts) = host_timed(lambda: torch_path(rows, q16, t), 1)
                    rq = torch.repeat_interleave(torch.arange(Q, device="cuda"), lims.diff())
                    a = set(zip(rq.tolist(), i.tolist()))
                    b = set(zip(tq.tolist(), tj.tolist()))
                    s_all = torch.mm(q16.float(), rows.float().T) if Q * N <= 1 << 31 else None
                    diff = a ^ b
                    near = all(abs(float(s_all[x, y]) - t) <= 1e-3 for x, y in diff) if s_all is not None else None
                    rec.update(torch_ms=tms, torch_hits=len(b), torch_equal_outside_band=near,
                               torch_differ_in_band=len(diff))
                emit(rec)
        if N == sizes[0]:  # the streamed case: a sharded copy of these rows
            with tempfile.TemporaryDirectory() as d:
                with search.IndexWriter(d, E, "cosine") as w:
                    for r0 in range(0, N, 1 << 18):
                        w.add(rows[r0:r0 + (1 << 18)].float().cpu())
                sh = search.ShardedIndex.open(d)
                for Q in (1024,):
                    q = mixture(Q, centres, args.spread, seed=2 + Q).float()
                    for h in (10, 1000):
                        t = thresholds[h]
                        call, (lims, s, i) = host_timed(lambda: sh.range_search(q, min_score=t), args.repeats)
                        ref = index.range_search(q, min_score=t)
                        topk_ms, _ = host_timed(lambda: sh.search(q, 128), args.repeats)
                        emit({"case": "streamed", "N": N, "Q": Q, "target_hits": h, "min_score": t, "call_ms": call,
                              "hits": int(lims[-1]), "hits_per_s": int(lims[-1]) / call * 1e3, "topk128_ms": topk_ms,
                              "equal_to_resident": all(torch.equal(x, y) for x, y in zip(ref, (lims, s, i)))})
                del sh
            search.release_host_memory()
        del index, rows
        torch.cuda.empty_cache()
    emit({"gpu": query_gpu()})
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
