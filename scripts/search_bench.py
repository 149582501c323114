"""Developer tool (GPU box): exact k-nearest-neighbour search (esm_b200.search) against the plain PyTorch path.

For each workload (Q queries, N database rows, width D, k) on seeded random unit rows in fp16 (cosine):
  * fused: esmb200_knn_search (search.knn; search_all for the all-against-all row), one wgmma GEMM + top-k kernel and
    a merge kernel, nothing but the [Q, k] results written;
  * plain: torch.mm(fp16, fp16, out_dtype=fp32) over database chunks of at most --chunk-bytes of fp32 scores, then
    torch.topk per chunk and a final topk over the chunks' candidates;
  * milliseconds (CUDA events around synchronised work, the median of --repeats after one warm-up), 2 Q N D FLOP over
    time, database bytes (N D 2) over time, which bound limits it (the larger of FLOP / 989e12 and bytes / 3.35e12),
    and the share of queries whose k indices the two paths return identically.
Prints one JSON line per workload and a final line with the card and its power limit (a read-only nvidia-smi query).

    python scripts/search_bench.py [--repeats 3] [--only 0,2] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esm_b200 import search  # noqa: E402

WORKLOADS = [  # Q, N, D, k, all-against-all
    (1, 570_000, 1280, 10, False),
    (1024, 570_000, 1280, 10, False),
    (1024, 570_000, 1280, 128, False),
    (4096, 5_000_000, 1280, 10, False),
    (100_000, 100_000, 1280, 10, True),
    (64, 570_000, 5120, 10, False),
]
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12  # H100 SXM data sheet: dense fp16, HBM3


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid; say what is missing
        return f"nvidia-smi unavailable: {e}"


def unit_rows(n, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, D), dtype=torch.float16, device="cuda")
    for r0 in range(0, n, 1 << 18):
        r1 = min(n, r0 + (1 << 18))
        x = torch.randn((r1 - r0, D), generator=g, device="cuda")
        out[r0:r1] = (x / x.norm(dim=1, keepdim=True)).half()
    return out


def timed(fn, repeats):
    fn()
    times = []
    for _ in range(repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        out = fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    return sorted(times)[len(times) // 2], out


def plain(a, x, k, self_rows, chunk_bytes):
    Q, N = a.shape[0], x.shape[0]
    qstep = Q if not self_rows else min(Q, 8192)
    best_s, best_i = [], []
    for q0 in range(0, Q, qstep):
        q1 = min(Q, q0 + qstep)
        rows = max(256, chunk_bytes // (4 * (q1 - q0)))
        cs, ci = [], []
        for n0 in range(0, N, rows):
            n1 = min(N, n0 + rows)
            sc = torch.mm(a[q0:q1], x[n0:n1].T, out_dtype=torch.float32)
            if self_rows and n0 < q1 and q0 < n1:
                i = torch.arange(max(q0, n0), min(q1, n1), device=a.device)
                sc[i - q0, i - n0] = float("-inf")
            v, j = torch.topk(sc, min(k, n1 - n0), dim=1)
            cs.append(v)
            ci.append(j + n0)
        v, j = torch.topk(torch.cat(cs, 1), k, dim=1)
        best_s.append(v)
        best_i.append(torch.cat(ci, 1).gather(1, j))
    return torch.cat(best_s), torch.cat(best_i)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--only", type=str, default=None, help="comma-separated workload numbers")
    ap.add_argument("--chunk-bytes", type=int, default=2_400_000_000)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("search_bench needs a CUDA device")
    gpu = query_gpu()
    only = None if args.only is None else {int(v) for v in args.only.split(",")}
    lines = []
    for w, (Q, N, D, k, self_rows) in enumerate(WORKLOADS):
        if only is not None and w not in only:
            continue
        x = unit_rows(N, D, seed=w)
        a = x if self_rows else unit_rows(Q, D, seed=1000 + w)
        index = search.EmbeddingIndex._from_rows(x, D, None, "cosine", None)
        fused = (lambda: index.search_all(k)) if self_rows else (lambda: search.knn(a, x, k))
        t_f, (fs, fi) = timed(fused, args.repeats)
        t_p, (ps, pi) = timed(lambda: plain(a, x, k, self_rows, args.chunk_bytes), args.repeats)
        same = float((fi == pi).all(1).float().mean())
        flop, nbytes = 2.0 * Q * N * D, 2.0 * N * D
        row = {"workload": w, "Q": Q, "N": N, "D": D, "k": k, "all_against_all": self_rows,
               "fused_ms": round(t_f, 3), "plain_ms": round(t_p, 3), "speedup": round(t_p / t_f, 2),
               "fused_tflops": round(flop / t_f / 1e9, 1), "fused_db_gbps": round(nbytes / t_f / 1e6, 1),
               "bound": "flops" if flop / PEAK_FLOPS > nbytes / PEAK_BYTES else "hbm",
               "share_of_bound": round(max(flop / PEAK_FLOPS, nbytes / PEAK_BYTES) / (t_f / 1e3), 3),
               "same_indices": round(same, 4), "gpu": gpu}
        print(json.dumps(row), flush=True)
        lines.append(row)
        del x, a, index, fs, fi, ps, pi
        torch.cuda.empty_cache()
    print(json.dumps({"gpu": gpu}), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            for row in lines:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
