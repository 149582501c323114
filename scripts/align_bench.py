"""Developer tool (GPU box): embedding alignment (esm_b200.align) at user-sized shapes.

Workloads (seeded random embeddings, E = 1280, local mode, z-score on, the default penalties):
  * "1024x10": 1,024 queries x 10 hits, every length drawn uniformly from 100 ... 1,000 (a search_cli k = 10 run);
  * "L4000": 4 pairs at La = Lb = 4,000.
For each: pairs/s and cells/s (GCUPS) end to end (CUDA events around align_pairs, after one warm-up), the kernel time
split between the similarity kernels and the programme (esmb200_profile_* records, tag 23, in launch order: similarity,
statistics, z-score, programme, traceback per chunk), and the bytes per cell the design moves (S' written by the GEMM,
read twice by the statistics for rows and columns each, read and rewritten by the z-score, read by the programme; one
direction byte written) with the time that traffic implies at 3.35 TB/s.
Against: a plain-PyTorch path on the GPU (torch.matmul similarity of the same fp16 rows, the z-score in torch, and a
batched anti-diagonal loop computing the local score only, on the first --plain-pairs pairs), whose scores on our S'
are compared bit for bit; and the float32 numpy restatement (tests/align_refs.py) on the CPU for --oracle-pairs pairs.
Prints one JSON line per measurement and a final line with the card and its power limit (a read-only nvidia-smi
query).

    python scripts/align_bench.py [--plain-pairs 256] [--oracle-pairs 4] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from esm_b200 import _lib, align  # noqa: E402
from esm_b200.search import prepare_rows  # noqa: E402

E = 1280
PEAK_BYTES = 3.35e12  # H100 SXM data sheet, HBM3
BYTES_PER_CELL = 4 + 16 + 8 + 4 + 1  # GEMM store, statistics reads, z-score read + write, programme read, direction


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return f"unknown ({exc})"


def workload(name, g):
    if name == "1024x10":
        lq = torch.randint(100, 1001, (1024,), generator=g).tolist()
        lt = torch.randint(100, 1001, (10240,), generator=g).tolist()
        qs = [torch.randn(L, E, generator=g, dtype=torch.float32).half().cuda() for L in lq]
        ts = [torch.randn(L, E, generator=g, dtype=torch.float32).half().cuda() for L in lt]
        return [qs[p // 10] for p in range(10240)], ts
    qs = [torch.randn(4000, E, generator=g).half().cuda() for _ in range(4)]
    ts = [torch.randn(4000, E, generator=g).half().cuda() for _ in range(4)]
    return qs, ts


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b)


def kernel_split(qs, ts):
    lib = _lib.load()
    _lib.check(lib.esmb200_profile_enable(100000))
    align.align_pairs(qs, ts)
    torch.cuda.synchronize()
    import ctypes
    n = 100000
    tags, ms = (ctypes.c_int32 * n)(), (ctypes.c_float * n)()
    got = lib.esmb200_profile_read(tags, ms, n)
    lib.esmb200_profile_enable(0)
    rec = [ms[i] for i in range(got) if tags[i] == 23]
    names = ("similarity", "statistics", "zscore", "programme", "traceback")
    return {k: round(sum(rec[i::5]), 3) for i, k in enumerate(names)}


def plain_scores(qs, ts, o, e):
    """torch.matmul similarity, the z-score in torch, a batched anti-diagonal local programme: scores only."""
    P = len(qs)
    La, Lb = max(q.shape[0] for q in qs), max(t.shape[0] for t in ts)
    S = torch.full((P, La, Lb), float("-inf"), device="cuda")
    for p, (q, t) in enumerate(zip(qs, ts)):
        a, b = prepare_rows(q, "cosine"), prepare_rows(t, "cosine")
        s = torch.matmul(a, b.T).float()
        z = 0.5 * ((s - s.mean(1, keepdim=True)) / s.std(1, unbiased=False, keepdim=True) +
                   (s - s.mean(0, keepdim=True)) / s.std(0, unbiased=False, keepdim=True))
        S[p, :s.shape[0], :s.shape[1]] = z
    return dp_scores(S, o, e), S


def dp_scores(S, o, e):
    P, La, Lb = S.shape
    zero = torch.zeros((), device=S.device)
    H = torch.zeros(P, La + 1, Lb + 1, device=S.device)
    Ea = torch.full_like(H, float("-inf"))
    Fa = torch.full_like(H, float("-inf"))
    for d in range(2, La + Lb + 1):
        i = torch.arange(max(1, d - Lb), min(La, d - 1) + 1, device=S.device)
        j = d - i
        ev = torch.maximum(H[:, i, j - 1] - o, Ea[:, i, j - 1] - e)
        fv = torch.maximum(H[:, i - 1, j] - o, Fa[:, i - 1, j] - e)
        h = torch.maximum(torch.maximum(H[:, i - 1, j - 1] + S[:, i - 1, j - 1], ev), torch.maximum(fv, zero))
        H[:, i, j], Ea[:, i, j], Fa[:, i, j] = torch.nan_to_num(h, nan=0.0), ev, fv
    return H.flatten(1).max(1).values


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--plain-pairs", type=int, default=256)
    ap.add_argument("--oracle-pairs", type=int, default=4)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(d)

    g = torch.Generator().manual_seed(0)
    for name in ("1024x10", "L4000"):
        qs, ts = workload(name, g)
        cells = sum(q.shape[0] * t.shape[0] for q, t in zip(qs, ts))
        align.align_pairs(qs[:64], ts[:64])  # warm-up
        times = []
        for _ in range(3):
            res, ms = timed(lambda: align.align_pairs(qs, ts))
            times.append(ms)
        ms = sorted(times)[1]
        split = kernel_split(qs, ts)
        kern = sum(split.values())
        emit({"workload": name, "pairs": len(qs), "cells": cells, "ms": round(ms, 2),
              "pairs_per_s": round(len(qs) / ms * 1e3, 1), "gcups": round(cells / ms / 1e6, 2),
              "kernel_ms": split, "kernel_gcups": round(cells / kern / 1e6, 2),
              "bytes_per_cell": BYTES_PER_CELL, "traffic_bound_ms": round(cells * BYTES_PER_CELL / PEAK_BYTES * 1e3, 2)})
        n = min(args.plain_pairs, len(qs)) if name == "1024x10" else 1
        sub_q, sub_t = qs[:n], ts[:n]
        ours, sims = align.align_pairs(sub_q, sub_t, return_similarity=True)
        Sp = torch.full((n, max(q.shape[0] for q in sub_q), max(t.shape[0] for t in sub_t)), float("-inf"),
                        device="cuda")
        for p, s in enumerate(sims):
            Sp[p, :s.shape[0], :s.shape[1]] = s
        (pl_scores, _), pl_ms = timed(lambda: plain_scores(sub_q, sub_t, align.GAP_OPEN, align.GAP_EXTEND))
        same = dp_scores(Sp, align.GAP_OPEN, align.GAP_EXTEND)
        _, lib_ms = timed(lambda: align.align_pairs(sub_q, sub_t))
        sub_cells = sum(q.shape[0] * t.shape[0] for q, t in zip(sub_q, sub_t))
        emit({"workload": name, "against": "plain PyTorch", "pairs": n, "library_ms": round(lib_ms, 2),
              "plain_ms": round(pl_ms, 2), "speedup": round(pl_ms / lib_ms, 1),
              "plain_gcups": round(sub_cells / pl_ms / 1e6, 3),
              "scores_equal_on_our_S": bool(torch.equal(same.cpu(), torch.tensor([r.score for r in ours])))})
        if name == "1024x10":
            import align_refs
            k = min(args.oracle_pairs, len(qs))
            t0 = time.perf_counter()
            for s in sims[:k]:
                align_refs.align(s.cpu().numpy(), "local", align.GAP_OPEN, align.GAP_EXTEND)
            dt = time.perf_counter() - t0
            oc = sum(s.numel() for s in sims[:k])
            emit({"workload": name, "against": "numpy restatement (CPU)", "pairs": k,
                  "oracle_gcups": round(oc / dt / 1e9, 4), "library_gcups": round(cells / ms / 1e6, 2)})
        del qs, ts
        torch.cuda.empty_cache()
    emit({"gpu": query_gpu()})
    if args.out:
        with open(args.out, "w") as f:
            f.writelines(json.dumps(d) + "\n" for d in lines)


if __name__ == "__main__":
    main()
