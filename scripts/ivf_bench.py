"""Developer tool (GPU box): the inverted-file index (esm_b200.search.IVFIndex) against exact search (EmbeddingIndex).

The data is synthetic: a seeded mixture of --centres clusters on the unit sphere (a centre plus Gaussian noise of norm
about --spread, normalised), E = 1280, fp16 cosine rows; the queries are drawn from the same mixture. Recall on real
ESM embeddings is not measured by this tool. For each N (1 M rows with nlist 1024, 10 M rows with nlist 4096):
  * build: k-means training (train_rows = 256 nlist, 20 iterations) and list building, seconds (host clock around
    synchronised work);
  * search: milliseconds per call (CUDA events, median of --repeats after a warm-up) for Q = 1, 1,024 and 8,192,
    k = 10 and nprobe in {8, 32, 128, nlist}, and for the exact search on the same rows;
  * recall@10 against the exact search, and at nprobe = nlist the share of queries whose indices equal the exact ones;
  * a torch.profiler breakdown of one call (N = 10 M, Q = 1,024, nprobe = 32) into the coarse step, the grouping
    kernels, the list scan and the merge.
Prints one JSON line per measurement and a final line with the card and its power limit (a read-only nvidia-smi
query), and writes them to --out if given.

    python scripts/ivf_bench.py [--repeats 3] [--sizes 1000000,10000000] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esm_b200 import search  # noqa: E402

E = 1280
NLIST = {1_000_000: 1024, 10_000_000: 4096}
QS = (1, 1024, 8192)


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid; say what is missing
        return f"nvidia-smi unavailable: {e}"


def mixture(n, centres, spread, seed):
    """fp16 unit rows [n, E] on the GPU: centre + noise of norm about `spread`, normalised (as prepare_rows does it,
    in float64 then rounded), generated in chunks so that no fp32 copy of the whole set exists."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((n, E), dtype=torch.float16, device="cuda")
    for r0 in range(0, n, 1 << 18):
        r1 = min(n, r0 + (1 << 18))
        lab = torch.randint(0, centres.shape[0], (r1 - r0,), generator=g, device="cuda")
        x = centres[lab].double() + spread * torch.randn((r1 - r0, E), generator=g, device="cuda",
                                                         dtype=torch.float64) / E ** 0.5
        out[r0:r1] = (x / x.norm(dim=1, keepdim=True)).half()
    return out


def timed(fn, repeats):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def breakdown(ivf, q, nprobe):
    """Kernel milliseconds of one search call by stage, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    ivf.search(q, 10, nprobe=nprobe)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ivf.search(q, 10, nprobe=nprobe)
        torch.cuda.synchronize()
    stages = {"coarse": 0.0, "grouping": 0.0, "scan": 0.0, "merge": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        name, ms = ev.key, ev.device_time_total / 1e3
        if "knn_topk_kernel" in name:
            stages["scan" if "true>" in name.replace(" ", "") or "Lb1EEE" in name else "coarse"] += ms
        elif "ivf_" in name:
            stages["grouping"] += ms
        elif "knn_merge_kernel" in name:
            stages["merge" if "true>" in name.replace(" ", "") or "Lb1EEE" in name else "coarse"] += ms
        else:
            stages["other"] += ms
    return {k: round(v, 3) for k, v in stages.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--sizes", type=str, default="1000000,10000000")
    ap.add_argument("--centres", type=int, default=20000)
    ap.add_argument("--spread", type=float, default=1.0)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ivf_bench needs a CUDA device")
    g = torch.Generator(device="cuda").manual_seed(0)
    centres = torch.nn.functional.normalize(torch.randn((args.centres, E), generator=g, device="cuda"), dim=1)
    for N in (int(s) for s in args.sizes.split(",")):
        nlist = NLIST.get(N, max(1, int(N ** 0.5)))
        rows = mixture(N, centres, args.spread, seed=1)
        exact = search.EmbeddingIndex._from_rows(rows, E, None, "cosine", None)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ivf = search.IVFIndex.from_index(exact, nlist=nlist)
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        sizes = (ivf.offsets[1:] - ivf.offsets[:-1]).float()
        emit({"N": N, "nlist": nlist, "build_s": round(build_s, 3), "train_rows": ivf.params["train_rows"],
              "iters": ivf.params["iters"], "list_rows_max": int(sizes.max()), "list_rows_mean": float(sizes.mean()),
              "empty_lists": int((sizes == 0).sum())}, args.out)
        for Q in QS:
            q = mixture(Q, centres, args.spread, seed=2 + Q).float()
            ex_ms = timed(lambda: exact.search(q, 10), args.repeats)
            _, want = exact.search(q, 10)
            emit({"N": N, "Q": Q, "k": 10, "exact_ms": round(ex_ms, 3)}, args.out)
            for nprobe in (8, 32, 128, nlist):
                ms = timed(lambda: ivf.search(q, 10, nprobe=nprobe), args.repeats)
                _, got = ivf.search(q, 10, nprobe=nprobe)
                recall = sum(len(set(a) & set(b)) for a, b in zip(want.tolist(), got.tolist())) / want.numel()
                rec = {"N": N, "nlist": nlist, "Q": Q, "k": 10, "nprobe": nprobe, "ivf_ms": round(ms, 3),
                       "exact_ms": round(ex_ms, 3), "speedup": round(ex_ms / ms, 2), "recall@10": round(recall, 4),
                       "lists_share": round(nprobe / nlist, 4)}
                if nprobe == nlist:
                    rec["identical_share"] = float((got == want).all(1).float().mean())
                emit(rec, args.out)
            if N == 10_000_000 and Q == 1024:
                emit({"N": N, "Q": Q, "nprobe": 32, "breakdown_ms": breakdown(ivf, q, 32)}, args.out)
            del q
        del ivf, exact, rows
        torch.cuda.empty_cache()
    emit({"gpu": query_gpu()}, args.out)


if __name__ == "__main__":
    main()
