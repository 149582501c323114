"""Developer tool (GPU box): streamed search over a sharded on-disk index (esm_b200.search.ShardedIndex) against the
resident EmbeddingIndex on the same rows.

  * writes seeded random unit rows (E = 1280, cosine) to a sharded index in a temporary directory, as many as
    --max-rows, 40% of the free RAM (the page cache must hold it) and 40% of the free disk allow, prints all three,
    and reads the files once to warm the page cache (caches are never dropped);
  * the separate rates of the streamed path: memory map to pinned slot (the refill threads), pinned slot to device
    (the copy stream), and the kernels over the whole database from device memory (CUDA events);
  * per (Q, k) with Q in {1, 1024, 8192} and k in {10, 128}: end-to-end ms and rows/s of ShardedIndex.search
    (host clock around the synchronised call, the median of --repeats after one warm-up), 2 Q N D FLOP over the
    end-to-end and kernel times, which of the three rates bounds the call, the resident EmbeddingIndex.search on the
    same rows (where they fit on the device) and the share of queries whose indices the two return identically;
  * the fixed cost of a call: registering and unregistering the page-locked ring, and a whole Q = 1 call on a
    65,536-row database (one chunk), first with the ring registered by the call, then with it kept from the last;
  * the streamed search at Q = 1 (the kernels negligible) with 4, 8 and 16 refill threads;
  * with --parent-tree (a checkout of the parent commit with its library built), scripts/search_bench.py's resident
    workloads alternately from that tree and from this one, --ab-rounds times each, to show what the kernel change
    costs the resident path.
Prints one JSON line per measurement, with the card and its power limit (a read-only nvidia-smi query).

    python scripts/search_stream_bench.py [--max-rows 8000000] [--repeats 3] [--parent-tree DIR] [--out r.jsonl]
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from esm_b200 import search  # noqa: E402

E = 1280
QS, KS = (1, 1024, 8192), (10, 128)


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid; say what is missing
        return f"nvidia-smi unavailable: {e}"


def free_ram_bytes():
    with open("/proc/meminfo") as f:
        info = {l.split(":")[0]: int(l.split()[1]) * 1024 for l in f}
    return info.get("MemAvailable", info.get("MemFree", 0))


def emit(row, lines):
    print(json.dumps(row), flush=True)
    lines.append(row)


def build_index(path, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    with search.IndexWriter(path, E, "cosine", shard_rows=1 << 20) as w:
        for r0 in range(0, N, 1 << 18):
            w.add(torch.randn((min(N, r0 + (1 << 18)) - r0, E), generator=g, device="cuda"))
    return search.ShardedIndex.open(path)


def refill_rate(index, rows):
    """Bytes per second from the memory maps into a registered (pinned) slot, over the whole database."""
    ring = search._HostRing(rows, index.padded_dim, False)
    try:
        t0 = time.perf_counter()
        with ThreadPoolExecutor(search.REFILL_THREADS) as pool:
            for g0 in range(0, len(index), rows):
                g1 = min(len(index), g0 + rows)
                index._read_parallel(pool, g0, g1, ring.rows[0].numpy(), None)
        dt = time.perf_counter() - t0
    finally:
        ring.release()
    return len(index) * index.padded_dim * 2 / dt


def h2d_rate(rows, D, repeats=20):
    ring = search._HostRing(rows, D, False)
    try:
        dst = torch.empty((rows, D), dtype=torch.float16, device="cuda")
        dst.copy_(ring.rows[0], non_blocking=True)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for _ in range(repeats):
            dst.copy_(ring.rows[0], non_blocking=True)
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e)
    finally:
        torch.cuda.synchronize()
        ring.release()
    return repeats * rows * D * 2 / (ms / 1e3)


def kernel_ms(q, x, k, chunk, sms):
    """CUDA-event time of the accumulate launches over the device-resident rows x in chunks, plus the decode."""
    Q = q.shape[0]
    keys = torch.zeros((Q, k), dtype=torch.int64, device="cuda")
    scratch = torch.empty(search.scratch_bytes(Q, Q, k, sms), dtype=torch.uint8, device="cuda")
    s_out = torch.empty((Q, k), device="cuda")
    i_out = torch.empty((Q, k), dtype=torch.int64, device="cuda")

    def run():
        keys.zero_()
        for g0 in range(0, x.shape[0], chunk):
            g1 = min(x.shape[0], g0 + chunk)
            for b0 in range(0, Q, search.QUERY_BATCH):
                b1 = min(Q, b0 + search.QUERY_BATCH)
                search.knn_accumulate(q[b0:b1], x[g0:g1], g0, k, keys[b0:b1], scratch, None, 1.0, -1,
                                      search.choose_splits(b1 - b0, g1 - g0, sms))
        search.knn_decode(keys, s_out, i_out)

    run()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    run()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), i_out


def ring_ms(rows, D, repeats=3):
    """Host ms to allocate and register the call's page-locked ring, and to unregister it (median of repeats)."""
    make, free = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        ring = search._HostRing(rows, D, False)
        t1 = time.perf_counter()
        ring.release()
        del ring
        free.append((time.perf_counter() - t1) * 1e3)
        make.append((t1 - t0) * 1e3)
    return statistics.median(make), statistics.median(free)


def timed_host(fn, repeats):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times), out


def ab_resident(parent_tree, rounds, gpu, lines):
    """scripts/search_bench.py's fused workloads 1-3, alternately from a built checkout of the parent commit and from
    this tree."""
    trees = {"parent": os.path.abspath(parent_tree), "new": ROOT}
    for r in range(rounds):
        for name in ("parent", "new") if r % 2 == 0 else ("new", "parent"):
            bench = os.path.join(trees[name], "scripts", "search_bench.py")
            env = {k: v for k, v in os.environ.items() if k != "ESMB200_LIB_PATH"}
            out = subprocess.run([sys.executable, bench, "--only", "1,2,3", "--repeats", "5"], env=env,
                                 capture_output=True, text=True, timeout=1800)
            if out.returncode != 0:
                raise SystemExit(f"search_bench.py failed on the {name} library:\n{out.stderr[-3000:]}")
            for line in out.stdout.splitlines():
                row = json.loads(line)
                if "workload" in row:
                    emit({"ab": name, "round": r, "workload": row["workload"], "Q": row["Q"], "N": row["N"],
                          "k": row["k"], "fused_ms": row["fused_ms"], "same_indices": row["same_indices"], "gpu": gpu},
                         lines)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-rows", type=int, default=8_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--parent-tree", type=str, default=None)
    ap.add_argument("--ab-rounds", type=int, default=2)
    ap.add_argument("--out", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("search_stream_bench needs a CUDA device")
    gpu = query_gpu()
    lines = []
    tmp = tempfile.mkdtemp(prefix="search_stream_bench_")
    try:
        row_bytes = search.padded_dim(E) * 2
        ram, disk = free_ram_bytes(), shutil.disk_usage(tmp).free
        N = max(1 << 18, min(args.max_rows, int(0.4 * ram) // row_bytes, int(0.4 * disk) // row_bytes))
        emit({"free_ram_gb": round(ram / 1e9, 1), "free_disk_gb": round(disk / 1e9, 1), "N": N,
              "db_gb": round(N * row_bytes / 1e9, 2), "gpu": gpu}, lines)
        t0 = time.perf_counter()
        index = build_index(os.path.join(tmp, "db"), N, seed=0)
        emit({"build_s": round(time.perf_counter() - t0, 1), "shards": len(index.shards)}, lines)
        D, sms = index.padded_dim, torch.cuda.get_device_properties(0).multi_processor_count
        slot_rows = search.MAX_SLOT_BYTES // (D * 2) // search.TILE * search.TILE
        warm = refill_rate(index, slot_rows)  # the first pass warms the page cache
        refill = refill_rate(index, slot_rows)
        h2d = h2d_rate(slot_rows, D)
        emit({"rate": "map_to_pinned", "first_pass_gbps": round(warm / 1e9, 2), "gbps": round(refill / 1e9, 2),
              "threads": search.REFILL_THREADS, "slot_mb": round(slot_rows * D * 2 / 1e6, 1)}, lines)
        emit({"rate": "pinned_to_device", "gbps": round(h2d / 1e9, 2)}, lines)
        # the fixed cost of every call: the ring registered and released, and a whole call on a one-chunk database
        make, free = ring_ms(slot_rows, D)
        small = build_index(os.path.join(tmp, "small"), 65_536, seed=2)
        q1 = torch.randn((1, E), generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
        search.release_host_memory()
        t0 = time.perf_counter()
        small.search(q1, 10)  # registers the ring
        torch.cuda.synchronize()
        t_first = (time.perf_counter() - t0) * 1e3
        t_small, _ = timed_host(lambda: small.search(q1, 10), max(args.repeats, 5))
        emit({"per_call": "ring", "register_ms": round(make, 1), "unregister_ms": round(free, 1),
              "slot_mb": round(slot_rows * D * 2 / 1e6, 1), "slots": search.RING_SLOTS,
              "small_db_rows": len(small), "small_db_q1_first_ms": round(t_first, 2),
              "small_db_q1_ms": round(t_small, 2),
              "chunks_at_N": -(-N // slot_rows)}, lines)
        # the resident rows, read from the same files
        free = torch.cuda.mem_get_info()[0]
        x = None
        if N * row_bytes < 0.45 * free:
            x = torch.empty((N, D), dtype=torch.float16, device="cuda")
            buf = torch.empty((slot_rows, D), dtype=torch.float16)
            for g0 in range(0, N, slot_rows):
                g1 = min(N, g0 + slot_rows)
                index.read_rows(g0, g1, buf.numpy()[: g1 - g0])
                x[g0:g1] = buf[: g1 - g0].to("cuda")
            resident = search.EmbeddingIndex._from_rows(x, E, None, "cosine", None)
        g = torch.Generator(device="cuda").manual_seed(1)
        for Q in QS:
            queries = torch.randn((Q, E), generator=g, device="cuda")
            for k in KS:
                t_e2e, (s, i) = timed_host(lambda: index.search(queries, k), args.repeats)
                flop = 2.0 * Q * N * D
                row = {"Q": Q, "k": k, "N": N, "e2e_ms": round(t_e2e, 2), "rows_per_s": round(N / t_e2e * 1e3),
                       "e2e_tflops": round(flop / t_e2e / 1e9, 1)}
                times = {"map_to_pinned": N * D * 2 / refill * 1e3, "pinned_to_device": N * D * 2 / h2d * 1e3}
                if x is not None:
                    chunk = min(slot_rows, -(-N // 256) * 256)
                    t_k, ik = kernel_ms(search.prepare_rows(queries, "cosine"), x, k, chunk, sms)
                    times["kernels"] = t_k
                    t_r, (sr, ir) = timed_host(lambda: resident.search(queries, k), args.repeats)
                    row.update({"kernel_ms": round(t_k, 2), "kernel_tflops": round(flop / t_k / 1e9, 1),
                                "resident_ms": round(t_r, 2), "stream_over_resident": round(t_r / t_e2e, 3),
                                "same_indices": round(float((i == ir).all(1).float().mean()), 4),
                                "kernel_same_indices": round(float((ik == ir).all(1).float().mean()), 4)})
                row["bound"] = max(times, key=times.get)
                row["bound_ms"] = {n: round(v, 1) for n, v in times.items()}
                row["gpu"] = gpu
                emit(row, lines)
                del s, i
        del x
        torch.cuda.empty_cache()
        q1 = torch.randn((1, E), generator=g, device="cuda")
        default_threads = search.REFILL_THREADS
        for threads in (4, 8, 16):
            search.REFILL_THREADS = threads
            t, _ = timed_host(lambda: index.search(q1, 10), args.repeats)
            emit({"Q": 1, "k": 10, "refill_threads": threads, "e2e_ms": round(t, 2),
                  "db_gbps": round(N * D * 2 / t / 1e6, 2), "gpu": gpu}, lines)
        search.REFILL_THREADS = default_threads
        if args.parent_tree:
            ab_resident(args.parent_tree, args.ab_rounds, gpu, lines)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        with open(args.out, "a") as f:
            for row in lines:
                f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
