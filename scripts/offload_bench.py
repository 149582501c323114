"""Streamed (cpu_offload) against resident forward at the ESM-2 15B shape: E 5120, 40 heads of 128, F 20480, 48 layers.

    python scripts/offload_bench.py [--distinct] [--rounds 3]

By default the model's ModuleList holds one seeded layer 48 times: host and device memory stay small, and the streamed
forward copies 48 layers' packed matrices exactly as 48 distinct layers would. --distinct builds 48 different fp16
layers instead (about 30 GB of parameters plus the 30 GB pinned arena on the host). The resident forward always runs
the repeated layer resident in HBM (48 distinct resident layers do not fit an 80 GB card).

For 4, 16 and 64 x 1024 tokens the resident forward, the streamed forward and one pinned host-to-device copy of a
layer's packed matrices are timed with device events, alternated for --rounds rounds in one process (medians
reported). A second shape, 650M (33 layers) at 64 x 1024 tokens, is where streaming should cost nothing. Prints one
JSON line per shape and batch size:
    streamed_over_resident   streamed / resident
    overlap_efficiency       streamed / max(resident, n_layers * copy)
    peak_device_gb           torch.cuda.max_memory_allocated() over one streamed forward (the library's own
                             allocations, q/k/v biases of 61 KB per 15B layer, are not counted)
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from esm_b200 import ESM2, _lib  # noqa: E402
from esm_b200.model import TransformerLayer  # noqa: E402

DEV = torch.device("cuda", 0)


def card():
    info = {"device": torch.cuda.get_device_name(DEV)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"] = [s.strip() for s in q.split(",")][:2]
    except Exception as e:  # reported, not fatal: the timings stand without it
        info["power_limit"] = f"unavailable ({e})"
    return info


def seeded_layer(E, H, seed, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    layer = TransformerLayer(E, 4 * E, H)
    with torch.no_grad():
        for name, p in layer.named_parameters():
            if name.endswith("weight") and p.dim() == 2:
                p.copy_(torch.randn(p.shape, generator=g) * p.shape[1] ** -0.5)
            elif "layer_norm" in name and name.endswith("weight"):
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
    return layer.to(dtype)


def model(E, H, n_layers, distinct=False):
    """ESM2 with seeded weights; the layer list is one layer repeated n_layers times unless `distinct`"""
    torch.manual_seed(0)  # the modules' default initialisation (LM head, LayerNorms): the same in every model built here
    m = ESM2(num_layers=1, embed_dim=E, attention_heads=H)
    with torch.no_grad():
        g = torch.Generator().manual_seed(1)
        m.embed_tokens.weight.copy_(torch.randn(m.embed_tokens.weight.shape, generator=g))
    if distinct:
        m.layers = nn.ModuleList([seeded_layer(E, H, 100 + i, torch.float16) for i in range(n_layers)])
    else:
        m.layers = nn.ModuleList([seeded_layer(E, H, 100)] * n_layers)
    m.num_layers = n_layers
    return m.eval()


def tokens(B, T, seed=7):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(4, 24, (B, T), generator=g)
    t[:, 0], t[:, -1] = 0, 2
    return t.to(DEV)


def timed(fn, reps=1):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def run_shape(name, E, H, n_layers, batches, rounds, distinct, T=1024):
    lib = _lib.load()
    packed = lib.esmb200_layer_packed_bytes(E, H, 4 * E, 0)
    streamed = model(E, H, n_layers, distinct).cpu_offload(DEV)
    host = torch.empty(packed, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(packed, dtype=torch.uint8, device=DEV)
    peak = {}
    with torch.no_grad():
        for B in batches:  # warm-up and peak memory of the streamed forward alone
            tok = tokens(B, T)
            streamed(tok)
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats(DEV)
            streamed(tok)
            torch.cuda.synchronize()
            peak[B] = torch.cuda.max_memory_allocated(DEV) / 1e9
        resident = model(E, H, n_layers).to(DEV)
        results = []
        for B in batches:
            tok = tokens(B, T)
            same = None if distinct else torch.equal(resident(tok)["logits"], streamed(tok)["logits"])
            torch.cuda.synchronize()
            t_res, t_st, t_copy = [], [], []
            for _ in range(rounds):
                t_res.append(timed(lambda: resident(tok)))
                t_st.append(timed(lambda: streamed(tok)))
                t_copy.append(timed(lambda: dst.copy_(host, non_blocking=True), reps=10))
            r, s, c = statistics.median(t_res), statistics.median(t_st), statistics.median(t_copy)
            results.append({
                "shape": name, "layers": n_layers, "distinct": distinct, "tokens": B * T, "batch": [B, T],
                "resident_ms": round(r, 2), "streamed_ms": round(s, 2), "copy_ms": round(c, 3),
                "h2d_gb_s": round(packed / c / 1e6, 2),
                "streamed_over_resident": round(s / r, 4),
                "overlap_efficiency": round(s / max(r, n_layers * c), 4),
                "peak_device_gb": round(peak[B], 3), "logits_equal": same,
                "rounds": {"resident_ms": [round(v, 2) for v in t_res], "streamed_ms": [round(v, 2) for v in t_st],
                           "copy_ms": [round(v, 3) for v in t_copy]},
            })
    del resident, streamed
    return results


def main():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--distinct", action="store_true", help="48 different fp16 layers (needs ~65 GB of free host memory)")
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--batches", type=int, nargs="+", default=[4, 16, 64], help="sequences of 1024 tokens")
    p.add_argument("--skip-650M", action="store_true")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("offload_bench.py measures on a CUDA (sm_90a) device; none is available")
    info = card()
    for r in run_shape("15B", 5120, 40, 48, args.batches, args.rounds, args.distinct):
        print(json.dumps({**r, **info}), flush=True)
    if not args.skip_650M:
        for r in run_shape("650M", 1280, 20, 33, [64], args.rounds, False):
            print(json.dumps({**r, **info}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
