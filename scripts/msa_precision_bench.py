"""Cost of the MSA Transformer's fp32x3 precision against fp16, timed with CUDA events (GPU).

    python scripts/msa_precision_bench.py [--seconds 1.5] [--rounds 3]

The BASELINE.json configs[4] shape: esm_msa1b width (12 layers, E = 768, H = 12, F = 3072), seeded random weights,
one unpadded 128 x 512 alignment.  Two workloads: the forward (`model(tokens)`, logits) and `predict_contacts` (row
attention maps of every layer + contact head).  The two precisions alternate for --rounds rounds; every (workload,
precision) window is warmed up and then repeated for at least --seconds.  Prints one JSON line with ms per call per
round, the median, the fp32x3 / fp16 ratio, the card, its power limit and the SM clock sampled after each window.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
from argparse import Namespace

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from esm_b200 import MSATransformer  # noqa: E402


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return [x.strip() for x in out[0].split(",")] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def time_calls(fn, seconds):
    fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    n = max(3, int(seconds * 1e3 / max(start.elapsed_time(stop), 1e-3)))
    start.record()
    for _ in range(n):
        fn()
    stop.record()
    stop.synchronize()
    clocks = smi("clocks.sm")
    return start.elapsed_time(stop) / n, n, (clocks[0] if clocks else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.5, help="least duration of each timed window")
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("msa_precision_bench.py needs a CUDA device")
    torch.manual_seed(0)
    model = MSATransformer(Namespace(layers=12, embed_dim=768, ffn_embed_dim=3072, attention_heads=12,
                                     max_positions=1024, embed_positions_msa=True)).eval().cuda()
    g = torch.Generator().manual_seed(1)
    tokens = torch.randint(4, 24, (1, 128, 512), generator=g)
    tokens[:, :, 0] = 0  # <cls>
    tokens = tokens.cuda()
    work = {"forward": lambda: model(tokens), "predict_contacts": lambda: model.predict_contacts(tokens)}
    res = {w: {p: [] for p in ("fp16", "fp32x3")} for w in work}
    clocks = []
    for _ in range(args.rounds):
        for prec in ("fp16", "fp32x3"):
            model.set_precision(prec)
            for w, fn in work.items():
                ms, n, clk = time_calls(fn, args.seconds)
                res[w][prec].append({"ms": round(ms, 3), "calls": n})
                clocks.append(clk)
    summary = {}
    for w in work:
        med = {p: statistics.median(r["ms"] for r in res[w][p]) for p in ("fp16", "fp32x3")}
        summary[w] = {"median_ms": med, "ratio": round(med["fp32x3"] / med["fp16"], 3)}
    card = smi("name,power.limit,clocks.max.sm")
    print(json.dumps({"shape": "1 x 128 x 512, 12 layers, E=768", "card": card[0] if card else None,
                      "power_limit_w": card[1] if card else None, "max_sm_clock_mhz": card[2] if card else None,
                      "sm_clock_mhz_after_windows": clocks, "summary": summary, "rounds": res}))


if __name__ == "__main__":
    main()
