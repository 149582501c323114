"""Attention entry points alone, timed with CUDA events (GPU).

    ESMB200_LIB_PATH=/path/to/libesmb200.so python scripts/attention_bench.py [--seconds 1.5]

Shapes: esmb200_attention at the ESM-2 650M benchmark shape (B, T, H) = (256, 1024, 20) and the 3B one (16, 512, 40),
and esmb200_column_attention at the MSA Transformer's (B, R, C, H) = (1, 128, 512, 12).  Each shape is warmed up, then
launched back to back for at least --seconds; prints one JSON line with ms per launch and TFLOP/s
(4 B H T^2 64 FLOP of QK^T and PV, padding not discounted), the card, its power limit and the SM clock sampled after
the timed window.  The library comes from ESMB200_LIB_PATH (default: the in-tree build), so the same script measures
two builds.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from esm_b200 import _lib  # noqa: E402


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def smi(fields):
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return [x.strip() for x in out[0].split(",")] if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def time_launches(fn, seconds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    n = max(5, int(seconds * 1e3 / max(start.elapsed_time(stop), 1e-3)))
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
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("attention_bench.py needs a CUDA device")
    lib = _lib.load()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator(device="cpu").manual_seed(0)
    results = {}

    for B, T, H in [(256, 1024, 20), (16, 512, 40)]:
        E = 64 * H
        qkv = (torch.randn(B * T, 3 * E, generator=g) * 0.5).half().cuda()
        pad = torch.zeros(B, T, dtype=torch.uint8, device="cuda")
        ctx = torch.empty(B * T, E, dtype=torch.float16, device="cuda")
        scratch = torch.empty(lib.esmb200_attention_scratch_bytes(B, T), dtype=torch.uint8, device="cuda")
        fn = lambda: _lib.check(lib.esmb200_attention(P(qkv), P(pad), P(ctx), None, B, T, H, P(scratch), stream))
        ms, n, clk = time_launches(fn, args.seconds)
        results[f"attention_B{B}_T{T}_H{H}"] = {"ms": round(ms, 4), "launches": n, "sm_clock_mhz": clk,
                                                "tflops": round(4.0 * B * H * T * T * 64 / ms / 1e9, 1)}
        del qkv, ctx, scratch

    B, R, C, H = 1, 128, 512, 12
    E = 64 * H
    qkv = (torch.randn(B * R * C, 3 * E, generator=g) * 0.5).half().cuda()
    pad = torch.zeros(B * C, R, dtype=torch.uint8, device="cuda")
    ctx = torch.empty(B * R * C, E, dtype=torch.float16, device="cuda")
    scratch = torch.empty(lib.esmb200_attention_scratch_bytes(B * C, R), dtype=torch.uint8, device="cuda")
    fn = lambda: _lib.check(lib.esmb200_column_attention(P(qkv), P(pad), P(ctx), B, R, C, H, P(scratch), stream))
    ms, n, clk = time_launches(fn, args.seconds)
    results[f"column_attention_B{B}_R{R}_C{C}_H{H}"] = {"ms": round(ms, 4), "launches": n, "sm_clock_mhz": clk,
                                                        "tflops": round(4.0 * B * C * H * R * R * 64 / ms / 1e9, 1)}

    card = smi("name,power.limit,clocks.max.sm")
    print(json.dumps({"lib": os.path.abspath(_lib.LIB_PATH), "card": card[0] if card else None,
                      "power_limit_w": card[1] if card else None, "max_sm_clock_mhz": card[2] if card else None,
                      "results": results}))


if __name__ == "__main__":
    main()
