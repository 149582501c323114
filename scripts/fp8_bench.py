"""fp16 vs fp8 precision on the bulk-embedding workload (esm2_t33_650M_UR50D, 256 sequences of 1024 tokens, seeded random
weights), alternated in one process:

  * end-to-end seq/s of model(tokens, repr_layers=[33]) per precision, `--rounds` alternations of `--steps` timed steps;
  * per-kernel times of the QKV, fc1 and fc2 GEMMs from the library's launch events (esmb200_profile_*), as TFLOP/s
    against the H100 SXM data-sheet dense peaks (989 fp16, 1979 fp8);
  * the error of the fp8 and fp16 outputs on the first `--check` sequences against the fp32-grade "fp32x3" mode;
  * the card's name and power limit, read in the same run.

    python scripts/fp8_bench.py [--batch 256] [--steps 3] [--warmup 1] [--rounds 2] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

PEAK = {"fp16": 989.0, "fp8": 1979.0}  # TFLOP/s, H100 SXM dense, data sheet (700 W)
T_QKV, T_FC1, T_FC2 = 1, 5, 6        # esmb200.h profile tags


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def tokens(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(4, 24, (B, T), generator=g)  # residue tokens of the ESM-1b alphabet
    t[:, 0], t[:, -1] = 0, 2                        # <cls> ... <eos>
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seq", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--check", type=int, default=8, help="sequences compared against the fp32x3 mode")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_bench.py measures on an H100; no CUDA device is available")
    from esm_b200 import _lib, pretrained
    lib = _lib.load()
    torch.manual_seed(0)
    model, _ = pretrained.load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=True)
    model = model.cuda().eval()
    L, E, F = model.num_layers, model.embed_dim, 4 * model.embed_dim
    tok = tokens(args.batch, args.seq, 1234).cuda()
    M = args.batch * args.seq
    flops = {T_QKV: 2.0 * M * 3 * E * E, T_FC1: 2.0 * M * F * E, T_FC2: 2.0 * M * E * F}
    names = {T_QKV: "qkv", T_FC1: "fc1", T_FC2: "fc2"}

    def step(t=tok):
        return model(t, repr_layers=[L])["representations"][L]

    result = {"card": card(), "workload": f"esm2_t33_650M_UR50D, {args.batch} x {args.seq} tokens, seeded random weights",
              "seq_per_s": {"fp16": [], "fp8": []}, "gemm": {}}
    for _ in range(args.rounds):
        for prec in ("fp16", "fp8"):
            model.set_precision(prec)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            result["seq_per_s"][prec].append(args.batch * args.steps / (e0.elapsed_time(e1) / 1e3))

    for prec in ("fp16", "fp8"):  # per-kernel pass, separate from the timed steps (events bracket every launch)
        model.set_precision(prec)
        step()
        torch.cuda.synchronize()
        n = 16 * L + 64
        _lib.check(lib.esmb200_profile_enable(n))
        step()
        torch.cuda.synchronize()
        tags, ms = (ctypes.c_int32 * n)(), (ctypes.c_float * n)()
        k = lib.esmb200_profile_read(tags, ms, n)
        _lib.check(lib.esmb200_profile_enable(0))
        for tag in (T_QKV, T_FC1, T_FC2):
            t = [ms[i] for i in range(k) if tags[i] == tag]
            mean_ms = sum(t) / len(t)
            tf = flops[tag] / (mean_ms / 1e3) / 1e12
            result["gemm"].setdefault(names[tag], {})[prec] = {
                "ms": round(mean_ms, 4), "tflops": round(tf, 1), "of_fp16_peak": round(tf / PEAK["fp16"], 3),
                "of_fp8_peak": round(tf / PEAK["fp8"], 3), "launches": len(t)}
    for g in result["gemm"].values():
        g["fp8_speedup"] = round(g["fp16"]["ms"] / g["fp8"]["ms"], 3)
    s16, s8 = max(result["seq_per_s"]["fp16"]), max(result["seq_per_s"]["fp8"])
    result["e2e_speedup"] = round(s8 / s16, 3)

    sub = tok[:args.check].contiguous()
    outs = {}
    for prec in ("fp32x3", "fp16", "fp8"):
        model.set_precision(prec)
        outs[prec] = step(sub).double()
    model.set_precision("fp16")
    ref = outs["fp32x3"]

    def err(a, b):
        return {"rel_fro": float((a - b).norm() / b.norm()), "max_abs": float((a - b).abs().max())}
    result["error"] = {"reference": "fp32x3 mode (fp32-grade)", "fp16_vs_ref": err(outs["fp16"], ref),
                       "fp8_vs_ref": err(outs["fp8"], ref), "fp8_vs_fp16": err(outs["fp8"], outs["fp16"])}
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
