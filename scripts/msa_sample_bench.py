"""Developer tool (GPU box): alignment sampling (esm_b200.sampling.msa_gibbs) with the MSA Transformer
(esm_msa1b_t12_100M_UR50S architecture: 12 layers x 768 x 12 heads, seeded random weights), 8 chains, every entry
designable and a block of 5 % of the entries, on 64 x 256 and 128 x 512 alignments (rows x columns with <cls>). All
chains run in one chunk, so each step is one axial-stack call on 8 alignments.

Prints one JSON line: the card and its power limit (a read-only nvidia-smi query) and, per shape,
  * seconds per step: msa_gibbs over --sweeps sweeps, device events around synchronised work;
  * the same number of esmb200_axial_stack_forward calls on a batch of the same shape ([8, R, C, 768]), timed in the
    same run, alternating with msa_gibbs, and the step-to-stack ratio (best of --repeats for each);
  * the sampler kernels' time per step from the library's profiler (tag 20: the order kernel and both kernels of
    esmb200_sample_rows), in a separate profiled run, and their share of a step.

    python scripts/msa_sample_bench.py [--sweeps 1] [--repeats 3] [--precision fp16] [--out results.jsonl]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TAG_SAMPLING = 20
SHAPES = [(64, 256), (128, 512)]


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid; say what is missing
        return f"nvidia-smi unavailable: {e}"


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3


def alignment(model, R, C, seed):
    """A random alignment [1, R, C]: <cls>, then amino acids with 10 % gaps."""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(4, 24, (1, R, C), generator=g)
    t[torch.rand((1, R, C), generator=g) < 0.1] = model.alphabet.get_idx("-")
    t[:, :, 0] = model.cls_idx
    return t


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--chains", type=int, default=8)
    p.add_argument("--block-fraction", type=float, default=0.05)
    p.add_argument("--sweeps", type=int, default=1)
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--precision", choices=["fp16", "fp32x3"], default="fp16")
    p.add_argument("--out", type=str, default=None, help="also append the JSON line to this file")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("msa_sample_bench.py measures on a CUDA (sm_90a) GPU; none is available")
    from esm_b200 import _lib, pretrained, sampling
    from esm_b200.msa import run_axial_stack

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, _ = pretrained.load_msa_model_and_alphabet("esm_msa1b_t12_100M_UR50S", allow_random_init=True,
                                                          device="cuda")
    model = model.eval().cuda()
    if a.precision != "fp16":
        model.set_precision(a.precision)
    lib = _lib.load()
    rec = {"gpu": query_gpu(), "model": "esm_msa1b_t12_100M_UR50S (random init)", "precision": a.precision,
           "chains": a.chains, "shapes": []}
    with torch.no_grad():
        for R, C in SHAPES:
            x0 = alignment(model, R, C, seed=R + C).cuda()
            n = R * (C - 1)
            k = max(1, round(a.block_fraction * n))
            steps = a.sweeps * -(-n // k)
            kw = dict(chains=a.chains, sweeps=a.sweeps, block=k, seed=1, max_tokens=a.chains * R * C)
            xb = model._stack_unpadded(x0.expand(a.chains, R, C).contiguous())  # [chains, R, C, E] fp32

            def stack_calls():
                for _ in range(steps):
                    run_axial_stack(list(model.layers), xb)

            sampling.msa_gibbs(model, x0, **kw)  # warm-up: every shape of the timed window
            stack_calls()
            step_s, stack_s = [], []
            for _ in range(a.repeats):
                step_s.append(timed(lambda: sampling.msa_gibbs(model, x0, **kw)) / steps)
                stack_s.append(timed(stack_calls) / steps)
            # profiled run of its own: the library's per-launch events around every kernel
            n_rec = 200000
            lib.esmb200_profile_enable(n_rec)
            sampling.msa_gibbs(model, x0, **kw)
            torch.cuda.synchronize()
            tags = (ctypes.c_int32 * n_rec)()
            ms = (ctypes.c_float * n_rec)()
            got = lib.esmb200_profile_read(tags, ms, n_rec)
            lib.esmb200_profile_enable(0)
            samp = sum(ms[i] for i in range(got) if tags[i] == TAG_SAMPLING)
            launches = sum(1 for i in range(got) if tags[i] == TAG_SAMPLING)
            rec["shapes"].append({
                "R": R, "C": C, "entries": n, "block": k, "steps": steps,
                "seconds_per_step": [round(v, 5) for v in step_s],
                "stack_seconds_per_call": [round(v, 5) for v in stack_s],
                "step_over_stack": round(min(step_s) / min(stack_s), 4),
                "stack_tokens_per_s": round(a.chains * R * C / min(step_s)),
                "sampler_launches": launches, "sampler_ms_per_step": round(samp / steps, 4),
                "sampler_share_of_step": round(samp / 1e3 / steps / min(step_s), 6)})
            del xb
            torch.cuda.empty_cache()
    line = json.dumps(rec)
    print(line, flush=True)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
