"""Developer tool (GPU box): Gibbs sampling (esm_b200.sampling) with ESM-2 650M (esm2_t33_650M_UR50D architecture,
seeded random weights): L = 256, 256 chains, block 8, so one sweep is 32 steps of one [256, 258] stack call each.

One JSON line per repeat with:
  * seconds per step and stack tokens/s: gibbs over --sweeps sweeps, CUDA events around synchronised work;
  * the plain stack model._stack on the same [256, 258] batch, timed over the same number of calls in the same run,
    alternating with gibbs, and the step-to-stack time ratio;
  * the sampler kernels' time per step from the library's profiler (tag 20: the order kernel and both kernels of
    esmb200_sample_rows), in a separate profiled sweep, and their share of a step.
The first line names the card and its power limit (a read-only nvidia-smi query).

    python scripts/sample_bench.py [--sweeps 1] [--repeats 3] [--precision fp16] [--out results.jsonl]
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
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3, out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--length", type=int, default=256)
    p.add_argument("--chains", type=int, default=256)
    p.add_argument("--block", type=int, default=8)
    p.add_argument("--sweeps", type=int, default=1)
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--precision", choices=["fp16", "fp32x3", "fp8"], default="fp16")
    p.add_argument("--out", type=str, default=None, help="also append the JSON lines to this file")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench.py measures on a CUDA (sm_90a) GPU; none is available")
    from esm_b200 import _lib, pretrained, sampling

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    emit({"gpu": query_gpu(), "model": "esm2_t33_650M_UR50D (random init)", "precision": a.precision})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, alphabet = pretrained.load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=True,
                                                             device="cuda")
    model = model.eval().cuda()
    if a.precision != "fp16":
        model.set_precision(a.precision)
    L, C, k = a.length, a.chains, a.block
    T = L + 2
    x0 = torch.tensor([[model.cls_idx] + [model.mask_idx] * L + [model.eos_idx]], device="cuda")
    steps = a.sweeps * -(-L // k)
    kw = dict(chains=C, sweeps=a.sweeps, block=k, seed=1, max_tokens=C * T)
    # the stack alone on a batch of the same shape: the chains with their first block masked
    batch = x0.expand(C, T).contiguous()

    def stack_calls():
        for _ in range(steps):
            model._stack(batch)

    with torch.no_grad():
        sampling.gibbs(model, x0, **kw)  # warm-up: every shape of the timed window
        stack_calls()
        lib = _lib.load()
        for r in range(a.repeats):
            gibbs_s, out = timed(lambda: sampling.gibbs(model, x0, **kw))
            stack_s, _ = timed(stack_calls)
            step_s, stack_step_s = gibbs_s / steps, stack_s / steps
            emit({"repeat": r, "L": L, "chains": C, "block": k, "steps": steps,
                  "seconds_per_step": round(step_s, 5), "stack_seconds_per_call": round(stack_step_s, 5),
                  "stack_tokens_per_s": round(C * T / step_s), "stack_alone_tokens_per_s": round(C * T / stack_step_s),
                  "step_over_stack": round(step_s / stack_step_s, 4),
                  "tokens_all_amino_acids": bool(((out["tokens"][:, 1:-1] >= 4) & (out["tokens"][:, 1:-1] < 24))
                                                 .all())})
        # profiled run of its own: the library's per-launch events around every kernel
        n_rec = 200000
        lib.esmb200_profile_enable(n_rec)
        sampling.gibbs(model, x0, **kw)
        torch.cuda.synchronize()
        tags = (ctypes.c_int32 * n_rec)()
        ms = (ctypes.c_float * n_rec)()
        got = lib.esmb200_profile_read(tags, ms, n_rec)
        lib.esmb200_profile_enable(0)
        samp = sum(ms[i] for i in range(got) if tags[i] == TAG_SAMPLING)
        launches = sum(1 for i in range(got) if tags[i] == TAG_SAMPLING)
        emit({"profiled_launches": got, "sampler_launches": launches,
              "sampler_ms_per_step": round(samp / steps, 4),
              "sampler_share_of_step": round(samp / 1e3 / steps / step_s, 5)})


if __name__ == "__main__":
    main()
