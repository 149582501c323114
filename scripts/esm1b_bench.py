"""Developer tool (GPU box): ESM-1b 650M (esm1b_t33_650M_UR50S) against ESM-2 650M (esm2_t33_650M_UR50D), seeded random
init, on 256 x 1024 synthetic tokens resident in HBM, last representation only (bench.py's configs[1] workload).
The two models are timed alternately inside ONE process with CUDA events (K steps after W warmup steps per round), so
clock drift hits both alike.  Prints one JSON line with sequences/s per model, the card, its power limit and the SM
clock observed right after the timed rounds.

    python scripts/esm1b_bench.py [--batch 256] [--steps 5] [--warmup 2] [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from esm_b200 import pretrained  # noqa: E402


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid; say what is missing
        return f"nvidia-smi unavailable: {e}"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=256)
    p.add_argument("--seq_len", type=int, default=1024)
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=2)
    p.add_argument("--rounds", type=int, default=3)
    a = p.parse_args()
    models = {
        "esm1b_t33_650M_UR50S": pretrained.load_model_and_alphabet("esm1b_t33_650M_UR50S", allow_random_init=True,
                                                                   device="cuda")[0],
        "esm2_t33_650M_UR50D": pretrained.load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=True,
                                                                  device="cuda")[0],
    }
    g = torch.Generator().manual_seed(1)
    tok = torch.randint(4, 24, (a.batch, a.seq_len), generator=g)
    tok[:, 0] = 0
    tok[:, -1] = 2
    tok = tok.cuda()
    ms = {k: [] for k in models}
    for _ in range(a.rounds):
        for name, model in models.items():
            for _ in range(a.warmup):
                model(tok, repr_layers=[33])
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.steps):
                model(tok, repr_layers=[33])
            e.record()
            torch.cuda.synchronize()
            ms[name].append(s.elapsed_time(e) / a.steps)
    gpu = query_gpu()
    res = {name: {"seq_per_s_median": round(a.batch / sorted(v)[len(v) // 2] * 1e3, 2),
                  "ms_per_step": [round(x, 1) for x in v]} for name, v in ms.items()}
    m1, m2 = (res[k]["seq_per_s_median"] for k in models)
    print(json.dumps({"workload": f"{a.batch} x {a.seq_len} tokens, repr_layers=[33], fp16 operands", "results": res,
                      "esm1b_over_esm2": round(m1 / m2, 4),
                      "gpu (name, power.limit, clocks.sm, clocks.max.sm)": gpu}))


if __name__ == "__main__":
    main()
