"""Developer tool (GPU box): the categorical Jacobian (esm_b200.jacobian) with ESM-2 650M (esm2_t33_650M_UR50D
architecture, seeded random weights), for proteins of --lengths residues (default 256 and 1022) in fp16 and fp32x3.

Per (precision, L), one JSON line with:
  * seconds per protein: categorical_jacobian on one synthetic protein, CUDA events around synchronised work (about
    19 L copies of L + 2 tokens, in chunks of the default 2^17 tokens), and the copies/s and tokens/s it gives;
  * the contact kernel alone: esmb200_jacobian_contacts on that protein's J, CUDA events over --kernel-iters launches;
  * the plain forward model(batch) on one chunk-sized batch [k, L + 2] of the same protein (warmed up once, then
    --forward-iters calls), its tokens/s, and the Jacobian's tokens/s over it.
The first line names the card and its power limit (a read-only nvidia-smi query).

    python scripts/jacobian_bench.py [--lengths 256 1022] [--precisions fp16 fp32x3] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

AA = "LAGVSERTIDPKQNFYMHWC"


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still valid; say what is missing
        return f"nvidia-smi unavailable: {e}"


def timed(fn, iters=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3 / iters, out


def protein(n, seed):
    g = torch.Generator().manual_seed(seed)
    return "".join(AA[i] for i in torch.randint(0, 20, (n,), generator=g).tolist())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lengths", type=int, nargs="+", default=[256, 1022])
    p.add_argument("--precisions", nargs="+", default=["fp16", "fp32x3"], choices=["fp16", "fp32x3"])
    p.add_argument("--kernel-iters", type=int, default=20)
    p.add_argument("--forward-iters", type=int, default=3)
    p.add_argument("--out", type=str, default=None, help="also append the JSON lines to this file")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("jacobian_bench.py measures on a CUDA (sm_90a) GPU; none is available")
    from esm_b200 import jacobian, pretrained
    from esm_b200.variants import _copies_per_chunk

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")

    emit({"gpu": query_gpu(), "model": "esm2_t33_650M_UR50D (random init)"})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, alphabet = pretrained.load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=True,
                                                             device="cuda")
    model = model.eval().cuda()
    for precision in a.precisions:
        model.set_precision(precision)
        for L in a.lengths:
            tokens = alphabet.get_batch_converter()([("p", protein(L, seed=L))])[2].cuda()
            T = L + 2
            k = _copies_per_chunk(T, None)
            batch = tokens.expand(k, T).contiguous()
            with torch.no_grad():
                model(batch)  # warm-up of the chunk shape
                fwd_s, _ = timed(lambda: model(batch), a.forward_iters)
            jac_s, out = timed(lambda: jacobian.categorical_jacobian(model, tokens, return_jacobian=True))
            J = out.pop("jacobian")
            jacobian.jacobian_contacts(J)
            kern_s, _ = timed(lambda: jacobian.jacobian_contacts(J), a.kernel_iters)
            copies = 19 * L  # every residue is canonical: one identity per position
            fwd_tps = k * T / fwd_s
            jac_tps = copies * T / jac_s
            emit({"precision": precision, "L": L, "seconds_per_protein": round(jac_s, 3), "copies": copies,
                  "copies_per_s": round(copies / jac_s, 1), "tokens_per_s": round(jac_tps),
                  "contacts_kernel_ms": round(kern_s * 1e3, 3), "J_bytes": J.numel() * 4,
                  "forward_batch": [k, T], "forward_tokens_per_s": round(fwd_tps),
                  "jacobian_over_forward_tokens_per_s": round(jac_tps / fwd_tps, 3),
                  "contacts_finite": bool(out["contacts"].isfinite().all())})
            del J, out
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
