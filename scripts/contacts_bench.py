"""Contacts with and without the attention stack: forward(tokens, return_contacts=True) against predict_contacts.

    python scripts/contacts_bench.py [--rounds 5] [--skip-650M] [--skip-15B]

1. configs[3] (esm2_t36_3B_UR50D shape, seeded random init, 16 x 512): the two calls alternated for --rounds rounds in
   one process after a warm-up of each, every call timed with device events (medians reported), each call's
   torch.cuda.max_memory_allocated measured on its own, and the two contact maps compared bit for bit.
2. predict_contacts alone on a 650M-shape (33 x 1280 x 20) 64 x 1024 batch: extract_cli's default token budget, whose
   attention stack (177 GB) the forward cannot allocate.
3. predict_contacts alone on a 15B-shape cpu_offload() model (one seeded layer repeated 48 times, as
   scripts/offload_bench.py builds it) for one protein of 2048 and of 4096 tokens (stacks of 32 and 129 GB).

Prints one JSON line per case; the first and the last line carry the card's name, power limit and SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from esm_b200 import pretrained  # noqa: E402

DEV = torch.device("cuda", 0)


def card():
    info = {"device": torch.cuda.get_device_name(DEV)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["max_sm_clock"] = [s.strip() for s in q.split(",")][:3]
    except Exception as e:  # reported, not fatal: the timings stand without it
        info["power_limit"] = f"unavailable ({e})"
    return info


def tokens(B, T, seed=1234):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(4, 24, (B, T), generator=g)
    t[:, 0], t[:, -1] = 0, 2
    return t.to(DEV)


def timed(fn):
    """(ms by device events, peak bytes allocated during the call above what was allocated before it, result)"""
    torch.cuda.synchronize(DEV)
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated(DEV) - base, out


def stack_gb(model, B, T):
    return 4 * B * model.num_layers * model.attention_heads * T * T / 1e9


def compare_3B(rounds):
    B, T = 16, 512
    model, _ = pretrained.load_model_and_alphabet("esm2_t36_3B_UR50D", allow_random_init=True)
    model = model.eval().to(DEV)
    tok = tokens(B, T)
    calls = {"forward": lambda: model(tok, return_contacts=True)["contacts"],
             "predict_contacts": lambda: model.predict_contacts(tok)}
    with torch.no_grad():
        outs = {k: timed(f)[2] for k, f in calls.items()}  # warm-up, also caches the workspace
        same = torch.equal(outs["forward"], outs["predict_contacts"])
        del outs
        ms = {k: [] for k in calls}
        peak = {k: 0 for k in calls}
        for _ in range(rounds):
            for k, f in calls.items():
                t, p, _ = timed(f)
                ms[k].append(t)
                peak[k] = max(peak[k], p)
    med = {k: statistics.median(v) for k, v in ms.items()}
    res = {"case": "configs[3] 3B 16x512", "batch": [B, T], "stack_gb": round(stack_gb(model, B, T), 2),
           "contacts_bit_identical": same,
           "forward_ms": round(med["forward"], 2), "predict_contacts_ms": round(med["predict_contacts"], 2),
           "forward_over_predict_contacts": round(med["forward"] / med["predict_contacts"], 4),
           "forward_peak_gb": round(peak["forward"] / 1e9, 3),
           "predict_contacts_peak_gb": round(peak["predict_contacts"] / 1e9, 3),
           "rounds_ms": {k: [round(v, 2) for v in vs] for k, vs in ms.items()}}
    del model
    torch.cuda.empty_cache()
    return res


def contacts_only(name, model, B, T, rounds):
    tok = tokens(B, T)
    with torch.no_grad():
        timed(lambda: model.predict_contacts(tok))  # warm-up
        ms, peak, finite = [], 0, True
        for _ in range(rounds):
            t, p, out = timed(lambda: model.predict_contacts(tok))
            ms.append(t)
            peak = max(peak, p)
            finite = finite and bool(torch.isfinite(out).all())
            del out
    return {"case": name, "batch": [B, T], "stack_gb": round(stack_gb(model, B, T), 2),
            "predict_contacts_ms": round(statistics.median(ms), 2), "predict_contacts_peak_gb": round(peak / 1e9, 3),
            "contacts_finite": finite, "rounds_ms": [round(v, 2) for v in ms]}


def main():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    p.add_argument("--rounds", type=int, default=5)
    p.add_argument("--skip-650M", action="store_true")
    p.add_argument("--skip-15B", action="store_true")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("contacts_bench.py measures on a CUDA (sm_90a) device; none is available")
    info = card()
    print(json.dumps({"card_before": info}), flush=True)
    print(json.dumps({**compare_3B(args.rounds), **info}), flush=True)
    if not args.skip_650M:
        model, _ = pretrained.load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=True)
        model = model.eval().to(DEV)
        print(json.dumps({**contacts_only("650M 64x1024", model, 64, 1024, args.rounds), **info}), flush=True)
        del model
        torch.cuda.empty_cache()
    if not args.skip_15B:
        import offload_bench
        from esm_b200.model import ContactPredictionHead
        model = offload_bench.model(5120, 40, 48)
        # offload_bench's model keeps the one-layer contact head of the ESM2 it starts from: one for 48 x 40 channels
        model.contact_head = ContactPredictionHead(48 * 40, model.prepend_bos, model.append_eos, eos_idx=model.eos_idx)
        model = model.cpu_offload(DEV)
        for T in (2048, 4096):
            r = contacts_only(f"15B cpu_offload 1x{T}", model, 1, T, max(1, min(args.rounds, 3)))
            print(json.dumps({**r, **info}), flush=True)
        del model
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
