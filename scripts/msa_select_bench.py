"""Developer tool (GPU box): greedy row selection for the MSA Transformer (esm_b200.msa_select) on deep alignments.

For N in {10^4, 10^5} rows, C in {256, 512} columns and k in {128, 256} picks, and at the three sizes the README gives
CPU times for (N = 5,000 and 20,000, C = 256), on seeded random alignments over the 20 amino acids and the gap:
  * seconds per selection of greedy_select_indices on an alignment already on the GPU (device events around
    synchronised work, every one of --repeats, both modes);
  * whether the picked rows, in selection order, equal the numpy restatement of the notebook's function
    (tests/msa_select_refs.py; --no-check skips it);
  * for scale, one predict_contacts of the MSA Transformer (esm_msa1b_t12_100M_UR50S architecture, seeded random
    weights, fp16) on the k selected rows.
Prints one JSON line with the card and its power limit (a read-only nvidia-smi query).

    python scripts/msa_select_bench.py [--repeats 3] [--no-check] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # msa_select_refs

# the grid above, then the sizes at which the notebook's own function was timed on the CPU (README, "Picking the rows")
CASES = [(N, C, k) for N in (10_000, 100_000) for C in (256, 512) for k in (128, 256)] + \
    [(5_000, 256, 128), (20_000, 256, 128), (20_000, 256, 256)]
LETTERS = "ACDEFGHIKLMNPQRSTVWY-"


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
    p.add_argument("--repeats", type=int, default=3)
    p.add_argument("--no-check", dest="check", action="store_false")
    p.add_argument("--out", type=str, default=None, help="also append the JSON line to this file")
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("msa_select_bench.py measures on a CUDA (sm_90a) GPU; none is available")
    from esm_b200 import msa_select, pretrained
    import msa_select_refs as ref

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, alphabet = pretrained.load_msa_model_and_alphabet("esm_msa1b_t12_100M_UR50S", allow_random_init=True,
                                                                 device="cuda")
    model = model.eval().cuda()
    lut = torch.zeros(256, dtype=torch.int64)
    for ch in LETTERS:
        lut[ord(ch)] = alphabet.get_idx(ch)
    rec = {"gpu": query_gpu(), "contacts_model": "esm_msa1b_t12_100M_UR50S (random init, fp16)", "cases": []}
    letters = np.frombuffer(LETTERS.encode(), dtype=np.uint8)
    for N, C, k in CASES:
        rows = letters[np.random.default_rng(N + C + k).integers(0, len(letters), (N, C))]
        dev = torch.from_numpy(rows).cuda()
        case = {"N": N, "C": C, "k": k}
        for mode in ("max", "min"):
            msa_select.greedy_select_indices(dev, k, mode)  # warm-up
            t_dev = [timed(lambda: msa_select.greedy_select_indices(dev, k, mode))[0] for _ in range(a.repeats)]
            case[mode] = {"seconds": [round(v, 6) for v in t_dev]}
            if a.check:
                got = msa_select._order(dev, k, mode).tolist()
                case[mode]["equals_restatement"] = got == ref.greedy_order(rows, k, mode)
        idx = msa_select.greedy_select_indices(dev, k, "max")
        tokens = torch.cat([torch.full((k, 1), alphabet.cls_idx, dtype=torch.int64),
                            lut[torch.from_numpy(rows[idx.cpu().numpy()]).long()]], 1)[None].cuda()
        with torch.no_grad():
            model.predict_contacts(tokens)  # warm-up
            case["predict_contacts_s"] = round(min(timed(lambda: model.predict_contacts(tokens))[0]
                                                   for _ in range(a.repeats)), 5)
        rec["cases"].append(case)
        print(json.dumps(case), flush=True)
        del dev, tokens
        torch.cuda.empty_cache()
    line = json.dumps(rec)
    print(line, flush=True)
    if a.out:
        with open(a.out, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
