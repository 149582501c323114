"""Developer tool (GPU box): variant-effect scoring with ESM-1v 650M (esm1v_t33_650M_UR90S_1 architecture, seeded
random weights) on the BLAT_ECOLX wild type (263 residues, examples/variant-prediction/README.md:12), two workloads:

  * masked-marginals over all 265 token positions;
  * pseudo-ppl of 32 single mutants (the library arm scores all 32; the reference arm scores 2 and is reported per
    mutant, since its batch-1 loop takes about L forwards per mutant).

Library arm: esm_b200.variants (masked copies batched into one stack call per chunk, LM head on the masked rows).
Reference arm: the unmodified reference model from oracle/_ref (made by build()), eager fp32 with TF32 off, running
predict.py's batch-1 loops (predict.py:118-144, 206-214). The arms alternate for --rounds rounds in one process, each
timed with CUDA events after a warm-up. Prints one JSON line with the times, the card, its power limit and SM clock.

    python scripts/variant_bench.py [--rounds 3] [--max-tokens 131072]
"""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.path.join(ROOT, "oracle", "_ref")

BLAT_ECOLX = ("HPETLVKVKDAEDQLGARVGYIELDLNSGKILESFRPEERFPMMSTFKVLLCGAVLSRVDAGQEQLGRRIHYSQNDLVEYSPVTEKHLTDGMTVRELCSAAIT"
              "MSDNTAANLLLTTIGGPKELTAFLHNMGDHVTRLDRWEPELNEAIPNDERDTTMPAAMATTLRKLLTGELLTLASRQQLIDWMEADKVAGPLLRSALPAGWFIA"
              "DKSGAGERGSRGIIAALGPDGKPSRIVVIYTTGSQATMDERNRQIAEIGASLIKHW")
AA = "ACDEFGHIKLMNPQRSTVWY"


def query_gpu():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
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
    p.add_argument("--rounds", type=int, default=3)
    p.add_argument("--mutants", type=int, default=32)
    p.add_argument("--ref-mutants", type=int, default=2)
    p.add_argument("--max-tokens", type=int, default=None)
    a = p.parse_args()
    if not os.path.isdir(os.path.join(REF, "esm")):
        raise SystemExit("oracle/_ref/esm is missing: run build() first (oracle/reference.py)")
    sys.path.insert(0, REF)
    import esm  # the reference, unmodified
    from esm1b_weights import make_esm1b_state_dict  # tests/esm1b_weights.py
    from esm_b200 import ProteinBertModel, variants

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, H = 33, 1280, 20
    args = argparse.Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                              max_positions=1024, emb_layer_norm_before=True, token_dropout=True)
    sd = make_esm1b_state_dict(L, E, H, seed=0)
    alphabet = esm.Alphabet.from_architecture("roberta_large")
    ref = esm.ProteinBertModel(args, alphabet)
    ref.load_state_dict(sd, strict=True)
    ref = ref.eval().cuda()
    lib = ProteinBertModel(args, "roberta_large")
    lib.load_state_dict(sd, strict=True)
    lib = lib.eval().cuda()
    del sd

    seq = BLAT_ECOLX
    rng = random.Random(0)
    muts = []
    for i in rng.sample(range(len(seq)), a.mutants):
        muts.append(f"{seq[i]}{i + 1}{rng.choice([c for c in AA if c != seq[i]])}")
    _, _, tokens = alphabet.get_batch_converter()([("protein1", seq)])
    tokens = tokens.cuda()

    def ref_masked_marginals():  # predict.py:206-215
        rows = []
        with torch.no_grad():
            for i in range(tokens.size(1)):
                t = tokens.clone()
                t[0, i] = alphabet.mask_idx
                rows.append(torch.log_softmax(ref(t)["logits"], dim=-1)[:, i])
        return torch.cat(rows)

    def ref_pppl(row):  # compute_pppl, predict.py:118-144
        wt, idx, mt = row[0], int(row[1:-1]) - 1, row[-1]
        s = seq[:idx] + mt + seq[idx + 1:]
        _, _, bt = alphabet.get_batch_converter()([("protein1", s)])
        lp = []
        with torch.no_grad():
            for i in range(1, len(s) - 1):
                t = bt.clone()
                t[0, i] = alphabet.mask_idx
                lp.append(torch.log_softmax(ref(t.cuda())["logits"], dim=-1)[0, i, alphabet.get_idx(s[i])].item())
        return sum(lp)

    # warm-up of every shape both arms use
    ref(tokens)
    variants.masked_marginals(lib, tokens, max_tokens=a.max_tokens)
    variants.pseudo_ppl(lib, lib.alphabet, seq, muts[:1], 1, a.max_tokens)

    t = {"lib_masked_marginals_s": [], "ref_masked_marginals_s": [], "lib_pppl_s_per_mutant": [],
         "ref_pppl_s_per_mutant": []}
    agree = {}
    for _ in range(a.rounds):
        dt, got = timed(lambda: variants.masked_marginals(lib, tokens, max_tokens=a.max_tokens))
        t["lib_masked_marginals_s"].append(dt)
        dt, want = timed(ref_masked_marginals)
        t["ref_masked_marginals_s"].append(dt)
        c = lambda x: x.double() - x.double().mean(-1, keepdim=True)
        agree["masked_marginals_centered_rel_fro"] = float((c(got) - c(want)).norm() / c(want).norm())
        dt, pl = timed(lambda: variants.pseudo_ppl(lib, lib.alphabet, seq, muts, 1, a.max_tokens))
        t["lib_pppl_s_per_mutant"].append(dt / len(muts))
        dt, pr = timed(lambda: [ref_pppl(m) for m in muts[:a.ref_mutants]])
        t["ref_pppl_s_per_mutant"].append(dt / a.ref_mutants)
        agree["pppl_max_rel"] = max(abs(x - y) / abs(y) for x, y in zip(pl, pr))
    gpu = query_gpu()
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    print(json.dumps({
        "workload": f"ESM-1v 650M (seeded random weights), BLAT_ECOLX wild type, T = {tokens.size(1)} tokens; "
                    f"masked-marginals over all positions; pseudo-ppl of {a.mutants} mutants "
                    f"(reference arm: {a.ref_mutants}); library fp16 operands, reference eager fp32 (TF32 off)",
        "seconds": {k: [round(x, 4) for x in v] for k, v in t.items()},
        "median_speedup": {"masked_marginals": round(med["ref_masked_marginals_s"] / med["lib_masked_marginals_s"], 2),
                           "pseudo_ppl_per_mutant": round(med["ref_pppl_s_per_mutant"] / med["lib_pppl_s_per_mutant"], 2)},
        "agreement": agree,
        "gpu (name, power.limit, clocks.sm, clocks.max.sm)": gpu}))


if __name__ == "__main__":
    main()
