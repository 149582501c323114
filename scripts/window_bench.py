"""Developer tool (GPU box): proteins longer than the window (esm_b200.windows) with ESM-1v 650M
(esm1v_t33_650M_UR90S_1 architecture, seeded random weights, 1022-residue windows), three timings:

  * masked-marginals over every token position of one 3000-residue synthetic protein (5 windows; one masked copy per
    window covering a position, about 1.7 copies per residue);
  * forward_windowed on 64 proteins of 2500 residues (4 windows each, 256 windows in one batch), last-layer
    representations and logits;
  * esmb200_window_merge alone on the merges of the second workload (the logits [64 x 2502, 33] and one
    representation [64 x 2502, 1280] from 256 x 1024 window rows), CUDA events over --merge-iters launches.

Each workload is warmed up once, then timed for --rounds rounds with CUDA events. Prints one JSON line with the times,
the merge's share of the windowed forward, the card's name and its power limit.

    python scripts/window_bench.py [--rounds 2] [--merge-iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

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


def protein(n, seed):
    g = torch.Generator().manual_seed(seed)
    return "".join(AA[i] for i in torch.randint(0, 20, (n,), generator=g).tolist())


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--merge-iters", type=int, default=50)
    p.add_argument("--window", type=int, default=1022)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("window_bench times the H100 path: no CUDA device")
    from esm1b_weights import make_esm1b_state_dict  # tests/esm1b_weights.py
    from esm_b200 import ProteinBertModel, variants, windows

    L, E, H, W = 33, 1280, 20, a.window
    args = argparse.Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                              max_positions=1024, emb_layer_norm_before=True, token_dropout=True)
    model = ProteinBertModel(args, "ESM-1b")
    model.load_state_dict(make_esm1b_state_dict(L, E, H, seed=0), strict=True)
    model = model.eval().cuda()
    convert = model.alphabet.get_batch_converter()
    _, _, long_tokens = convert([("p", protein(3000, 1))])
    _, _, batch = convert([(str(i), protein(2500, 100 + i)) for i in range(64)])
    batch = batch.cuda()

    # the merges of the batch workload, built as forward_windowed builds them
    T = batch.shape[1]
    Tw = W + 2
    idx, w, out_rows, nw = [], [], [], 0
    for b in range(64):
        plan = windows.Plan(2500, W, 1, 1)
        pos, win, row, wt = plan.terms()
        out_rows.append(b * T + pos)
        idx.append((nw + win) * Tw + row)
        w.append(wt)
        nw += plan.K
    idx, w = torch.cat(idx).cuda(), torch.cat(w).cuda()
    seg = windows.segments(torch.cat(out_rows), 64 * T).cuda()
    src_logits = torch.randn((nw * Tw, 33), device="cuda")
    src_repr = torch.randn((nw * Tw, E), device="cuda")

    def merge_only(src):
        windows.merge_rows(src, idx, w, seg)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.merge_iters):
            windows.merge_rows(src, idx, w, seg)
        e.record()
        torch.cuda.synchronize()
        return s.elapsed_time(e) / 1e3 / a.merge_iters

    mm = lambda: variants.masked_marginals(model, long_tokens, window=W)
    fw = lambda: model.forward_windowed(batch, W, repr_layers=[L])
    mm()
    fw()
    t = {"masked_marginals_3000_s": [], "forward_windowed_64x2500_s": [], "merge_logits_s": [], "merge_repr_s": []}
    for _ in range(a.rounds):
        t["masked_marginals_3000_s"].append(timed(mm)[0])
        t["forward_windowed_64x2500_s"].append(timed(fw)[0])
        t["merge_logits_s"].append(merge_only(src_logits))
        t["merge_repr_s"].append(merge_only(src_repr))
    med = {k: sorted(v)[len(v) // 2] for k, v in t.items()}
    plan3000 = windows.Plan(3000, W, 1, 1)
    copies = plan3000.terms()[0].numel()
    print(json.dumps({
        "workload": f"ESM-1v 650M (seeded random weights), fp16 operands, window {W} residues; masked-marginals of one "
                    f"3000-residue protein ({plan3000.K} windows, {copies} masked copies of {Tw} tokens); "
                    f"forward_windowed of 64 x 2500 residues ({nw} windows) with logits and the last representation",
        "seconds": {k: [round(x, 6) for x in v] for k, v in t.items()},
        "merge_share_of_forward_windowed": round((med["merge_logits_s"] + med["merge_repr_s"])
                                                 / med["forward_windowed_64x2500_s"], 5),
        "merge_repr_GB_per_s": round(4.0 * (idx.numel() + 64 * T) * E / med["merge_repr_s"] / 1e9, 1),
        "gpu (name, power.limit, clocks.sm, clocks.max.sm)": query_gpu()}))


if __name__ == "__main__":
    main()
