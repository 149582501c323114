"""Generates tests/golden/esm1b_*.pt by running the UNMODIFIED reference ProteinBertModel (ESM-1b / ESM-1v,
esm/model/esm1.py with arch "roberta_large", imported from /root/reference) on the deterministic weights of
tests/esm1b_weights.make_esm1b_state_dict and tokens of oracle.weights.make_tokens.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_esm1b.py [case ...]
Same fields as make_golden.py, plus the model arguments under "config".  The weights are re-created from the config on
whichever machine runs the tests (checksum stored and verified).  To keep the files small, the per-token outputs of a
case are stored for the token positions [rows[0], rows[1]) only: representations and logits [B, rows, ...], the
attention sub-sample [B, layers, heads, rows, T] (query rows), and the contacts for the same rows minus <cls>
("contacts_rows").  The T = 1024 case keeps its last 8 positions, which use the highest rows of the position table.
"""
import os
import sys
from argparse import Namespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))  # tests/
sys.path.insert(0, "/root/reference")

import esm  # noqa: E402  (the reference)
from esm1b_weights import make_esm1b_state_dict  # noqa: E402  (tests/esm1b_weights.py)
from oracle.weights import make_tokens  # noqa: E402

CASES = {
    # name: (layers, E, H, lengths, total_len, n_mask, repr_layers, token_dropout, emb_layer_norm_before, mid_pads,
    #        stored rows or None for all)
    # (a) padded, <mask> tokens, token dropout, emb_layer_norm_before, and a <pad> inside the third sequence
    "esm1b_tiny_L2_E128_H2": (2, 128, 2, [38, 21, 30], 40, 2, [0, 1, 2], True, True, [(2, 9)], None),
    # (b) no token dropout, no emb_layer_norm_before
    "esm1b_mid_L3_E256_H4": (3, 256, 4, [46, 30], 48, 1, [0, 3], False, False, [], None),
    # (c) T = 1024: sequence 0 reaches the last row of the position table (max_positions + padding_idx)
    "esm1b_edge_L1_E128_H2_T1024": (1, 128, 2, [1022, 600], 1024, 3, [1], True, True, [], (1016, 1024)),
}


def checksum(sd):
    return float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))


def model_args(L, E, H, token_dropout, ln_before):
    return dict(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                max_positions=1024, token_dropout=token_dropout, emb_layer_norm_before=ln_before)


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    only = set(sys.argv[1:])
    for name, (L, E, H, lengths, total, n_mask, repr_layers, td, lnb, mid_pads, rows) in CASES.items():
        if only and name not in only:
            continue
        sd = make_esm1b_state_dict(L, E, H, seed=0, emb_layer_norm_before=lnb)
        args = model_args(L, E, H, td, lnb)
        model = esm.ProteinBertModel(Namespace(**args), esm.Alphabet.from_architecture("roberta_large"))
        model.load_state_dict(sd, strict=True)
        model.eval()
        tokens = make_tokens(lengths, total, seed=1234, n_mask=n_mask)
        for b, t in mid_pads:
            tokens[b, t] = 1
        with torch.no_grad():
            out = model(tokens, repr_layers=repr_layers, need_head_weights=True, return_contacts=True)
        r0, r1 = rows or (0, total)
        c0, c1 = max(r0 - 1, 0), min(r1 - 1, total - 2)  # contact index i is token position i + 1
        layers, heads = sorted({0, L - 1}), sorted({0, H - 1})
        fixture = {
            "config": {"num_layers": L, "embed_dim": E, "attention_heads": H, "seed": 0, "model_args": args},
            "state_dict_checksum": checksum(sd),
            "tokens": tokens,
            "repr_layers": repr_layers,
            "rows": [r0, r1],
            "logits": out["logits"][:, r0:r1].clone(),
            "representations": {k: v[:, r0:r1].clone() for k, v in out["representations"].items()},
            "attentions_sub_layers": layers,
            "attentions_sub_heads": heads,
            "attentions_sub": out["attentions"][:, layers][:, :, heads][..., r0:r1, :].clone(),
            "contacts_rows": [c0, c1],
            "contacts": out["contacts"][:, c0:c1].clone(),
            "reference": "facebookresearch/esm @ 2b36991 (fair-esm 2.0.1), torch %s, CPU fp32" % torch.__version__,
        }
        path = os.path.join(HERE, name + ".pt")
        torch.save(fixture, path)
        print(name, "->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
