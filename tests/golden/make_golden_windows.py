"""Generates tests/golden/windows/esm1b_L2_E128_H2_P64.pt by running the UNMODIFIED reference ProteinBertModel (ESM-1b /
ESM-1v, esm/model/esm1.py with arch "roberta_large", imported from /root/reference) on every window crop of a protein
longer than the model's position table, and on masked copies of those crops.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_windows.py
The model has max_positions = 64, so the 150-residue protein cannot run whole; with a window of W = 62 residues
(W + <cls> + <eos> = 64 tokens) it runs as 4 crops starting at residues 0, 29, 58 and 88 (esm_b200/windows.py; the
starts are pinned in the file). Each crop is tokenised as a protein of its own. Stored per crop: the logits and the
last layer's representation [K, W + 2, ...]; and for a few token positions of the whole protein, the logits row of the
masked position in each crop that covers it (the crop with that residue masked). The weights are re-created from the
config on whichever machine runs the tests (checksum stored and verified); the test merges these outputs with the
documented weights and compares the library's windowed forward and scorers to them.
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

NAME = "esm1b_L2_E128_H2_P64"  # in tests/golden/windows/: the layer-stack fixtures at tests/golden/*.pt share a schema
L, E, H, P = 2, 128, 2, 64
N_RES, W = 150, 62
STARTS = [0, 29, 58, 88]
# token positions (<cls> = 0): <cls>, residues in one, two and three crops, the last residue, <eos>
MASKED = [0, 1, 31, 45, 60, 75, 100, 150, 151]
AMINO = "LAGVSERTIDPKQNFYMHWC"


def checksum(sd):
    return float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    g = torch.Generator().manual_seed(2024)
    sequence = "".join(AMINO[i] for i in torch.randint(0, len(AMINO), (N_RES,), generator=g).tolist())
    sd = make_esm1b_state_dict(L, E, H, seed=0, emb_layer_norm_before=True, max_positions=P)
    args = dict(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                max_positions=P, token_dropout=True, emb_layer_norm_before=True)
    alphabet = esm.Alphabet.from_architecture("roberta_large")
    model = esm.ProteinBertModel(Namespace(**args), alphabet)
    model.load_state_dict(sd, strict=True)
    model.eval()
    convert = alphabet.get_batch_converter()
    crops = [sequence[s:s + W] for s in STARTS]
    _, _, tokens = convert([(f"crop{k}", c) for k, c in enumerate(crops)])
    assert tokens.shape == (len(STARTS), W + 2)
    masked = {}
    with torch.no_grad():
        out = model(tokens, repr_layers=[L])
        for t in MASKED:
            rows = []
            for k, s in enumerate(STARTS):
                if t == 0:
                    r = 0 if k == 0 else None
                elif t == N_RES + 1:
                    r = W + 1 if k == len(STARTS) - 1 else None
                else:
                    r = t - s if s <= t - 1 < s + W else None
                if r is None:
                    continue
                copy = tokens[k:k + 1].clone()
                copy[0, r] = alphabet.mask_idx
                rows.append((k, r, model(copy)["logits"][0, r].clone()))
            masked[t] = rows
    fixture = {
        "config": {"num_layers": L, "embed_dim": E, "attention_heads": H, "seed": 0, "model_args": args},
        "state_dict_checksum": checksum(sd),
        "sequence": sequence,
        "window": W,
        "starts": STARTS,
        "window_tokens": tokens,
        "logits": out["logits"].clone(),
        "representations": out["representations"][L].clone(),
        "masked": masked,
        "reference": "facebookresearch/esm @ 2b36991 (fair-esm 2.0.1), torch %s, CPU fp32" % torch.__version__,
    }
    path = os.path.join(HERE, "windows", NAME + ".pt")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save(fixture, path)
    print(NAME, "->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
