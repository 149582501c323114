"""The small deterministic models behind tests/golden/variants.json, shared by tests/golden/make_golden_variants.py
(which scores them with the reference's predict.py) and the tests (which rebuild them and compare esm_b200's scores).

Each model is rebuilt from its config on whichever machine runs the tests; the state-dict checksum stored in the
fixture is verified first. `write_checkpoint` writes a model as the .pt file (and, where the reference's loader wants
one, the "-contact-regression.pt" companion, pretrained.py:67-77) that `--model-location` takes."""
from __future__ import annotations

import os
from argparse import Namespace
from typing import Dict

import torch

from esm1b_weights import make_esm1b_state_dict  # tests/esm1b_weights.py
from oracle.msa_oracle import make_msa_state_dict
from oracle.weights import make_state_dict

REGRESSION = ("contact_head.regression.weight", "contact_head.regression.bias")

# name -> config. The file name matters to the reference's loader: "esm2*" selects the ESM-2 format, anything else
# the v1 ("args") format; every file gets the regression companion (the loader wants one unless "esm1v" is in the name).
MODELS = {
    "esm2_t2_tiny": dict(kind="esm2", layers=2, embed_dim=128, attention_heads=2, seed=0, token_dropout=True),
    "esm1b_t2_tiny": dict(kind="esm1b", layers=2, embed_dim=128, attention_heads=2, seed=0,
                          emb_layer_norm_before=True, token_dropout=True),
    "msa_t2_tiny": dict(kind="msa", layers=2, embed_dim=128, attention_heads=2, ffn_embed_dim=512, seed=0),
}


def checksum(sd: Dict[str, torch.Tensor]) -> float:
    return float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))


def state_dict(cfg) -> Dict[str, torch.Tensor]:
    L, E, H, seed = cfg["layers"], cfg["embed_dim"], cfg["attention_heads"], cfg["seed"]
    if cfg["kind"] == "esm2":
        return make_state_dict(L, E, H, seed=seed)
    if cfg["kind"] == "esm1b":
        return make_esm1b_state_dict(L, E, H, seed=seed, emb_layer_norm_before=cfg["emb_layer_norm_before"])
    return make_msa_state_dict(L, E, cfg["ffn_embed_dim"], H, seed=seed)


def model_args(cfg) -> Namespace:
    """The checkpoint's "args" (v1 formats) or cfg["model"] (ESM-2)."""
    L, E, H = cfg["layers"], cfg["embed_dim"], cfg["attention_heads"]
    if cfg["kind"] == "esm2":
        return Namespace(encoder_layers=L, encoder_embed_dim=E, encoder_attention_heads=H,
                         token_dropout=cfg["token_dropout"])
    if cfg["kind"] == "esm1b":
        return Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                         max_positions=1024, token_dropout=cfg["token_dropout"])
    return Namespace(arch="msa_transformer", layers=L, embed_dim=E, ffn_embed_dim=cfg["ffn_embed_dim"],
                     attention_heads=H, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
                     max_tokens_per_msa=2 ** 14, max_tokens=2 ** 14, max_positions=1024, embed_positions_msa=True)


def write_checkpoint(name: str, cfg, directory: str) -> str:
    """Write model `name` as `directory/name.pt` (+ companion); returns the .pt path."""
    sd = state_dict(cfg)
    model = {k: v for k, v in sd.items() if k not in REGRESSION}  # the regression weights go to the companion
    if cfg["kind"] == "msa":
        # the checkpoints name the two attention blocks the other way round (pretrained.py:119)
        swap = lambda k: k.replace("row", "column") if "row" in k else k.replace("column", "row")
        model = {swap(k): v for k, v in model.items()}
    path = os.path.join(directory, name + ".pt")
    if cfg["kind"] == "esm2":
        torch.save({"cfg": {"model": model_args(cfg)}, "model": model}, path)
    else:
        torch.save({"args": model_args(cfg), "model": model}, path)
    torch.save({"model": {k: sd[k] for k in REGRESSION}}, os.path.join(directory, name + "-contact-regression.pt"))
    return path

