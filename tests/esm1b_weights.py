"""Deterministic ESM-1b / ESM-1v weights shared by tests/golden/make_golden_esm1b.py (which runs the reference on them)
and the tests that re-create them to compare esm_b200 against the committed outputs.  Same conventions as
oracle.weights.make_state_dict (seeded CPU generator, randomised LayerNorm gains/biases and biases, q/k gain 1.5)."""
from __future__ import annotations

from typing import Dict

import torch

from oracle.weights import VOCAB


def make_esm1b_state_dict(num_layers: int, embed_dim: int, num_heads: int, seed: int = 0, qk_gain: float = 1.5,
                          emb_layer_norm_before: bool = True, max_positions: int = 1024) -> Dict[str, torch.Tensor]:
    """ESM-1b / ESM-1v (esm/model/esm1.py, arch roberta_large) weights under the reference's keys: the ESM-2 layer
    without rot_emb, a learned position table embed_positions.weight [max_positions + padding_idx + 1, E] drawn with
    std 1 (an off-by-one in the position index moves the output by O(1)), and the optional emb_layer_norm_before.
    LayerNorm gains/biases and all biases are randomised like make_state_dict's."""
    g = torch.Generator().manual_seed(seed)
    E, F = embed_dim, 4 * embed_dim

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g, dtype=torch.float32) * std

    sd: Dict[str, torch.Tensor] = {}
    emb = rn(VOCAB, E, std=1.0)
    emb[1].zero_()  # padding_idx row
    sd["embed_tokens.weight"] = emb
    sd["embed_positions.weight"] = rn(max_positions + 1 + 1, E, std=1.0)  # padding_idx = 1 (modules.py:232-238)
    w_std = E ** -0.5
    for i in range(num_layers):
        p = f"layers.{i}."
        for name in ("q_proj", "k_proj", "v_proj", "out_proj"):
            gain = qk_gain if name in ("q_proj", "k_proj") else 1.0
            sd[p + f"self_attn.{name}.weight"] = rn(E, E, std=w_std * gain)
            sd[p + f"self_attn.{name}.bias"] = rn(E, std=0.1)
        sd[p + "self_attn_layer_norm.weight"] = 1.0 + rn(E, std=0.2)
        sd[p + "self_attn_layer_norm.bias"] = rn(E, std=0.1)
        sd[p + "fc1.weight"] = rn(F, E, std=w_std)
        sd[p + "fc1.bias"] = rn(F, std=0.1)
        sd[p + "fc2.weight"] = rn(E, F, std=F ** -0.5)
        sd[p + "fc2.bias"] = rn(E, std=0.1)
        sd[p + "final_layer_norm.weight"] = 1.0 + rn(E, std=0.2)
        sd[p + "final_layer_norm.bias"] = rn(E, std=0.1)
    sd["contact_head.regression.weight"] = rn(1, num_layers * num_heads, std=1.0)
    sd["contact_head.regression.bias"] = rn(1, std=0.1)
    if emb_layer_norm_before:
        sd["emb_layer_norm_before.weight"] = 1.0 + rn(E, std=0.2)
        sd["emb_layer_norm_before.bias"] = rn(E, std=0.1)
    sd["emb_layer_norm_after.weight"] = 1.0 + rn(E, std=0.2)
    sd["emb_layer_norm_after.bias"] = rn(E, std=0.1)
    sd["lm_head.weight"] = sd["embed_tokens.weight"]  # tied, esm1.py:101-105
    sd["lm_head.bias"] = rn(VOCAB, std=0.1)
    sd["lm_head.dense.weight"] = rn(E, E, std=w_std)
    sd["lm_head.dense.bias"] = rn(E, std=0.1)
    sd["lm_head.layer_norm.weight"] = 1.0 + rn(E, std=0.2)
    sd["lm_head.layer_norm.bias"] = rn(E, std=0.1)
    return sd
