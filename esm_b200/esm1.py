"""Host-side mirror of the reference's ESM-1b / ESM-1v model, esm.model.esm1.ProteinBertModel with arch "roberta_large"
(/root/reference/esm/model/esm1.py:22-200), dispatching to libesmb200.so.

ESM-1b (esm1b_t33_650M_UR50S) and the five ESM-1v models (esm1v_t33_650M_UR90S_1 ... _5) are the ESM-2 650M stack
without rotary embeddings: the same pre-LN TransformerLayer (33 x 1280 x 20 heads, FFN 5120, no bias_kv), positions
from a learned table added in the embedding prologue, an optional emb_layer_norm_before, the same LM and contact heads.
The forward is ESM2's (model.ProteinLanguageModel): esmb200_esm1b_embed -> one esmb200_stack_forward with no rotary
tables (contacts fused) -> RobertaLMHead.forward_native -> final LayerNorm.

ESM-1 (arch "protein_bert_base": bias_kv attention, sinusoidal positions, ESM1LayerNorm, embed_out) is not supported.
"""
from __future__ import annotations

from argparse import Namespace
from typing import Union

import torch
import torch.nn as nn

from . import _lib
from .alphabet import Alphabet
from .model import ProteinLanguageModel, _ptr, _stream
from .msa import LearnedPositionalEmbedding


class ProteinBertModel(ProteinLanguageModel):
    """Drop-in for esm.model.esm1.ProteinBertModel (ESM-1b / ESM-1v): same constructor `(args, alphabet)`, same
    state-dict keys (embed_positions.weight [max_positions + padding_idx + 1, E], emb_layer_norm_before.* when
    args.emb_layer_norm_before), same forward contract and result dict (esm1.py:116-193)."""

    def __init__(self, args: Union[Namespace, dict], alphabet: Union[Alphabet, str] = "ESM-1b"):
        super().__init__()
        if isinstance(args, dict):
            args = Namespace(**args)
        if getattr(args, "arch", "roberta_large") != "roberta_large":
            raise ValueError(f"esm_b200 runs ESM-1b / ESM-1v (arch 'roberta_large') only; got arch {args.arch!r}: "
                             "ESM-1 (bias_kv attention) is not supported")
        self.args = args
        if isinstance(alphabet, str):
            alphabet = Alphabet.from_architecture(alphabet)
        self.model_version = "ESM-1b"
        E = args.embed_dim
        # esm1.py:67-105, in the reference's construction order
        self._init_encoder(args.layers, E, args.attention_heads, args.ffn_embed_dim, alphabet,
                           getattr(args, "token_dropout", False), False)
        self.embed_positions = LearnedPositionalEmbedding(args.max_positions, E, self.padding_idx)
        self.emb_layer_norm_before = nn.LayerNorm(E) if getattr(args, "emb_layer_norm_before", False) else None
        self._init_head(E)

    def _rope_tables(self, T: int):
        return None, None  # learned positions, added by the prologue

    def _embed(self, tokens: torch.Tensor, x: torch.Tensor) -> None:
        """esm1.py:121-139"""
        B, T, E = x.shape
        table = self._mirror("embed_tokens", self.embed_tokens.weight)
        pos = self._mirror("embed_positions", self.embed_positions.weight)
        ln = self.emb_layer_norm_before
        ln_w = self._mirror("ln_before.w", ln.weight) if ln is not None else None
        ln_b = self._mirror("ln_before.b", ln.bias) if ln is not None else None
        _lib.check(_lib.load().esmb200_esm1b_embed(
            _ptr(tokens), _ptr(table), _ptr(pos), _ptr(ln_w), _ptr(ln_b), ln.eps if ln is not None else 1e-5,
            int(self.token_dropout), self.padding_idx, self.mask_idx, _ptr(x), B, T, E, _stream()))

    def _stack(self, tokens, *args, **kwargs):
        """forward's stack step (also the variant scorers'), behind the reference's length check."""
        max_positions = self.embed_positions.max_positions
        if tokens.size(1) > max_positions:  # modules.py:242-246
            raise ValueError(f"Sequence length {tokens.size(1)} above maximum  sequence length of {max_positions}")
        return super()._stack(tokens, *args, **kwargs)
