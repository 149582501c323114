"""MSA-Transformer axial block on the sm_90a kernels — host-side mirror of
/root/reference/esm/modules.py:145-221 (AxialTransformerLayer, NormalizedResidualBlock :360-392,
FeedForwardNetwork :395-418) and /root/reference/esm/axial_attention.py (RowSelfAttention :11-130,
ColumnSelfAttention :133-239), with the reference's parameter names so its state dicts load.

CUDA path for BASELINE.json configs[4] (SURVEY §8f #3).  All the arithmetic of the block runs in libesmb200.so:
  * LayerNorm -> fp16, q/k/v projection (+ bias, q scale; no rotary embedding), out-projection + residual,
    fc1 + erf-GELU, fc2 + residual: the same wgmma GEMM / LayerNorm kernels as the ESM-2 path;
  * tied row attention (logits summed over the R rows, axial_attention.py:87): esmb200_tied_row_attention — a tensor-core
    contraction over K = R*64 that walks the alignment rows with TMA boxes taken straight from the projection output,
    a row softmax (with the reference's -10000 fill on padded key columns), and the P.V update with V tiles as the
    MN-major operand (csrc/tied_attention.cuh);
  * column attention: the flash-attention kernel with strided TMA boxes, one "sequence" of R rows per alignment column,
    no regrouping copy (csrc/attention8.cuh, AttnParams::cols); when the maps are asked for, the probability kernel
    writes them from the same strided view (csrc/attention_probs.cuh, ProbsParams::cols).
The layers run in one esmb200_axial_stack_forward call, with or without attention maps; PyTorch only holds the buffers.

Padding: the reference fills padded keys with -10000, this path gives them probability exactly 0 in the column
attention — identical unless every key of a column is padded (there the reference averages v uniformly, this path
returns 0); such positions are themselves padding.  head_dim 64, inference only.

Precision: fp16 MMA operands by default; `MSATransformer.set_precision("fp32x3")` runs every GEMM and attention operand
of the axial stack and the LM head as an fp16 hi | lo pair (DESIGN.md section 4).
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

import ctypes
from argparse import Namespace
from typing import Dict, Sequence, Union

from . import _lib
from .alphabet import Alphabet
from .model import ContactPredictionHead, RobertaLMHead, _ptr, _stream, _workspace


class _AttnParams(nn.Module):
    """q/k/v/out projections under the reference's names (axial_attention.py:30-34, 151-155)."""

    def __init__(self, embed_dim: int, num_heads: int):
        super().__init__()
        self.num_heads = num_heads
        self.head_dim = embed_dim // num_heads
        self.k_proj = nn.Linear(embed_dim, embed_dim)
        self.v_proj = nn.Linear(embed_dim, embed_dim)
        self.q_proj = nn.Linear(embed_dim, embed_dim)
        self.out_proj = nn.Linear(embed_dim, embed_dim)


class _FFNParams(nn.Module):
    def __init__(self, embed_dim: int, ffn_dim: int):
        super().__init__()
        self.fc1 = nn.Linear(embed_dim, ffn_dim)
        self.fc2 = nn.Linear(ffn_dim, embed_dim)


class _ResidualBlock(nn.Module):
    """`layer` + `layer_norm` containers of NormalizedResidualBlock (modules.py:360-373)."""

    def __init__(self, layer: nn.Module, embed_dim: int):
        super().__init__()
        self.layer = layer
        self.layer_norm = nn.LayerNorm(embed_dim)


class AxialTransformerLayer(nn.Module):
    """Drop-in for esm.modules.AxialTransformerLayer (modules.py:145-221) at inference."""

    def __init__(self, embedding_dim: int = 768, ffn_embedding_dim: int = 3072, num_attention_heads: int = 8,
                 dropout: float = 0.1, attention_dropout: float = 0.1, activation_dropout: float = 0.1,
                 max_tokens_per_msa: int = 2 ** 14) -> None:
        super().__init__()
        if embedding_dim != 64 * num_attention_heads:
            raise ValueError("esm_b200 supports head_dim == 64 only")
        self.embedding_dim = embedding_dim
        self.ffn_embedding_dim = ffn_embedding_dim
        self.num_heads = num_attention_heads
        self.row_self_attention = _ResidualBlock(_AttnParams(embedding_dim, num_attention_heads), embedding_dim)
        self.column_self_attention = _ResidualBlock(_AttnParams(embedding_dim, num_attention_heads), embedding_dim)
        self.feed_forward_layer = _ResidualBlock(_FFNParams(embedding_dim, ffn_embedding_dim), embedding_dim)
        self._handles = None
        self._handles_key = None
        self.precision = 0  # 0 = fp16 MMA operands, 1 = "fp32x3" (esmb200.h: esmb200_layer_weights.precision)

    # ---- C-ABI handles: (row attention-only layer, column attention + feed-forward layer) ----------------------
    def handles(self):
        ps = list(self.parameters())
        key = (self.precision,) + tuple((p.data_ptr(), p._version) for p in ps)
        if self._handles is not None and key == self._handles_key:
            return self._handles
        self.release()
        for p in ps:
            if not p.is_cuda:
                raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only: move the model with .cuda(); "
                                        "there is no CPU fallback")
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise _lib.Esmb200Error("esm_b200 expects contiguous fp32 master parameters")
        lib = _lib.load()

        def create(attn_blk: _ResidualBlock, ffn_blk: Optional[_ResidualBlock]):
            a = attn_blk.layer
            w = _lib.LayerWeights()
            w.embed_dim, w.num_heads, w.ffn_dim = self.embedding_dim, self.num_heads, self.ffn_embedding_dim
            w.ln_eps = attn_blk.layer_norm.eps
            w.precision = self.precision
            w.ln1_weight, w.ln1_bias = attn_blk.layer_norm.weight.data_ptr(), attn_blk.layer_norm.bias.data_ptr()
            for n in ("q", "k", "v", "out"):
                lin = getattr(a, n + "_proj")
                setattr(w, n + "_weight", lin.weight.data_ptr())
                setattr(w, n + "_bias", lin.bias.data_ptr())
            if ffn_blk is not None:
                f = ffn_blk.layer
                w.ln2_weight, w.ln2_bias = ffn_blk.layer_norm.weight.data_ptr(), ffn_blk.layer_norm.bias.data_ptr()
                w.fc1_weight, w.fc1_bias = f.fc1.weight.data_ptr(), f.fc1.bias.data_ptr()
                w.fc2_weight, w.fc2_bias = f.fc2.weight.data_ptr(), f.fc2.bias.data_ptr()
            out = ctypes.c_void_p()
            with torch.cuda.device(ps[0].device):
                _lib.check(lib.esmb200_layer_create(ctypes.byref(w), _stream(), ctypes.byref(out)))
            return out

        row = create(self.row_self_attention, None)
        col = create(self.column_self_attention, self.feed_forward_layer)
        self._handles, self._handles_key = (row, col), key
        return self._handles

    def release(self):
        if self._handles is not None:
            lib = _lib.load()
            for h in self._handles:
                lib.esmb200_layer_destroy(h)
            self._handles, self._handles_key = None, None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    @torch.no_grad()
    def forward(self, x: torch.Tensor, self_attn_mask: Optional[torch.Tensor] = None,
                self_attn_padding_mask: Optional[torch.Tensor] = None, need_head_weights: bool = False):
        """x: (R, C, B, E) like the reference (modules.py:195-221); self_attn_padding_mask: (B, R, C) bool.
        Returns x, or (x, column_attn, row_attn)."""
        if self_attn_mask is not None:
            raise NotImplementedError
        if not x.is_cuda:
            raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
        R, C, B, E = x.shape
        xb = x.permute(2, 0, 1, 3).contiguous().float()  # [B,R,C,E], updated in place by the residual epilogues
        row_probs, col_probs = self.forward_batch_major(xb, self_attn_padding_mask, need_head_weights)
        out = xb.permute(1, 2, 0, 3).to(x.dtype)
        if need_head_weights:
            return out, col_probs, row_probs
        return out

    @torch.no_grad()
    def forward_batch_major(self, xb: torch.Tensor, padding_mask: Optional[torch.Tensor] = None,
                            need_probs: bool = False):
        """In-place layer on the batch-major residual stream xb [B,R,C,E] fp32 (what MSATransformer keeps between
        layers), one esmb200_axial_stack_forward call.  padding_mask [B,R,C] bool or None.  Returns (row_attn
        [H,B,C,C], column_attn [H,C,B,R,R]), the reference's layouts (axial_attention.py:87,206), or (None, None)."""
        if not need_probs:
            run_axial_stack([self], xb, padding_mask)
            return None, None
        B, R, C, _ = xb.shape
        col = torch.empty((B, C, self.num_heads, R, R), dtype=torch.float32, device=xb.device)
        row = run_axial_stack([self], xb, padding_mask, (0,), {0: col})[0]
        return row, col.permute(2, 1, 0, 3, 4).contiguous()


def run_axial_stack(layers: Sequence[AxialTransformerLayer], xb: torch.Tensor,
                    padding_mask: Optional[torch.Tensor] = None, row_attn_layers: Sequence[int] = (),
                    col_attn: Optional[Dict[int, torch.Tensor]] = None):
    """esmb200_axial_stack_forward on xb [B,R,C,E] fp32 in place (msa_transformer.py:190-201's loop).
    Returns {layer index: row attention [H,B,C,C] fp32} for the indices in row_attn_layers.  col_attn: {layer index:
    contiguous fp32 [B,C,H,R,R] buffer on xb's device}, filled with the column attention maps of those layers."""
    if not xb.is_cuda:
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
    assert xb.dtype == torch.float32 and xb.is_contiguous()
    lib = _lib.load()
    B, R, C, E = xb.shape
    n = len(layers)
    Fd, H = layers[0].ffn_embedding_dim, layers[0].num_heads
    dev = xb.device
    with torch.cuda.device(dev):
        hs = [l.handles() for l in layers]
        rows = (ctypes.c_void_p * n)(*[h[0] for h in hs])
        cols = (ctypes.c_void_p * n)(*[h[1] for h in hs])
        if layers[0].precision:  # every layer of one call shares the precision (EINVAL otherwise)
            nbytes = lib.esmb200_axial_workspace_bytes_split(E, Fd, B, R, C)
        else:
            nbytes = lib.esmb200_axial_workspace_bytes(E, Fd, B, R, C)
        ws = _workspace(nbytes, dev)
        pm = cm = None
        if padding_mask is not None:
            pm = padding_mask.to(device=dev, dtype=torch.uint8).contiguous()
            assert pm.shape == (B, R, C)
            cm = pm.permute(0, 2, 1).contiguous()
        attns = (ctypes.c_void_p * n)()
        out = {}
        for i in row_attn_layers:
            out[i] = torch.empty((H, B, C, C), dtype=torch.float32, device=dev)
            attns[i] = out[i].data_ptr()
        col_ptrs = (ctypes.c_void_p * n)()
        for i, t in (col_attn or {}).items():
            assert t.shape == (B, C, H, R, R) and t.dtype == torch.float32 and t.is_contiguous() and t.device == dev
            col_ptrs[i] = t.data_ptr()
        _lib.check(lib.esmb200_axial_stack_forward(rows, cols, n, _ptr(xb), _ptr(pm), _ptr(cm), B, R, C,
                                                   attns if row_attn_layers else None, col_ptrs if col_attn else None,
                                                   _ptr(ws), ws.numel(), _stream()))
    return out


class LearnedPositionalEmbedding(nn.Embedding):
    """Parameter container with the reference's shape (modules.py:224-239: max_positions + padding_idx + 1 rows);
    the lookup itself is part of esmb200_msa_embed (MSA Transformer) or esmb200_esm1b_embed (ESM-1b / ESM-1v)."""

    def __init__(self, num_embeddings: int, embedding_dim: int, padding_idx: int):
        super().__init__(num_embeddings + padding_idx + 1, embedding_dim, padding_idx)
        self.max_positions = num_embeddings


class MSATransformer(nn.Module):
    """Drop-in for esm.model.msa_transformer.MSATransformer (msa_transformer.py:20-238) at inference: same
    constructor (`args` namespace + alphabet), same state-dict keys, same forward contract
    `model(tokens [B,R,C], repr_layers, need_head_weights, return_contacts)` -> dict with `logits`,
    `representations`, and — when asked — `row_attentions`, `col_attentions`, `contacts`.

    `return_contacts=True` implies `need_head_weights=True` like the reference (msa_transformer.py:149-150), i.e. the
    result also carries `col_attentions` [B,L,H,C,R,R] (4.8 GB for a 128 x 512 MSA).  `predict_contacts()` — which only
    returns the contacts — skips the column maps; set `model.contacts_without_col_attentions = True` to get the same
    saving from `model(tokens, return_contacts=True)`."""

    def __init__(self, args: Union[Namespace, dict, None] = None, alphabet: Union[Alphabet, str] = "MSA Transformer",
                 **kwargs):
        super().__init__()
        if args is None:
            args = Namespace(**kwargs)
        elif isinstance(args, dict):
            args = Namespace(**args)
        defaults = dict(layers=12, embed_dim=768, ffn_embed_dim=3072, attention_heads=12, max_positions=1024,
                        embed_positions_msa=True)
        for k, v in defaults.items():
            if not hasattr(args, k):
                setattr(args, k, v)
        self.args = args
        if isinstance(alphabet, str):
            alphabet = Alphabet.from_architecture(alphabet)
        self.alphabet = alphabet
        self.alphabet_size = len(alphabet)
        self.padding_idx = alphabet.padding_idx
        self.mask_idx = alphabet.mask_idx
        self.cls_idx = alphabet.cls_idx
        self.eos_idx = alphabet.eos_idx
        self.prepend_bos = alphabet.prepend_bos
        self.append_eos = alphabet.append_eos
        E = args.embed_dim
        self.embed_tokens = nn.Embedding(self.alphabet_size, E, padding_idx=self.padding_idx)
        if getattr(args, "embed_positions_msa", False):
            emb_dim = getattr(args, "embed_positions_msa_dim", E)
            self.msa_position_embedding = nn.Parameter(0.01 * torch.randn(1, 1024, 1, emb_dim))
        else:
            self.register_parameter("msa_position_embedding", None)
        self.layers = nn.ModuleList([AxialTransformerLayer(E, args.ffn_embed_dim, args.attention_heads)
                                     for _ in range(args.layers)])
        self.contact_head = ContactPredictionHead(args.layers * args.attention_heads, self.prepend_bos,
                                                  self.append_eos, eos_idx=self.eos_idx)
        self.embed_positions = LearnedPositionalEmbedding(args.max_positions, E, self.padding_idx)
        self.emb_layer_norm_before = nn.LayerNorm(E)
        self.emb_layer_norm_after = nn.LayerNorm(E)
        self.lm_head = RobertaLMHead(embed_dim=E, output_dim=self.alphabet_size, weight=self.embed_tokens.weight)
        self.precision = "fp16"

    contacts_without_col_attentions = False  # True: return_contacts alone does not materialise col_attentions

    PRECISIONS = {"fp16": 0, "fp32x3": 1}

    def set_precision(self, name: str) -> "MSATransformer":
        """"fp16" (default): fp16 MMA operands, fp32 accumulation — the fast path.
        "fp32x3": every MMA operand of the axial stack and the LM head (LayerNorm outputs, weights, q, k, v, the tied
        row-attention and column-attention probabilities, context, FFN hidden) is an fp16 hi + lo pair and every product
        runs hi*hi + lo*hi + hi*lo into the fp32 accumulator: fp32-grade parity with the reference at several times the
        tensor work (DESIGN.md sections 4 and 6)."""
        if name not in self.PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(self.PRECISIONS)}")
        self.precision = name
        for layer in self.layers:
            layer.precision = self.PRECISIONS[name]
        return self

    @property
    def num_layers(self) -> int:
        return self.args.layers

    def max_tokens_per_msa_(self, value: int) -> None:
        """Accepted for API compatibility (msa_transformer.py:228-238): the reference chunks its attention above
        `max_tokens_per_msa` to bound memory; the kernels here never materialise per-row score tensors."""

    @torch.no_grad()
    def forward(self, tokens, repr_layers=[], need_head_weights=False, return_contacts=False):
        if return_contacts and not self.contacts_without_col_attentions:
            need_head_weights = True  # msa_transformer.py:149-150
        repr_layers = set(repr_layers)
        tokens, x, hidden, row_attn, col_attn = self._stack(tokens, repr_layers, need_head_weights, return_contacts)
        lib = _lib.load()
        B, R, C = tokens.shape
        E, N = self.args.embed_dim, self.args.layers
        want_rows = need_head_weights or return_contacts
        dev = tokens.device
        with torch.cuda.device(dev):
            ln = self.emb_layer_norm_after
            logits = self.lm_head.forward_native(x.view(B, R * C, E), ln.weight, ln.bias, ln.eps,
                                                 self.PRECISIONS[self.precision]).view(B, R, C, -1)
            _lib.check(lib.esmb200_layernorm(_ptr(x), _ptr(ln.weight), _ptr(ln.bias), _ptr(x), B * R * C, E, ln.eps,
                                             _stream()))
        if N in repr_layers:
            hidden[N] = x  # the last representation is post-LayerNorm (msa_transformer.py:204-209)
        result = {"logits": logits, "representations": hidden}
        if want_rows:
            # H,B,C,C per layer -> B,L,H,C,C (msa_transformer.py:196-197,215)
            row_attentions = torch.stack([row_attn[i].permute(1, 0, 2, 3) for i in range(N)], 1)
            result["row_attentions"] = row_attentions
            if need_head_weights:
                # B,C,H,R,R per layer -> B,L,H,C,R,R
                result["col_attentions"] = torch.stack([col_attn[i].permute(0, 2, 1, 3, 4) for i in range(N)], 1)
            if return_contacts:
                result["contacts"] = self.contact_head(tokens, row_attentions)
        return result

    def _lm_head_rows(self, x_rows: torch.Tensor) -> torch.Tensor:
        """The LM head (msa_transformer.py:204-210) on selected rows [n,E] of the pre-LN stream: fp32 logits [n,V]."""
        ln = self.emb_layer_norm_after
        return self.lm_head.forward_native(x_rows.unsqueeze(0), ln.weight, ln.bias, ln.eps,
                                           self.PRECISIONS[self.precision])[0]

    def _stack(self, tokens, repr_layers=frozenset(), need_head_weights=False, return_contacts=False):
        """The stack step of `forward` (msa_transformer.py:147-201): embedding prologue and the axial layers.
        Returns (tokens contiguous, x, hidden, row_attn, col_attn): x is the fp32 residual stream [B,R,C,E] BEFORE
        emb_layer_norm_after, hidden {i: representation} for the requested layers below num_layers, row_attn
        {layer: [H,B,C,C]} and col_attn {layer: [B,C,H,R,R]} when the maps are asked for."""
        assert tokens.ndim == 3
        if not tokens.is_cuda:
            raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only: pass tokens.cuda(); no CPU fallback")
        lib = _lib.load()
        tokens = tokens.contiguous()
        B, R, C = tokens.shape
        E, N, H = self.args.embed_dim, self.args.layers, self.args.attention_heads
        if C > self.embed_positions.max_positions:  # modules.py:243-247
            raise ValueError(f"Sequence length {C} above maximum  sequence length of {self.embed_positions.max_positions}")
        mp = self.msa_position_embedding
        if mp is not None and R > 1024:           # msa_transformer.py:158-163
            raise RuntimeError("Using model with MSA position embedding trained on maximum MSA "
                               f"depth of 1024, but received {R} alignments.")
        padding_mask = tokens.eq(self.padding_idx)  # B, R, C
        if not bool(padding_mask.any()):            # msa_transformer.py:152-153
            padding_mask = None
        repr_layers = set(repr_layers)
        hidden: Dict[int, torch.Tensor] = {}
        want_rows = need_head_weights or return_contacts
        dev = tokens.device
        with torch.cuda.device(dev):
            x = torch.empty((B, R, C, E), dtype=torch.float32, device=dev)
            ln = self.emb_layer_norm_before
            _lib.check(lib.esmb200_msa_embed(_ptr(tokens), _ptr(self.embed_tokens.weight),
                                             _ptr(self.embed_positions.weight), _ptr(mp),
                                             mp.shape[-1] if mp is not None else 0, _ptr(ln.weight), _ptr(ln.bias),
                                             ln.eps, _ptr(x), B, R, C, E, self.padding_idx, _stream()))
            if 0 in repr_layers:
                hidden[0] = x.clone()
            row_attn: Dict[int, torch.Tensor] = {}
            col_attn = {i: torch.empty((B, C, H, R, R), dtype=torch.float32, device=dev)
                        for i in range(N)} if need_head_weights else {}
            # whole segments of the stack per C-ABI call, split at the requested representations
            stops = sorted({i for i in repr_layers if 0 < i < N} | {N})
            start = 0
            for stop in stops:
                idx = list(range(start, stop))
                got = run_axial_stack([self.layers[i] for i in idx], x, padding_mask,
                                      list(range(len(idx))) if want_rows else (),
                                      {k: col_attn[i] for k, i in enumerate(idx)} if need_head_weights else None)
                for k, t in got.items():
                    row_attn[start + k] = t
                if stop < N:
                    hidden[stop] = x.clone()
                start = stop
        return tokens, x, hidden, row_attn, col_attn

    def _stack_unpadded(self, tokens: torch.Tensor) -> torch.Tensor:
        """`_stack` for contiguous tokens [B,R,C] on the device that the caller has checked hold no <pad> and fit the
        position embeddings: the embedding prologue and one axial-stack call without a padding mask. It never reads
        tokens back to the host, so loops over it (sampling.msa_gibbs) do not synchronise. Returns the fp32 residual
        stream [B,R,C,E] before emb_layer_norm_after."""
        lib = _lib.load()
        B, R, C = tokens.shape
        E = self.args.embed_dim
        mp = self.msa_position_embedding
        dev = tokens.device
        with torch.cuda.device(dev):
            x = torch.empty((B, R, C, E), dtype=torch.float32, device=dev)
            ln = self.emb_layer_norm_before
            _lib.check(lib.esmb200_msa_embed(_ptr(tokens), _ptr(self.embed_tokens.weight),
                                             _ptr(self.embed_positions.weight), _ptr(mp),
                                             mp.shape[-1] if mp is not None else 0, _ptr(ln.weight), _ptr(ln.bias),
                                             ln.eps, _ptr(x), B, R, C, E, self.padding_idx, _stream()))
            run_axial_stack(list(self.layers), x)
        return x

    def predict_contacts(self, tokens):
        """msa_transformer.py:222-223; only the contacts are returned, so the column attention maps are not built."""
        prev = self.contacts_without_col_attentions
        self.contacts_without_col_attentions = True
        try:
            return self(tokens, return_contacts=True)["contacts"]
        finally:
            self.contacts_without_col_attentions = prev
