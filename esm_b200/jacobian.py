"""Categorical Jacobian of a masked protein language model, and the unsupervised contact map it gives (Zhang,
Wayment-Steele, Brixi, Wang, Kern & Ovchinnikov, PNAS 2024), for ESM-2, ESM-1b and ESM-1v.

    from esm_b200 import jacobian
    out = jacobian.categorical_jacobian(model, tokens, max_tokens=None, return_jacobian=False)
    out["contacts"]   # [L, L] fp32
    out["jacobian"]   # [L, 20, L, 20] fp32, only with return_jacobian=True

Definition, for one protein: tokens [1, T] with <cls> first, <eos> last and no padding; residues at token positions
1 ... L, L = T - 2 >= 2; AA = AMINO_ACIDS, the alphabet's 20 canonical tokens in alphabet order; logits(x) the fp32
LM-head output forward(x)["logits"].
  1. f_wt[j, b] = logits(x)[1 + j, AA[b]].
  2. x^(ia) is x with token 1 + i set to AA[a]; J[i, a, j, b] = logits(x^(ia))[1 + j, AA[b]] - f_wt[j, b]. Identity
     substitutions (AA[a] equal to the wild-type token) are not run: their rows are exactly +0, the rows running them
     would give, since the stack is batch-invariant. A non-canonical wild-type residue (X, B, ...) has no identity
     substitution, so all 20 copies run at its position.
  3-6. The contact map: J centred along each of its four axes, N[i, j] = the Frobenius norm of the 20 x 20 block
     (i, j) with N[i, i] = 0, APC (esm/modules.py:32-41) with the diagonal zeroed again, then (A + A^T) / 2. This runs
     on the GPU in esmb200_jacobian_contacts (include/esmb200.h), without a centred copy of J.

The substitution copies, ordered by (i, a) row-major without the identities, are built on the device and run through
the stack in chunks of at most `max_tokens` tokens (variants._copies_per_chunk): one stack call per chunk, then the LM
head on the chunk's whole residual stream, as forward runs it. A copy's rows do not depend on the other copies of its
chunk, so J is the same bits for every `max_tokens` and equals model(x^(ia))["logits"] - model(x)["logits"] on those
rows and columns.

Cost: J is held on the device, 1,600 L^2 bytes (1.67 GB at L = 1022, 14.4 GB at L = 3000), plus one chunk's stack
workspace and the contact pass's scratch (esmb200_jacobian_scratch_bytes, about 1/25 of J). The stack runs about
19 L copies of L + 2 tokens: the Jacobian's work is that many forwards.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _lib
from .model import ProteinLanguageModel, _ptr, _stream
from .variants import _copies_per_chunk, _device

AMINO_ACIDS = "LAGVSERTIDPKQNFYMHWC"


def jacobian_contacts(jac: torch.Tensor) -> torch.Tensor:
    """Contact map [L, L] fp32 of a categorical Jacobian jac [L, 20, L, 20] (fp32, contiguous, on the GPU) by steps
    3-6 of the definition (esmb200_jacobian_contacts). jac is not modified."""
    if not jac.is_cuda:
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
    if jac.dtype != torch.float32 or jac.dim() != 4 or jac.shape[1] != 20 or jac.shape[3] != 20 \
            or jac.shape[0] != jac.shape[2] or not jac.is_contiguous():
        raise ValueError("jac must be a contiguous fp32 [L, 20, L, 20] tensor")
    L = jac.shape[0]
    if L < 2:
        raise ValueError(f"the contact map needs at least 2 residues, got {L}")
    lib = _lib.load()
    with torch.cuda.device(jac.device):
        nbytes = lib.esmb200_jacobian_scratch_bytes(L)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=jac.device)
        out = torch.empty((L, L), dtype=torch.float32, device=jac.device)
        _lib.check(lib.esmb200_jacobian_contacts(_ptr(jac), L, _ptr(scratch), nbytes, _ptr(out), _stream()))
    return out


def _amino_acid_offset(model) -> int:
    """Token id of AMINO_ACIDS[0]; the 20 follow it in alphabet order (ids 4 ... 23 in the ESM-1b / ESM-2 alphabet)."""
    ids = [model.alphabet.get_idx(c) for c in AMINO_ACIDS]
    if ids != list(range(ids[0], ids[0] + len(AMINO_ACIDS))):
        raise ValueError(f"the model's alphabet does not hold {AMINO_ACIDS} as consecutive tokens")
    return ids[0]


def _check(model, tokens) -> torch.Tensor:
    """The refusals of categorical_jacobian, all before any launch. Returns tokens as int64 [1, T] on the host."""
    from .msa import MSATransformer
    if isinstance(model, MSATransformer):
        raise ValueError("categorical_jacobian runs ESM-2, ESM-1b and ESM-1v; the MSA Transformer is not supported")
    if not isinstance(model, ProteinLanguageModel):
        raise ValueError(f"categorical_jacobian needs an ESM2 or ProteinBertModel, got {type(model).__name__}")
    if model.precision == "fp8":
        raise ValueError("categorical_jacobian refuses fp8 precision: its logits carry about 5 % relative error, more "
                         "than the substitution effects the Jacobian measures; use fp16 or fp32x3")
    return _framed_protein(model, tokens, "the categorical Jacobian")


def _framed_protein(model, tokens, what: str) -> torch.Tensor:
    """The framing checks the categorical Jacobian and the sampler share, before any launch: tokens is one unpadded
    protein [1, T] of integers with <cls> first, <eos> last and at least 2 residues (`what` names the caller in the
    last message). Returns tokens as int64 [1, T] on the host."""
    tokens = torch.as_tensor(tokens)
    if tokens.dtype.is_floating_point or tokens.dtype == torch.bool:
        raise ValueError(f"tokens must be an integer tensor, got {tokens.dtype}")
    if tokens.dim() != 2 or tokens.shape[0] != 1:
        raise ValueError(f"tokens must be one protein [1, T], got shape {tuple(tokens.shape)}")
    tokens = tokens.cpu().long()
    if bool(tokens.eq(model.padding_idx).any()):
        raise ValueError("tokens must not contain padding")
    T = tokens.shape[1]
    if T < 2 or int(tokens[0, 0]) != model.cls_idx or int(tokens[0, -1]) != model.eos_idx:
        raise ValueError("tokens must start with <cls> and end with <eos>")
    if T - 2 < 2:
        raise ValueError(f"{what} needs at least 2 residues, got {T - 2}")
    return tokens


def _substitution_rows(model, tokens: torch.Tensor, copies: torch.Tensor, aa0: int) -> torch.Tensor:
    """Logits [m, L, 20] (residue rows, AMINO_ACIDS columns) of the copies of tokens [1, T] (on the model's device)
    with token 1 + copies[k] // 20 set to aa0 + copies[k] % 20: one stack call, then the LM head on the whole residual
    stream of the batch."""
    m, T = copies.numel(), tokens.shape[1]
    batch = tokens.expand(m, T).clone()
    batch[torch.arange(m, device=tokens.device), copies // 20 + 1] = copies % 20 + aa0
    x = model._stack(batch)[1]
    E = x.shape[-1]
    with torch.cuda.device(x.device):
        logits = model._lm_head_rows(x.view(-1, E))
    return logits.view(m, T, -1)[:, 1:T - 1, aa0:aa0 + 20]


@torch.no_grad()
def categorical_jacobian(model, tokens: torch.Tensor, max_tokens: Optional[int] = None,
                         return_jacobian: bool = False) -> Dict[str, torch.Tensor]:
    """The categorical Jacobian of `model` (ESM2 or ProteinBertModel: ESM-1b, ESM-1v; resident or cpu_offload(),
    fp16 or fp32x3 precision, also after model.half()) at one protein tokens [1, T], and its contact map.
    Returns {"contacts": [L, L] fp32} and, with return_jacobian, "jacobian": J [L, 20, L, 20] fp32 (module docstring).
    Chunks hold at most `max_tokens` tokens (default variants.DEFAULT_MAX_TOKENS), at least one copy; the result does
    not depend on it. Refused with ValueError before any launch: the MSA Transformer, fp8 precision, tokens that are not
    one unpadded protein framed by <cls> and <eos>, and fewer than 2 residues."""
    host = _check(model, tokens)
    aa0 = _amino_acid_offset(model)
    T = host.shape[1]
    L = T - 2
    flat = torch.arange(20 * L)
    copies = flat[host[0, 1 + flat // 20] != aa0 + flat % 20]  # (i, a) row-major, identities skipped
    dev = _device(model)
    tok = host.to(dev)
    x = model._stack(tok)[1]  # the wild type: forward(x)["logits"] on the residue rows and amino-acid columns
    with torch.cuda.device(x.device):
        f_wt = model._lm_head_rows(x.view(-1, x.shape[-1]))[1:T - 1, aa0:aa0 + 20]
    copies = copies.to(dev)
    jac = torch.zeros((20 * L, L, 20), dtype=torch.float32, device=dev)
    k = _copies_per_chunk(T, max_tokens)
    for s in range(0, copies.numel(), k):
        idx = copies[s:s + k]
        jac.index_copy_(0, idx, _substitution_rows(model, tok, idx, aa0) - f_wt)
    jac = jac.view(L, 20, L, 20)
    out = {"contacts": jacobian_contacts(jac)}
    if return_jacobian:
        out["jacobian"] = jac
    return out
