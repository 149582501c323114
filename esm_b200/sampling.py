"""Gibbs sampling from a masked protein language model: sequences from ESM-2, ESM-1b and ESM-1v, alignments from the
MSA Transformer. Batched chains, block updates of the designable entries in a random order per sweep, and a
counter-based random stream, so that a sample depends only on (seed, chain, step, entry).

    from esm_b200 import sampling
    out = sampling.gibbs(model, tokens, positions=None, chains=1, sweeps=1, block=1, temperature=1.0, seed=0,
                         max_tokens=None)
    out["tokens"]   # int64 [chains, T] on the model's device
    out["logp"]     # fp32 [chains, steps]
    out = sampling.msa_gibbs(model, tokens, designable=None, chains=1, sweeps=1, block=1, temperature=1.0, seed=0,
                             gaps=True, max_tokens=None)
    out["tokens"]   # int64 [chains, R, C] on the model's device
    out["logp"]     # fp32 [chains, steps]

Definition. A chain is an alignment of R rows and C columns whose column 0 is <cls>. Its residue entries (r, j),
1 <= j < C, have the flat index p = r * (C - 1) + (j - 1) < 2^20. The designable entries D are resampled, every other
entry is fixed and never changes, whatever token it holds; a <mask> is allowed at a designable entry only. The drawable
tokens A are a list of token ids. Every chain starts from tokens. k = min(block, |D|).

R(c0, c1, c2, c3) is Philox4x32-10 with counter (c0, c1, c2, c3) and key (seed mod 2^32, seed >> 32); a word r gives
the uniform u = ((r >> 8) + 0.5) * 2^-24, rounded toward zero to fp32 (exact for u < 1/2, always in (0, 1)).

For each sweep w (0-based) and chain c (global index 0 ... chains-1):
  1. Order: D sorted ascending by R(w, c, p, 0).x * 2^20 + p, cut into consecutive blocks of k (the last one may be
     shorter, equally for every chain). Steps are the blocks, counted over all sweeps as s; there are
     sweeps * ceil(|D| / k) of them.
  2. Step s: the chain's current tokens with <mask> at the block's entries run through the stack; the fp32 LM-head
     logits l at those entries give, for each p and a < |A|, z_a = fp32(l[A_a] / temperature) and
     g_a = -logf(-logf(u_a)), u_a from word a mod 4 of R(s, c, p, 1 + a div 4). The new token is A[a*],
     a* = argmax_a (z_a + g_a), a tie to the smallest a. All entries of the block are written together (a block
     update). log q = log_softmax(z)[a*], by esmb200_log_softmax_rows' formula: (z - max) - logf(sum expf(z - max)).
  3. In sweep 0 of a de novo start, entries not yet visited are still <mask> when their neighbours are drawn
     (iterative decoding in random order); after sweep 0 no designable entry holds <mask>.
logp[c, s] is the sum of step s's log q in block order (fp32).

Sequences (gibbs). tokens [1, T] is one protein with <cls> first, <eos> last and no padding, 2 ... 65535 residues at
token positions 1 ... L: the layout R = 1, C = T - 1, so entry p is residue p, token 1 + p, and <eos> is no entry.
positions D (residue indices in [0, L), distinct; default all) are designable, so `<cls> <mask>*L <eos>` starts de
novo generation. A is the 20 amino acids of jacobian.AMINO_ACIDS in that order.

Alignments (msa_gibbs). tokens [1, R, C] is one alignment in the MSA alphabet: column 0 of every row is <cls>, there is
no <pad> and no <eos>, R <= 1024 (the MSA position embedding) and 2 <= C <= max_positions. designable is None (every
entry) or bool [R, C - 1], so <mask> rows appended to a real alignment generate new family members. A is the 20 amino
acids of jacobian.AMINO_ACIDS in that order and, with gaps=True, the gap "-" as A[20].

Execution. The chains run in chunks of at most `max_tokens` tokens (variants._copies_per_chunk, at least one chain);
each chunk runs all its sweeps. The order of a sweep is esmb200_sample_order's keys sorted on the device. A step is one
stack call on the chunk's masked copies, the LM head on the block's entries only, then esmb200_sample_rows, which
draws the tokens and writes them into the chains' device state in place. Nothing in the sweep loop waits for the host:
the MSA Transformer's stack runs without a padding mask (MSATransformer._stack_unpadded). The stacks are
batch-invariant and every draw depends only on (seed, chain, step, entry), so the result is the same bits for every
max_tokens.

Cost: each step is one stack call on the chains' copies (in chunks); the sampler kernels and the head on the block's
entries are small beside it.
"""
from __future__ import annotations

import ctypes
import math
import numbers
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .jacobian import AMINO_ACIDS, _amino_acid_offset, _framed_protein
from .model import ProteinLanguageModel, _ptr, _stream
from .variants import _copies_per_chunk, _device

_COUNTER = 1 << 32  # chains and steps are Philox counter words
_MAX_RESIDUES = 65535  # gibbs' documented limit (its docstring, DESIGN.md section 1)
_MAX_MSA_ROWS = 1024  # the MSA position embedding
_MAX_ENTRIES = 1 << 20  # the order key holds the entry index in 20 bits


def _count(name: str, v) -> int:
    if isinstance(v, bool) or not isinstance(v, numbers.Integral):
        raise ValueError(f"{name} must be an integer, got {v!r}")
    if v < 1:
        raise ValueError(f"{name} must be >= 1, got {v}")
    return int(v)


def _check(model, tokens, positions, chains, sweeps, block, temperature, seed):
    """The refusals of gibbs, all before any launch. Returns (host tokens int64 [1, T], designable positions int64
    [n] on the host, temperature as fp32, chains, sweeps, block, seed)."""
    from .msa import MSATransformer
    if isinstance(model, MSATransformer):
        raise ValueError("gibbs samples ESM-2, ESM-1b and ESM-1v; the MSA Transformer is not supported")
    if not isinstance(model, ProteinLanguageModel):
        raise ValueError(f"gibbs needs an ESM2 or ProteinBertModel, got {type(model).__name__}")
    host = _framed_protein(model, tokens, "sampling")
    L = host.shape[1] - 2
    if L > _MAX_RESIDUES:
        raise ValueError(f"sampling takes at most {_MAX_RESIDUES} residues, got {L}")
    if positions is None:
        pos = torch.arange(L)
    else:
        pos = torch.as_tensor(positions)
        if pos.numel() == 0:
            raise ValueError("positions must not be empty")
        if pos.dtype.is_floating_point or pos.dtype == torch.bool:
            raise ValueError(f"positions must be integers, got {pos.dtype}")
        pos = pos.cpu().long().reshape(-1)
        if not bool(((pos >= 0) & (pos < L)).all()):
            raise ValueError(f"positions must lie in [0, {L})")
        if pos.unique().numel() != pos.numel():
            raise ValueError("positions must be distinct")
    fixed = torch.ones(L, dtype=torch.bool)
    fixed[pos] = False
    if bool((host[0, 1:L + 1][fixed] == model.mask_idx).any()):
        raise ValueError("a <mask> token may only sit at a designable position")
    return (host, pos) + _check_run(pos.numel(), "positions", chains, sweeps, block, temperature, seed)


def _check_run(n, what, chains, sweeps, block, temperature, seed):
    """The checks gibbs and msa_gibbs share for n designable `what`: counts, the Philox counter ranges of chains and
    steps, temperature and seed. Returns (temperature as fp32, chains, sweeps, block, seed)."""
    chains, sweeps, block = _count("chains", chains), _count("sweeps", sweeps), _count("block", block)
    if chains > _COUNTER:
        raise ValueError(f"chains must be at most 2^32, got {chains}")
    k = min(block, n)
    if sweeps * -(-n // k) > _COUNTER:
        raise ValueError(f"sweeps * ceil(|{what}| / block) must be at most 2^32")
    t = float(temperature)
    if not math.isfinite(t) or t <= 0:
        raise ValueError(f"temperature must be finite and > 0, got {temperature!r}")
    t32 = ctypes.c_float(t).value
    if not (0 < t32 < math.inf):
        raise ValueError(f"temperature {temperature!r} is not a finite positive fp32 value")
    if isinstance(seed, bool) or not isinstance(seed, numbers.Integral) or not 0 <= seed < 1 << 64:
        raise ValueError(f"seed must be an integer in [0, 2^64), got {seed!r}")
    return t32, chains, sweeps, block, int(seed)


@torch.no_grad()
def gibbs(model, tokens: torch.Tensor, positions: Optional[Sequence[int]] = None, chains: int = 1, sweeps: int = 1,
          block: int = 1, temperature: float = 1.0, seed: int = 0,
          max_tokens: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Gibbs sampling from `model` (ESM2 or ProteinBertModel: ESM-1b, ESM-1v; any precision, resident or
    cpu_offload()) started at one protein tokens [1, T], by the definition in the module docstring. Returns
    {"tokens": int64 [chains, T], "logp": fp32 [chains, sweeps * ceil(n / block)]} on the model's device, n the number
    of designable positions. The result does not depend on max_tokens (default variants.DEFAULT_MAX_TOKENS tokens per
    stack call, at least one chain). Refused with ValueError before any launch: the MSA Transformer, tokens that are
    not one unpadded protein framed by <cls> and <eos> of 2 ... 65535 residues, a <mask> at a fixed position, empty,
    out-of-range or repeated positions, chains, sweeps or block below 1, a temperature that is not finite and > 0, and
    a seed outside [0, 2^64)."""
    host, pos, tau, chains, sweeps, block, seed = _check(model, tokens, positions, chains, sweeps, block, temperature,
                                                         seed)
    aa0 = _amino_acid_offset(model)
    T = host.shape[1]
    amino_acids = list(range(aa0, aa0 + len(AMINO_ACIDS)))
    return _sweep(model, host, pos, amino_acids, (1, T - 1, T), lambda b: model._stack(b)[1], tau, chains, sweeps,
                  block, seed, max_tokens)


def _check_msa(model, tokens, designable, chains, sweeps, block, temperature, seed):
    """The refusals of msa_gibbs, all before any launch. Returns (host tokens int64 [1, R, C], designable entries p
    int64 [n] ascending on the host, temperature as fp32, chains, sweeps, block, seed)."""
    from .msa import MSATransformer
    if isinstance(model, ProteinLanguageModel):
        raise ValueError("msa_gibbs samples alignments from the MSA Transformer; for ESM-2, ESM-1b and ESM-1v use "
                         "sampling.gibbs")
    if not isinstance(model, MSATransformer):
        raise ValueError(f"msa_gibbs needs an MSATransformer, got {type(model).__name__}")
    host = torch.as_tensor(tokens)
    if host.dtype.is_floating_point or host.dtype == torch.bool:
        raise ValueError(f"tokens must be an integer tensor, got {host.dtype}")
    if host.dim() != 3 or host.shape[0] != 1:
        raise ValueError(f"tokens must be one alignment [1, R, C], got shape {tuple(host.shape)}")
    host = host.cpu().long()
    _, R, C = host.shape
    if C < 2:
        raise ValueError(f"an alignment needs C >= 2 columns (<cls> and a residue), got {C}")
    if R > _MAX_MSA_ROWS:
        raise ValueError(f"msa_gibbs takes at most {_MAX_MSA_ROWS} rows, got {R}")
    if C > model.embed_positions.max_positions:
        raise ValueError(f"C = {C} is above the model's max_positions {model.embed_positions.max_positions}")
    if R * (C - 1) > _MAX_ENTRIES:
        raise ValueError(f"msa_gibbs takes at most 2^20 residue entries R * (C - 1), got {R * (C - 1)}")
    if bool((host == model.padding_idx).any()) or bool((host == model.eos_idx).any()):
        raise ValueError("tokens must be one unpadded alignment with no <pad> and no <eos>")
    if not bool((host[0, :, 0] == model.cls_idx).all()):
        raise ValueError("every row of the alignment must start with <cls>")
    if designable is None:
        des = torch.ones((R, C - 1), dtype=torch.bool)
    else:
        des = torch.as_tensor(designable)
        if des.dtype != torch.bool or tuple(des.shape) != (R, C - 1):
            raise ValueError(f"designable must be a bool tensor of shape [R, C - 1] = [{R}, {C - 1}], got "
                             f"{des.dtype} {tuple(des.shape)}")
        des = des.cpu()
        if not bool(des.any()):
            raise ValueError("designable must hold at least one True entry")
    if bool((host[0, :, 1:][~des] == model.mask_idx).any()):
        raise ValueError("a <mask> token may only sit at a designable entry")
    entries = des.reshape(-1).nonzero().reshape(-1)
    return (host, entries) + _check_run(entries.numel(), "designable", chains, sweeps, block, temperature, seed)


def _drawable(model, gaps: bool):
    """The token ids of A: the 20 amino acids in AMINO_ACIDS order, then "-" when gaps."""
    ids = [model.alphabet.get_idx(c) for c in AMINO_ACIDS + ("-" if gaps else "")]
    if len(set(ids)) != len(ids) or model.alphabet.unk_idx in ids:
        raise ValueError("the model's alphabet does not hold the 20 amino acids and the gap as distinct tokens")
    return ids


@torch.no_grad()
def msa_gibbs(model, tokens: torch.Tensor, designable: Optional[torch.Tensor] = None, chains: int = 1, sweeps: int = 1,
              block: int = 1, temperature: float = 1.0, seed: int = 0, gaps: bool = True,
              max_tokens: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Gibbs sampling from an MSATransformer (fp16 or fp32x3) started at one alignment tokens [1, R, C], by the
    definition in the module docstring. Returns {"tokens": int64 [chains, R, C], "logp": fp32 [chains, sweeps *
    ceil(n / block)]} on the model's device, n the number of designable entries. The result does not depend on
    max_tokens (default variants.DEFAULT_MAX_TOKENS tokens per stack call, at least one chain). Refused with ValueError
    before any launch: a sequence model (use gibbs), tokens that are not one alignment [1, R, C] with <cls> in column 0
    and no <pad> or <eos>, C < 2, R > 1024, C > max_positions, more than 2^20 residue entries (a model with
    max_positions above 1025), a <mask> at a fixed entry, a designable that is not bool [R, C - 1] with a True entry,
    chains, sweeps or block below 1, chains or steps above 2^32, a temperature that is not finite and > 0, and a seed
    outside [0, 2^64)."""
    host, entries, tau, chains, sweeps, block, seed = _check_msa(model, tokens, designable, chains, sweeps, block,
                                                                 temperature, seed)
    _, R, C = host.shape
    return _sweep(model, host, entries, _drawable(model, bool(gaps)), (R, C, R * C), model._stack_unpadded, tau,
                  chains, sweeps, block, seed, max_tokens)


def _sweep(model, host, entries, drawable, layout, stack, tau, chains, sweeps, block, seed, max_tokens):
    """The sweep loop of gibbs and msa_gibbs after their checks, by the definition in the module docstring. host: the
    start tokens [1, ...] of one chain; entries: the designable entries p int64 [n] on the host; drawable: the token ids
    of A; layout: (R, C, chain_stride), chain_stride the number of tokens of a chain; stack: the masked batch
    [m, ...] -> its pre-LN residual stream."""
    R, C, chain_stride = layout
    n = entries.numel()
    k = min(block, n)
    blocks = -(-n // k)
    steps = sweeps * blocks
    lib = _lib.load()
    dev = _device(model)
    if dev.type != "cuda":
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only: move the model to the GPU; no CPU fallback")
    tok, entries = host.to(dev), entries.to(dev)
    token_set = torch.tensor(drawable, dtype=torch.int32, device=dev)
    out = torch.empty((chains,) + tuple(host.shape[1:]), dtype=torch.int64, device=dev)
    logp = torch.empty((chains, steps), dtype=torch.float32, device=dev)
    per = _copies_per_chunk(chain_stride, max_tokens)
    with torch.cuda.device(dev):
        for c0 in range(0, chains, per):
            m = min(per, chains - c0)
            state = out[c0:c0 + m]  # the chains' tokens, updated in place by esmb200_sample_rows
            state.copy_(tok.expand_as(state))
            base = torch.arange(m, device=dev).unsqueeze(1) * chain_stride  # flat token of each copy's (0, 0)
            for w in range(sweeps):
                keys = torch.empty((m, n), dtype=torch.int64, device=dev)
                _lib.check(lib.esmb200_sample_order(_ptr(entries), n, m, c0, w, seed, _ptr(keys), _stream()))
                order = keys.sort(dim=1).values.bitwise_and_((1 << 20) - 1)  # key mod 2^20 = the entry
                for b in range(blocks):
                    s = w * blocks + b
                    blk = order[:, b * k:(b + 1) * k].contiguous()
                    kb = blk.shape[1]
                    # token (p / W) C + 1 + p % W of each copy, W = C - 1
                    flat = (base + blk + blk.div(C - 1, rounding_mode="floor") + 1).view(-1)
                    batch = state.clone()
                    batch.view(-1).index_fill_(0, flat, model.mask_idx)
                    x = stack(batch)
                    logits = model._lm_head_rows(x.view(-1, x.shape[-1]).index_select(0, flat))
                    logq = torch.empty(m * kb, dtype=torch.float32, device=dev)
                    _lib.check(lib.esmb200_sample_rows(_ptr(logits), logits.stride(0), m * kb, _ptr(token_set),
                                                       len(drawable), tau, seed, s, c0, kb, _ptr(blk), _ptr(state),
                                                       chain_stride, R, C, _ptr(logq), _ptr(logp[c0:, s]), steps,
                                                       _stream()))
    return {"tokens": out, "logp": logp}
