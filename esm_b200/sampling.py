"""Sequence generation from a masked protein language model (ESM-2, ESM-1b, ESM-1v) by Gibbs sampling: batched chains,
block updates of the designable positions in a random order per sweep, and a counter-based random stream, so that a
sample depends only on (seed, chain, step, position).

    from esm_b200 import sampling
    out = sampling.gibbs(model, tokens, positions=None, chains=1, sweeps=1, block=1, temperature=1.0, seed=0,
                         max_tokens=None)
    out["tokens"]   # int64 [C, T] on the model's device
    out["logp"]     # fp32 [C, steps]

Definition. tokens [1, T] is one protein with <cls> first, <eos> last and no padding; residues sit at token positions
1 ... L. positions D (residue indices in [0, L), distinct; default all) are designable, every other residue is fixed
and never changes, whatever token it holds. A <mask> is allowed at a designable position only, so `<cls> <mask>*L
<eos>` starts de novo generation. Only the 20 amino acids AA = jacobian.AMINO_ACIDS are sampled. Every chain starts
from tokens. k = min(block, |D|).

R(c0, c1, c2, c3) is Philox4x32-10 with counter (c0, c1, c2, c3) and key (seed mod 2^32, seed >> 32); a word r gives
the uniform u = ((r >> 8) + 0.5) * 2^-24, rounded toward zero to fp32 (exact for u < 1/2, always in (0, 1)).

For each sweep w (0-based) and chain c (global index 0 ... C-1):
  1. Order: D sorted ascending by R(w, c, p, 0).x * 65536 + p, cut into consecutive blocks of k (the last one may be
     shorter, equally for every chain). Steps are the blocks, counted over all sweeps as s; there are
     W * ceil(|D| / k) of them.
  2. Step s: the chain's current tokens with <mask> at the block's positions run through the stack; the fp32 LM-head
     logits l at rows 1 + p of the block give, for each p and a < 20, z_a = fp32(l[AA_a] / temperature) and
     g_a = -logf(-logf(u_a)), u_a from word a mod 4 of R(s, c, p, 1 + a div 4). The new token is AA[a*],
     a* = argmax_a (z_a + g_a), a tie to the smallest a. All positions of the block are written together (a block
     update). log q = log_softmax(z)[a*], by esmb200_log_softmax_rows' formula: (z - max) - logf(sum expf(z - max)).
  3. In sweep 0 of a de novo start, positions not yet visited are still <mask> when their neighbours are drawn
     (iterative decoding in random order); after sweep 0 no designable position holds <mask>.
logp[c, s] is the sum of step s's log q in block order (fp32).

The chains run in chunks of at most `max_tokens` tokens (variants._copies_per_chunk, at least one chain); each chunk
runs all its sweeps. A step is one stack call on the chunk's masked copies, the LM head on the block rows only, then
esmb200_sample_rows, which draws the tokens and writes them into the chains' device state in place. The order of a
sweep is esmb200_sample_order's keys sorted on the device. Nothing in the sweep loop waits for the host. The stack is
batch-invariant and every draw depends only on (seed, chain, step, position), so the result is the same bits for
every max_tokens.

Cost: each step is one stack call on C copies of T tokens (in chunks); the sampler kernel and the head on C k rows
are small beside it.
"""
from __future__ import annotations

import ctypes
import math
import numbers
from typing import Dict, Optional, Sequence

import torch

from . import _lib
from .jacobian import _amino_acid_offset, _framed_protein
from .model import ProteinLanguageModel, _ptr, _stream
from .variants import _copies_per_chunk, _device

_COUNTER = 1 << 32  # chains and steps are Philox counter words
_MAX_RESIDUES = 65535  # the order key holds the position in 16 bits


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
    chains, sweeps, block = _count("chains", chains), _count("sweeps", sweeps), _count("block", block)
    if chains > _COUNTER:
        raise ValueError(f"chains must be at most 2^32, got {chains}")
    k = min(block, pos.numel())
    if sweeps * -(-pos.numel() // k) > _COUNTER:
        raise ValueError("sweeps * ceil(|positions| / block) must be at most 2^32")
    t = float(temperature)
    if not math.isfinite(t) or t <= 0:
        raise ValueError(f"temperature must be finite and > 0, got {temperature!r}")
    t32 = ctypes.c_float(t).value
    if not (0 < t32 < math.inf):
        raise ValueError(f"temperature {temperature!r} is not a finite positive fp32 value")
    if isinstance(seed, bool) or not isinstance(seed, numbers.Integral) or not 0 <= seed < 1 << 64:
        raise ValueError(f"seed must be an integer in [0, 2^64), got {seed!r}")
    return host, pos, t32, chains, sweeps, block, int(seed)


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
    n = pos.numel()
    k = min(block, n)
    blocks = -(-n // k)
    steps = sweeps * blocks
    lib = _lib.load()
    dev = _device(model)
    if dev.type != "cuda":
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only: move the model to the GPU; no CPU fallback")
    tok, pos = host.to(dev), pos.to(dev)
    out = torch.empty((chains, T), dtype=torch.int64, device=dev)
    logp = torch.empty((chains, steps), dtype=torch.float32, device=dev)
    per = _copies_per_chunk(T, max_tokens)
    with torch.cuda.device(dev):
        for c0 in range(0, chains, per):
            m = min(per, chains - c0)
            state = out[c0:c0 + m]  # the chains' tokens, updated in place by esmb200_sample_rows
            state.copy_(tok.expand(m, T))
            row1 = torch.arange(m, device=dev).unsqueeze(1) * T + 1  # flat row of each copy's first residue
            for w in range(sweeps):
                keys = torch.empty((m, n), dtype=torch.int64, device=dev)
                _lib.check(lib.esmb200_sample_order(_ptr(pos), n, m, c0, w, seed, _ptr(keys), _stream()))
                order = keys.sort(dim=1).values.bitwise_and_(0xFFFF)  # key mod 65536 = the position
                for b in range(blocks):
                    s = w * blocks + b
                    blk = order[:, b * k:(b + 1) * k].contiguous()
                    kb = blk.shape[1]
                    batch = state.clone()
                    batch.scatter_(1, blk + 1, model.mask_idx)
                    x = model._stack(batch)[1]
                    logits = model._lm_head_rows(x.view(-1, x.shape[-1]).index_select(0, (row1 + blk).view(-1)))
                    logq = torch.empty(m * kb, dtype=torch.float32, device=dev)
                    _lib.check(lib.esmb200_sample_rows(_ptr(logits), logits.stride(0), m * kb, aa0, tau, seed, s, c0,
                                                       kb, _ptr(blk), _ptr(state), T, _ptr(logq),
                                                       _ptr(logp[c0:, s]), steps, _stream()))
    return {"tokens": out, "logp": logp}
