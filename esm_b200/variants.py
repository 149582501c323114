"""Variant-effect scoring on the library: the three scoring strategies of the reference's
examples/variant-prediction/predict.py, with its semantics, on batched masked copies.

    masked_marginals  predict.py:169-178 (MSA Transformer), :205-215 (ESM-2, ESM-1b / ESM-1v)
    wt_marginals      predict.py:192-194
    pseudo_ppl        compute_pppl, predict.py:118-144
    label_scores      label_row, predict.py:107-115
    read_msa          predict.py:21-42, without Biopython

predict.py runs one batch-1 forward per masked position (and, for pseudo-ppl, per mutant). Here the masked copies are
built on the device with integer tensor ops and run in chunks of at most `max_tokens` tokens (at least one copy per
chunk): one stack call per chunk, the LM head on the masked rows only (one row per copy; the other rows of a copy are
never projected onto the vocabulary), then esmb200_log_softmax_rows. A copy's rows do not depend on the other copies
of its chunk, so the result does not depend on `max_tokens`.

Reproduced as the reference has it (the command line must give predict.py's numbers):
  * pseudo_ppl masks token positions 1 ... len(sequence) - 2 and scores position i at the residue sequence[i], i.e.
    the token one to the right of the masked one; the last residue is never masked. The per-position fp32 values
    are summed as Python floats in position order.
  * label_scores reads position 1 + idx (the <cls> token comes first) and subtracts in fp32.

With `window`, masked_marginals, wt_marginals and pseudo_ppl score proteins longer than the model's window through the
overlapping windows of esm_b200.windows: a masked position gets one masked copy per window that covers it, the copies'
logit rows are merged with the windows' weights (esmb200_window_merge) and log_softmax runs on the merged row.
window=None is the unwindowed path, unchanged; a protein of at most `window` residues scores bit for bit as without it.
"""
from __future__ import annotations

import itertools
import re
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib, windows
from .model import _ptr, _stream

# Budget of one chunk, in tokens. Per token at E = 1280 (650M), one stack call needs its workspace
# (esmb200_workspace_bytes: 12,960 B per token at T = 1024) plus the fp32 residual stream (4 * E = 5,120 B): ~18 KB.
# 2^17 tokens are ~2.4 GB.
DEFAULT_MAX_TOKENS = 2 ** 17

WT_MISMATCH = "The listed wildtype does not match the provided sequence"  # predict.py:109,120


def log_softmax_rows(logits: torch.Tensor, target: Optional[torch.Tensor] = None) -> torch.Tensor:
    """torch.log_softmax(logits, -1) on fp32 CUDA rows [n, V] (V <= 64, unit column stride) via
    esmb200_log_softmax_rows. With target (int64 [n], values in [0, V)): the [n] log-probabilities of those columns."""
    if not logits.is_cuda:
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1:
        raise ValueError("logits must be fp32 [n, V] with unit column stride")
    n, V = logits.shape
    lib = _lib.load()
    with torch.cuda.device(logits.device):
        if target is not None:
            target = target.to(device=logits.device, dtype=torch.int64).contiguous()
            if target.shape != (n,):
                raise ValueError("target must be [n]")
            if n and not bool(((target >= 0) & (target < V)).all()):
                raise ValueError(f"targets must lie in [0, {V})")
            out = torch.empty((n,), dtype=torch.float32, device=logits.device)
        else:
            out = torch.empty((n, V), dtype=torch.float32, device=logits.device)
        _lib.check(lib.esmb200_log_softmax_rows(_ptr(logits), logits.stride(0) if n else V, n, V, _ptr(target),
                                                _ptr(out), _stream()))
    return out


def _device(model) -> torch.device:
    return next(model.parameters()).device


def _copies_per_chunk(tokens_per_copy: int, max_tokens: Optional[int]) -> int:
    budget = DEFAULT_MAX_TOKENS if max_tokens is None else int(max_tokens)
    return max(1, budget // tokens_per_copy)


def _head_rows(model, batch: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    """One stack call on `batch`, then the LM head on the flat row indices `rows` of its residual stream: fp32 [n,V]."""
    x = model._stack(batch)[1]
    E = x.shape[-1]
    with torch.cuda.device(x.device):
        return model._lm_head_rows(x.view(-1, E).index_select(0, rows))


@torch.no_grad()
def masked_marginals(model, tokens: torch.Tensor, positions: Optional[Sequence[int]] = None,
                     max_tokens: Optional[int] = None, window: Optional[int] = None) -> torch.Tensor:
    """Row k: log_softmax(logits) at positions[k] of the copy of `tokens` with positions[k] masked, fp32 [n, V].
    tokens [1, T] (ESM-2, ESM-1b / ESM-1v; predict.py:205-215) or [1, R, C] (MSA Transformer, predict.py:169-178: the
    mask goes at [0, 0, positions[k]] and the row is read from alignment row 0). positions default to all T (C).
    window (sequence models): the logits of each position merged over the windows that cover it."""
    if window is not None:
        window = windows.check_window(model, window)
    dev = _device(model)
    tokens = tokens.to(dev)
    if tokens.dim() not in (2, 3) or tokens.shape[0] != 1:
        raise ValueError("tokens must be one sequence [1, T] or one MSA [1, R, C]")
    per_copy = tokens[0].numel()
    L = tokens.shape[-1]
    if positions is None:
        positions = torch.arange(L)
    positions = torch.as_tensor(positions)
    if positions.dtype.is_floating_point or positions.dtype == torch.bool:
        raise TypeError(f"positions must be integers, got {positions.dtype}")
    positions = positions.to("cpu", torch.int64).view(-1)
    if positions.numel() and not bool(((positions >= 0) & (positions < L)).all()):
        raise ValueError(f"positions must lie in [0, {L})")
    if window is not None:
        if tokens.dim() != 2:
            raise ValueError("window applies to sequence models only: MSA windowing is not supported")
        return log_softmax_rows(_windowed_masked_logits(model, tokens, window, torch.zeros_like(positions),
                                                        positions, max_tokens))
    positions = positions.to(dev)
    k = _copies_per_chunk(per_copy, max_tokens)
    out = []
    for s in range(0, positions.numel(), k):
        pos = positions[s:s + k]
        m = pos.numel()
        batch = tokens.expand(m, *tokens.shape[1:]).clone()
        copy = torch.arange(m, device=dev)
        if tokens.dim() == 3:
            batch[copy, 0, pos] = model.mask_idx
        else:
            batch[copy, pos] = model.mask_idx
        out.append(log_softmax_rows(_head_rows(model, batch, copy * per_copy + pos)))
    if not out:
        return torch.empty((0, model.alphabet_size), dtype=torch.float32, device=dev)
    return torch.cat(out)


@torch.no_grad()
def wt_marginals(model, tokens: torch.Tensor, window: Optional[int] = None) -> torch.Tensor:
    """log_softmax(logits) of the unmasked sequence, fp32 [T, V] (predict.py:192-194). tokens [1, T].
    window: the logits merged over the windows (ProteinLanguageModel.forward_windowed)."""
    if window is not None:
        window = windows.check_window(model, window)
    tokens = tokens.to(_device(model))
    if tokens.dim() != 2 or tokens.shape[0] != 1:
        raise ValueError("tokens must be one sequence [1, T]")
    if window is not None:
        return log_softmax_rows(model._windowed(tokens, window)["logits"][0])
    x = model._stack(tokens)[1]
    with torch.cuda.device(x.device):
        return log_softmax_rows(model._lm_head_rows(x.view(-1, x.shape[-1])))


def parse_mutation(row: str, offset_idx: int = 0) -> Tuple[str, int, str]:
    """"AiB" -> (wild type "A", 0-based index i - offset_idx, mutant "B") (predict.py:108,119)."""
    return row[0], int(row[1:-1]) - offset_idx, row[-1]


def label_scores(token_log_probs: torch.Tensor, alphabet, sequence: str, mutations: Sequence[str],
                 offset_idx: int = 0) -> List[float]:
    """label_row (predict.py:107-115) for each mutation: lp[1 + idx, mt] - lp[1 + idx, wt] in fp32, as Python floats.
    token_log_probs [T, V] or [1, T, V]. Letters outside the alphabet count as <unk> (Alphabet.get_idx). A wild type
    that does not match `sequence` raises the reference's AssertionError."""
    lp = token_log_probs.detach()
    if lp.dim() == 3:
        lp = lp[0]
    lp = lp.float().cpu()
    out = []
    for row in mutations:
        wt, idx, mt = parse_mutation(row, offset_idx)
        assert sequence[idx] == wt, WT_MISMATCH
        out.append((lp[1 + idx, alphabet.get_idx(mt)] - lp[1 + idx, alphabet.get_idx(wt)]).item())
    return out


@torch.no_grad()
def pseudo_ppl(model, alphabet, sequence: str, mutations: Sequence[str], offset_idx: int = 0,
               max_tokens: Optional[int] = None, window: Optional[int] = None) -> List[float]:
    """compute_pppl (predict.py:118-144) for each mutation, batched across mutants and positions: every mutant is a
    substitution, so all copies share one length T. For the mutated sequence s, token position i in 1 ... len(s) - 2
    is masked and scored at alphabet.get_idx(s[i]) (the reference's indexing, kept as is); the fp32 values are summed
    as Python floats in position order. window: each position's logits merged over the windows that cover it."""
    if window is not None:
        window = windows.check_window(model, window)
    seqs = []
    for row in mutations:
        wt, idx, mt = parse_mutation(row, offset_idx)
        assert sequence[idx] == wt, WT_MISMATCH
        seqs.append(sequence[:idx] + mt + sequence[idx + 1:])
    if not seqs:
        return []
    dev = _device(model)
    _, _, toks = alphabet.get_batch_converter()([("protein1", s) for s in seqs])
    M, T = toks.shape
    P = max(len(sequence) - 2, 0)  # predict.py:138: range(1, len(sequence) - 1)
    if P == 0:
        return [0 for _ in seqs]  # sum([]) as the reference computes it
    toks = toks.to(dev)
    target = torch.tensor([alphabet.get_idx(s[i]) for s in seqs for i in range(1, P + 1)], dtype=torch.int64)
    target = target.to(dev)
    if window is not None:
        logits = _windowed_masked_logits(model, toks, window, torch.arange(M).repeat_interleave(P),
                                         torch.arange(1, P + 1).repeat(M), max_tokens)
        flat = log_softmax_rows(logits, target).cpu().tolist()
        return [sum(flat[j * P:(j + 1) * P]) for j in range(M)]
    mutant = torch.arange(M, device=dev).repeat_interleave(P)
    position = torch.arange(1, P + 1, device=dev).repeat(M)
    k = _copies_per_chunk(T, max_tokens)
    vals = []
    for s in range(0, M * P, k):
        pos = position[s:s + k]
        m = pos.numel()
        batch = toks.index_select(0, mutant[s:s + k])
        copy = torch.arange(m, device=dev)
        batch[copy, pos] = alphabet.mask_idx
        vals.append(log_softmax_rows(_head_rows(model, batch, copy * T + pos), target[s:s + k]))
    flat = torch.cat(vals).cpu().tolist()
    return [sum(flat[j * P:(j + 1) * P]) for j in range(M)]


def _windowed_masked_logits(model, toks: torch.Tensor, window: int, row: torch.Tensor, pos: torch.Tensor,
                            max_tokens: Optional[int]) -> torch.Tensor:
    """Merged logits fp32 [q, V] of queries (row[k], pos[k]): sequence row[k] of toks [M, T] (unpadded, one length)
    with token position pos[k] masked, one masked copy per window covering pos[k] (esm_b200.windows). The copies of
    all queries run in chunks of at most max_tokens tokens, as the unwindowed scorers run theirs."""
    dev = _device(model)
    M, T = toks.shape
    bos, eos = int(model.prepend_bos), int(model.append_eos)
    plan = windows.Plan(T - bos - eos, window, bos, eos)
    Tw = plan.tokens
    ext = torch.cat([toks.to(dev), torch.full((M, 1), model.padding_idx, dtype=toks.dtype, device=dev)], 1)
    wtok = ext[:, plan.gather(T, Tw).to(dev)].reshape(M * plan.K, Tw)
    tpos, twin, trow, tw = plan.terms()
    first = windows.segments(tpos, T)  # terms of token position t: [first[t], first[t + 1])
    pos, row = pos.cpu(), row.cpu()
    counts = first[pos + 1] - first[pos]
    seg = torch.zeros(pos.numel() + 1, dtype=torch.int64)
    seg[1:] = counts.cumsum(0)
    term = first[pos].repeat_interleave(counts) + torch.arange(int(seg[-1])) - seg[:-1].repeat_interleave(counts)
    copy_win = (row.repeat_interleave(counts) * plan.K + twin[term]).to(dev)
    copy_row = trow[term].to(dev)
    k = _copies_per_chunk(Tw, max_tokens)
    out = []
    for s in range(0, copy_win.numel(), k):
        r = copy_row[s:s + k]
        m = r.numel()
        batch = wtok.index_select(0, copy_win[s:s + k])
        copy = torch.arange(m, device=dev)
        batch[copy, r] = model.mask_idx
        out.append(_head_rows(model, batch, copy * Tw + r))
    if not out:
        return torch.empty((0, model.alphabet_size), dtype=torch.float32, device=dev)
    logits = torch.cat(out)
    return windows.merge_rows(logits, torch.arange(logits.shape[0]), tw[term], seg)


_INSERTION = re.compile(r"[a-z.*]")


def remove_insertions(sequence: str) -> str:
    """An a3m row without its insertions (lowercase letters and '.') and stop symbols ('*'), as predict.py:21-29
    aligns the rows."""
    return _INSERTION.sub("", sequence)


def _fasta_records(path):
    """(description, sequence) per FASTA record, as Biopython's FASTA parser gives them: the description is the whole
    header line after '>', the sequence the following lines joined, without spaces. Lines before the first header are
    skipped."""
    title, lines = None, []
    with open(path) as f:
        for line in f:
            if line.startswith(">"):
                if title is not None:
                    yield title, "".join(lines).replace(" ", "").replace("\r", "")
                title, lines = line[1:].rstrip(), []
            elif title is not None:
                lines.append(line.rstrip())
    if title is not None:
        yield title, "".join(lines).replace(" ", "").replace("\r", "")


def read_msa(filename, nseq: int) -> List[Tuple[str, str]]:
    """predict.py:32-42: the first nseq records of an a3m file as (description, sequence without insertions)."""
    return [(desc, remove_insertions(seq)) for desc, seq in itertools.islice(_fasta_records(filename), nseq)]
