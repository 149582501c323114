"""Pairwise alignment of proteins by their per-residue embeddings, on the GPU (the EBA / pLM-BLAST family of methods).

search_cli finds a query's nearest proteins by mean embedding, but a hit has no residue correspondence. This module
builds one: a residue-by-residue similarity matrix from the two proteins' per-residue embeddings (extract_cli
--include per_tok) and an affine-gap dynamic programme over it.

    from esm_b200 import align
    res = align.align_pairs([qa, qb], [ta, tb], mode="local")     # lists of [L, E] tensors, any float dtype / device
    res[0].score, res[0].query_span, res[0].target_span, res[0].ops, res[0].pairs(), res[0].cigar()
    text = align.to_a3m(query_seq, [(label, target_seq, res[0]), ...])   # query-anchored a3m for the MSA Transformer

Definition (include/esmb200.h at esmb200_align). Rows are normalised and rounded to fp16 as the cosine index does it
(search.prepare_rows); S[i, j] = q_i . t_j with fp32 accumulation; with zscore (default) S' = the mean of S's row and
column z-scores, else S' = S. The programme runs on S' in fp32 with gap open o and extend e, ties broken in a fixed
evaluation order, so a pair's result depends only on the pair: not on the other pairs in a call, on how they are
chunked (max_cells) or on the device.

The default penalties are untuned: no labelled benchmark was available to tune them against. Pass your own for
anything that matters.
"""
from __future__ import annotations

import ctypes
import math
import re
from dataclasses import dataclass
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import torch

from . import _lib
from .model import _ptr, _stream
from .search import prepare_rows

MODES = {"local": _lib.ALIGN_LOCAL, "global": _lib.ALIGN_GLOBAL}
GAP_OPEN = 1.0     # untuned
GAP_EXTEND = 0.1   # untuned
MAX_CELLS = 1 << 28  # cells per chunk: 1 GiB of S' and about 0.25 GiB of direction bytes


@dataclass(frozen=True)
class Alignment:
    """One pair's result: score (fp32 value as a float), query_span and target_span (0-based, end exclusive) and
    ops, the op string in query->target order: 'M' a query residue aligned to a target residue, 'Q' a query residue
    against a gap, 'T' a target residue against a gap."""
    score: float
    query_span: Tuple[int, int]
    target_span: Tuple[int, int]
    ops: str

    def pairs(self) -> List[Tuple[int, int]]:
        """(query index, target index) of every aligned residue pair, 0-based, in order."""
        i, j = self.query_span[0], self.target_span[0]
        out = []
        for op in self.ops:
            if op == "M":
                out.append((i, j))
            i += op in "MQ"
            j += op in "MT"
        return out

    def cigar(self) -> str:
        """The ops run-length encoded, e.g. '12M2T30M1Q4M' ('' for an empty alignment)."""
        return "".join(f"{len(m.group(0))}{m.group(0)[0]}" for m in re.finditer(r"M+|Q+|T+", self.ops))


def _check_penalties(mode: str, gap_open, gap_extend) -> None:
    if mode not in MODES:
        raise ValueError(f"mode must be 'local' or 'global', got {mode!r}")
    for name, v in (("gap_open", gap_open), ("gap_extend", gap_extend)):
        if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
            raise ValueError(f"{name} must be a finite number >= 0, got {v!r}")


def _check_max_cells(max_cells) -> int:
    if max_cells is None:
        return MAX_CELLS
    if isinstance(max_cells, bool) or not isinstance(max_cells, int) or max_cells < 1:
        raise ValueError(f"max_cells must be a positive int, got {max_cells!r}")
    return max_cells


def _chunks(cells: Sequence[int], max_cells: int) -> List[Tuple[int, int]]:
    """Consecutive pair ranges [a, b) of at most max_cells cells each; a pair larger than max_cells is refused."""
    out, a, acc = [], 0, 0
    for p, c in enumerate(cells):
        if c > max_cells:
            raise ValueError(f"pair {p} has {c} cells, more than max_cells = {max_cells}")
        if acc + c > max_cells:
            out.append((a, p))
            a, acc = p, 0
        acc += c
    if a < len(cells):
        out.append((a, len(cells)))
    return out


def _device(device) -> torch.device:
    if device is None:
        if not torch.cuda.is_available():
            raise _lib.Esmb200Error("esm_b200.align runs on CUDA (sm_90a) only and has no CPU path")
        return torch.device("cuda", torch.cuda.current_device())
    device = torch.device(device)
    if device.type != "cuda":
        raise ValueError(f"alignment runs on a CUDA device, got {device}")
    return device


def _offsets(lengths: Sequence[int], dev) -> torch.Tensor:
    off = [0]
    for n in lengths:
        off.append(off[-1] + n)
    return torch.tensor(off, dtype=torch.int64, device=dev)


def _scratch(P: int, n_q: int, n_t: int, n_cells: int, dev) -> torch.Tensor:
    nbytes = _lib.load().esmb200_align_scratch_bytes(P, n_q, n_t, n_cells)
    return torch.empty(max(nbytes, 256), dtype=torch.uint8, device=dev)


def _run_dp(s: torch.Tensor, La: Sequence[int], Lb: Sequence[int], offs, scratch, mode: str, gap_open: float,
            gap_extend: float) -> List[Alignment]:
    """esmb200_align on one chunk whose S' (flat fp32) and offsets are on the device."""
    q_off, t_off, s_off = offs
    P, n_q, n_t, n_cells = len(La), sum(La), sum(Lb), s.numel()
    dev = s.device
    scores = torch.empty(P, dtype=torch.float32, device=dev)
    spans = torch.empty((P, 4), dtype=torch.int32, device=dev)
    ops = torch.empty(n_q + n_t, dtype=torch.uint8, device=dev)
    n_ops = torch.empty(P, dtype=torch.int32, device=dev)
    lib = _lib.load()
    _lib.check(lib.esmb200_align(_ptr(s), _ptr(q_off), _ptr(t_off), _ptr(s_off), P, n_q, n_t, n_cells, MODES[mode],
                                 float(gap_open), float(gap_extend), _ptr(scratch), scratch.numel(), _ptr(scores),
                                 _ptr(spans), _ptr(ops), _ptr(n_ops), _stream()))
    scores, spans, n_ops, ops = scores.tolist(), spans.tolist(), n_ops.tolist(), ops.cpu().numpy().tobytes()
    out, base = [], 0
    for p in range(P):
        q0, q1, t0, t1 = spans[p]
        out.append(Alignment(scores[p], (q0, q1), (t0, t1), ops[base:base + n_ops[p]].decode("ascii")))
        base += La[p] + Lb[p]
    return out


def _matrix_checks(mats) -> None:
    for k, m in enumerate(mats):
        if not isinstance(m, torch.Tensor) or m.dim() != 2 or not m.dtype.is_floating_point:
            raise TypeError(f"similarity {k} must be a 2-D floating-point tensor [La, Lb]")
        if m.shape[0] < 1 or m.shape[1] < 1:
            raise ValueError(f"similarity {k} is {tuple(m.shape)}: La and Lb must be at least 1")
        if not bool(torch.isfinite(m).all()):
            raise ValueError(f"similarity {k} holds non-finite values")


def align_matrices(similarities: Sequence[torch.Tensor], mode: str = "local", gap_open: float = GAP_OPEN,
                   gap_extend: float = GAP_EXTEND, max_cells: Optional[int] = None, device=None) -> List[Alignment]:
    """The dynamic programme alone on caller-chosen S' matrices ([La, Lb], taken as float32, any device)."""
    _check_penalties(mode, gap_open, gap_extend)
    max_cells = _check_max_cells(max_cells)
    _matrix_checks(similarities)
    dev = _device(device)
    La = [int(m.shape[0]) for m in similarities]
    Lb = [int(m.shape[1]) for m in similarities]
    out: List[Alignment] = []
    with torch.cuda.device(dev):
        for a, b in _chunks([x * y for x, y in zip(La, Lb)], max_cells):
            s = torch.cat([m.to(device=dev, dtype=torch.float32).reshape(-1) for m in similarities[a:b]])
            offs = (_offsets(La[a:b], dev), _offsets(Lb[a:b], dev),
                    _offsets([x * y for x, y in zip(La[a:b], Lb[a:b])], dev))
            scratch = _scratch(b - a, sum(La[a:b]), sum(Lb[a:b]), s.numel(), dev)
            out += _run_dp(s, La[a:b], Lb[a:b], offs, scratch, mode, gap_open, gap_extend)
    return out


def align_pairs(queries: Sequence[torch.Tensor], targets: Sequence[torch.Tensor], mode: str = "local",
                gap_open: float = GAP_OPEN, gap_extend: float = GAP_EXTEND, zscore: bool = True,
                max_cells: Optional[int] = None, return_similarity: bool = False, device=None):
    """Align queries[p] to targets[p] for every p: [L, E] per-residue embeddings (any float dtype and device; a pair
    shares E). Returns a list of Alignment, and with return_similarity also the list of S' (fp32 [La, Lb] on the
    device). The same tensor given several times is normalised once."""
    _check_penalties(mode, gap_open, gap_extend)
    max_cells = _check_max_cells(max_cells)
    if not isinstance(zscore, bool):
        raise TypeError("zscore must be a bool")
    queries, targets = list(queries), list(targets)
    if len(queries) != len(targets):
        raise ValueError(f"{len(queries)} queries for {len(targets)} targets")
    for what, xs in (("query", queries), ("target", targets)):
        for k, x in enumerate(xs):
            if not isinstance(x, torch.Tensor) or x.dim() != 2 or not x.dtype.is_floating_point:
                raise TypeError(f"{what} {k} must be a 2-D floating-point tensor [L, E]")
            if x.shape[0] < 1:
                raise ValueError(f"{what} {k} has no residues")
    for k, (q, t) in enumerate(zip(queries, targets)):
        if q.shape[1] != t.shape[1]:
            raise ValueError(f"pair {k}: the query has width {q.shape[1]}, the target {t.shape[1]}")
    dev = _device(device)
    rows: Dict[int, torch.Tensor] = {}

    def prepared(x: torch.Tensor, what: str) -> torch.Tensor:
        if id(x) not in rows:  # per protein, so its rows never depend on what else is in the call
            rows[id(x)] = prepare_rows(x.to(dev), "cosine", what)
        return rows[id(x)]

    for q, t in zip(queries, targets):
        prepared(q, "query embeddings")
        prepared(t, "target embeddings")
    La = [int(q.shape[0]) for q in queries]
    Lb = [int(t.shape[0]) for t in targets]
    lib = _lib.load()
    results: List[Alignment] = []
    sims: List[torch.Tensor] = []
    with torch.cuda.device(dev):
        for a, b in _chunks([x * y for x, y in zip(La, Lb)], max_cells):
            qa = torch.cat([rows[id(q)] for q in queries[a:b]])
            ta = torch.cat([rows[id(t)] for t in targets[a:b]])
            la, lb = La[a:b], Lb[a:b]
            cells = [x * y for x, y in zip(la, lb)]
            offs = (_offsets(la, dev), _offsets(lb, dev), _offsets(cells, dev))
            P, n_q, n_t, n_cells = b - a, sum(la), sum(lb), sum(cells)
            s = torch.empty(n_cells, dtype=torch.float32, device=dev)
            scratch = _scratch(P, n_q, n_t, n_cells, dev)
            _lib.check(lib.esmb200_align_similarity(_ptr(qa), _ptr(ta), qa.shape[1], _ptr(offs[0]), _ptr(offs[1]),
                                                    _ptr(offs[2]), P, n_q, n_t, n_cells, int(zscore), _ptr(s),
                                                    _ptr(scratch), scratch.numel(), _stream()))
            results += _run_dp(s, la, lb, offs, scratch, mode, gap_open, gap_extend)
            if return_similarity:
                c0 = 0
                for x, y in zip(la, lb):
                    sims.append(s[c0:c0 + x * y].view(x, y))
                    c0 += x * y
    return (results, sims) if return_similarity else results


def a3m_row(query_len: int, target_seq: str, aln: Alignment) -> str:
    """The target's a3m row against a query of query_len residues: one upper-case target residue or '-' per query
    column, target insertions in lower case, query columns outside the alignment '-'."""
    q0, q1 = aln.query_span
    t0, t1 = aln.target_span
    if q1 > query_len or t1 > len(target_seq):
        raise ValueError(f"alignment spans query {aln.query_span} / target {aln.target_span} beyond the sequences "
                         f"({query_len} / {len(target_seq)} residues)")
    cols = ["-"] * query_len
    inserts = [""] * (query_len + 1)  # inserts[k]: target residues between query columns k - 1 and k
    i, j = q0, t0
    for op in aln.ops:
        if op == "M":
            cols[i] = target_seq[j].upper()
            i, j = i + 1, j + 1
        elif op == "Q":
            i += 1
        else:
            inserts[i] += target_seq[j].lower()
            j += 1
    return "".join(inserts[k] + cols[k] for k in range(query_len)) + inserts[query_len]


def to_a3m(query_seq: str, hits: Iterable[Tuple[str, str, Alignment]], query_label: str = "query") -> str:
    """A query-anchored a3m: the query first, then one row per (label, target sequence, alignment) in the given
    order. variants.read_msa reads every row back at the query's length (lower-case insertions removed)."""
    lines = [f">{query_label}", query_seq]
    for label, seq, aln in hits:
        lines += [f">{label}", a3m_row(len(query_seq), seq, aln)]
    return "\n".join(lines) + "\n"
