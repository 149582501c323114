"""CPU restatement of a range search's result (esmb200_knn_range + esmb200_knn_range_finish, esm_b200/search.py), on
the biased keys of search_refs (the kernel's uint64 key minus 2^63, so torch orders it)."""
from __future__ import annotations

import torch

from search_refs import biased_keys, decode


def csr_of_hits(b: torch.Tensor, rows: torch.Tensor, Q: int, max_hits=None):
    """(lims int64 [Q + 1], biased keys) of appended hits (biased keys b [nnz], query rows [nnz], any order): each
    query's keys descending, the first max_hits kept."""
    out, lims = [], [0]
    for q in range(Q):
        kq = torch.sort(b[rows == q], descending=True).values
        kq = kq if max_hits is None else kq[:max_hits]
        out.append(kq)
        lims.append(lims[-1] + kq.numel())
    return torch.tensor(lims, dtype=torch.int64), (torch.cat(out) if out else torch.empty(0, dtype=torch.int64))


def range_expected(s: torch.Tensor, mask: torch.Tensor, tau: torch.Tensor, row0: int = 0, max_hits=None):
    """(lims, scores fp32, idx int64) for designed scores s float64 [Q, N] (exact in fp32) and thresholds tau [Q]:
    the candidates with s >= tau, by key descending."""
    b = biased_keys(s, mask, row0)
    hit = mask & (s >= tau.double()[:, None])
    q, j = hit.nonzero(as_tuple=True)
    lims, keys = csr_of_hits(b[q, j], q, s.shape[0], max_hits)
    sc, ix = decode(keys)
    return lims, sc, ix
