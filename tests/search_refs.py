"""float64 restatement of esmb200_knn_search (esm_b200/search.py) and the check its results are held to.

For fp16 operands A [Q, D], X [N, D], the exact score is s(i, j) = alpha (A_i . X_j) + beta_j in float64. The kernel's
fp32 score differs from it by at most
    tol(i, j) = alpha gemm_acc_bound(|A_i| . |X_j|, D, A_i . X_j) + 2^-23 |s(i, j)|
(the tensor-core accumulation, then one fma rounding). So if the kernel returns the set R for query i, every returned
j and every left-out candidate j' satisfy s(i, j) + tol(i, j) >= s(i, j') - tol(i, j'): the returned indices equal the
exact top k except inside the ambiguity band at the k-th score, where rounding may swap candidates.
"""
from __future__ import annotations

import torch

from kernel_refs import gemm_acc_bound

U32 = 2.0 ** -24


def exact(A16: torch.Tensor, X16: torch.Tensor, alpha: float = 1.0, beta=None):
    """(s, tol) float64 [Q, N] on A16's device."""
    a, x = A16.double(), X16.double().to(A16.device)
    dot = a @ x.T
    s = alpha * dot
    if beta is not None:
        s = s + beta.double().to(A16.device)[None]
    tol = alpha * gemm_acc_bound(a.abs() @ x.abs().T, A16.shape[1], dot) + 2 * U32 * s.abs()
    return s, tol


def candidates_mask(Q: int, N: int, self_offset: int, device, q0: int = 0) -> torch.Tensor:
    """bool [Q, N]: False at j == i + self_offset (rows q0 + i of the full query set)."""
    m = torch.ones((Q, N), dtype=torch.bool, device=device)
    if self_offset >= 0:
        i = torch.arange(Q, device=device)
        j = i + q0 + self_offset
        keep = j < N
        m[i[keep], j[keep]] = False
    return m


def topk_exact(s: torch.Tensor, k: int, mask: torch.Tensor):
    """The exact top k of float64 scores under (score descending, index ascending), as (scores, idx)."""
    Q, N = s.shape
    s = s.masked_fill(~mask, float("-inf"))
    # a stable sort of -s keeps ascending index among equal scores
    order = torch.sort(-s, dim=1, stable=True).indices[:, :k]
    return s.gather(1, order), order


def band_width(s: torch.Tensor, tol: torch.Tensor, k: int, mask: torch.Tensor) -> torch.Tensor:
    """Per query, the candidates whose interval [s - tol, s + tol] meets the k-th exact score's interval: the width
    of the ambiguity band (>= 1: the k-th itself)."""
    sk, ik = topk_exact(s, k, mask)
    kth, kt = sk[:, -1:], tol.gather(1, ik[:, -1:])
    near = (s + tol >= kth - kt) & (s - tol <= kth + kt) & mask
    return near.sum(1)


def check(scores: torch.Tensor, idx: torch.Tensor, s: torch.Tensor, tol: torch.Tensor, mask: torch.Tensor) -> None:
    """Assert that (scores fp32 [Q, k], idx int64 [Q, k]) are a valid answer for exact scores s [Q, N] with bounds tol
    and candidates mask: distinct candidates, each score within tol of the exact one, ordered by (score descending,
    index ascending), and the set exact up to the ambiguity band."""
    Q, k = idx.shape
    dev = s.device
    idx = idx.to(dev)
    scores = scores.to(dev)
    assert int(idx.min()) >= 0 and int(idx.max()) < s.shape[1], "index out of range"
    assert bool(mask.gather(1, idx).all()), "a left-out candidate was returned"
    srt = torch.sort(idx, dim=1).values
    assert bool((srt[:, 1:] != srt[:, :-1]).all()), "an index returned twice"
    se, te = s.gather(1, idx), tol.gather(1, idx)
    err = (scores.double() - se).abs()
    assert bool((err <= te).all()), f"score off its exact value by {float((err - te).max()):.3e} past the bound"
    if k > 1:
        a, b = scores[:, :-1], scores[:, 1:]
        ok = (a > b) | ((a == b) & (idx[:, :-1] < idx[:, 1:]))
        assert bool(ok.all()), "results not ordered by (score descending, index ascending)"
    inside = (se + te).min(1).values
    out = (s - tol).masked_fill(~mask, float("-inf")).scatter(1, idx, float("-inf")).max(1).values
    bad = inside < out
    assert not bool(bad.any()), f"{int(bad.sum())} queries miss a neighbour outside the ambiguity band"


def check_chunked(scores, idx, A16, X16, alpha=1.0, beta=None, self_offset=-1, chunk_elems=1 << 26):
    """check() over query chunks, so that [chunk, N] float64 matrices stay small."""
    Q, N = A16.shape[0], X16.shape[0]
    step = max(1, chunk_elems // N)
    for q0 in range(0, Q, step):
        q1 = min(Q, q0 + step)
        s, tol = exact(A16[q0:q1], X16, alpha, beta)
        check(scores[q0:q1], idx[q0:q1], s, tol, candidates_mask(q1 - q0, N, self_offset, s.device, q0))
