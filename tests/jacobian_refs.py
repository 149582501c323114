"""Float64 references of the categorical Jacobian contact map (esm_b200/jacobian.py, steps 3-6 of its definition):
`contacts_f64`, the vectorised definition the GPU tests gate against, and `contacts_brute_force`, the same map with
every mean, norm and sum written out as loops, which pins the definition itself (tests/test_jacobian_host.py)."""
from __future__ import annotations

import itertools

import torch


def contacts_f64(jac: torch.Tensor) -> torch.Tensor:
    """jac [L,20,L,20] -> C [L,L] float64 on jac's device: centre along each axis, block Frobenius norms with a zero
    diagonal, APC (esm/modules.py:32-41) with a zero diagonal, symmetrise."""
    jc = jac.double()
    for axis in range(4):
        jc = jc - jc.mean(axis, keepdim=True)
    n = jc.pow(2).sum((1, 3)).sqrt()
    n.fill_diagonal_(0)
    a = n - n.sum(1, keepdim=True) * n.sum(0, keepdim=True) / n.sum()
    a.fill_diagonal_(0)
    return (a + a.T) / 2


def contacts_brute_force(jac: torch.Tensor) -> torch.Tensor:
    """The same map element by element: Jc[i,a,j,b] is the inclusion-exclusion sum over subsets S of the four axes of
    (-1)^|S| times the mean of J over S (the product of the four centring projections), the norms, APC sums and
    symmetrisation are Python loops."""
    J = jac.double().cpu()
    L, A = J.shape[0], J.shape[1]
    dims = (L, A, L, A)
    means = {}
    for r in range(5):
        for S in itertools.combinations(range(4), r):
            means[S] = J.mean(S, keepdim=True) if S else J
    N = [[0.0] * L for _ in range(L)]
    for i in range(L):
        for j in range(L):
            if i == j:
                continue
            q = 0.0
            for a in range(A):
                for b in range(A):
                    idx = (i, a, j, b)
                    v = 0.0
                    for S, m in means.items():
                        k = tuple(0 if d in S else idx[d] for d in range(4))
                        v += (-1) ** len(S) * float(m[k])
                    q += v * v
            N[i][j] = q ** 0.5
    assert dims == tuple(J.shape)
    row = [sum(N[i][j] for j in range(L)) for i in range(L)]
    col = [sum(N[i][j] for i in range(L)) for j in range(L)]
    tot = sum(row)
    Amat = [[0.0 if i == j else N[i][j] - row[i] * col[j] / tot for j in range(L)] for i in range(L)]
    return torch.tensor([[(Amat[i][j] + Amat[j][i]) / 2 for j in range(L)] for i in range(L)], dtype=torch.float64)
