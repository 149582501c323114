"""Float64 references of the categorical Jacobian contact map (esm_b200/jacobian.py, steps 3-6 of its definition):
`contacts_f64`, the vectorised definition the GPU tests gate against; `contacts_f64_chunked`, the same map one slab of
i at a time, for a J whose float64 copies would not fit; and `contacts_brute_force`, the same map with every mean, norm
and sum written out as loops, which pins the definition itself (tests/test_jacobian_host.py)."""
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


def contacts_f64_chunked(jac: torch.Tensor, rows: int):
    """contacts_f64 for a J too large for a float64 copy: returns (C [L,L] float64, max N, max|J|) on jac's device,
    where max N is taken over every block, the diagonal included, before it is zeroed. Float64 slabs of `rows` values
    of i are formed one at a time:
      1. the marginal sums over i (S_i [20,L,20]) and over j (S_j [L,20,20]), and max|J|;
      2. per slab, the centring along i and j, X = J - S_i/L - S_j/L + S/L^2 with S = sum_j S_i, then each 20 x 20
         block (i, j) centred along a and along b and its Frobenius norm. The four centrings are commuting projections,
         so this equals centring the whole J along each axis in turn.
    APC and the symmetrisation then run on N [L,L] as in contacts_f64."""
    L = jac.shape[0]
    s_i = torch.zeros((20, L, 20), dtype=torch.float64, device=jac.device)
    s_j = torch.empty((L, 20, 20), dtype=torch.float64, device=jac.device)
    jmax = 0.0
    for i0 in range(0, L, rows):
        x = jac[i0:i0 + rows].double()
        s_i += x.sum(0)
        s_j[i0:i0 + rows] = x.sum(2)
        jmax = max(jmax, float(x.abs().max()))
    s = s_i.sum(1)
    n = torch.empty((L, L), dtype=torch.float64, device=jac.device)
    for i0 in range(0, L, rows):
        x = jac[i0:i0 + rows].double()
        x -= s_i[None] / L
        x -= s_j[i0:i0 + rows, :, None, :] / L
        x += s[None, :, None, :] / (L * L)
        x -= x.mean(1, keepdim=True)
        x -= x.mean(3, keepdim=True)
        n[i0:i0 + rows] = x.pow(2).sum((1, 3)).sqrt()
    del x
    nmax = float(n.max())
    n.fill_diagonal_(0)
    a = n - n.sum(1, keepdim=True) * n.sum(0, keepdim=True) / n.sum()
    a.fill_diagonal_(0)
    return (a + a.T) / 2, nmax, jmax


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
