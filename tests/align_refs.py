"""Restatements of the embedding alignment (include/esmb200.h at esmb200_align_similarity / esmb200_align):

  * sim_f64 / zscore_f64: the similarity and its z-score enhancement in float64 on the kernel's own fp16 rows, and
    sim_bound: the fp32 accumulation bound the kernel's S is held to;
  * dp: the dynamic programme in float32 numpy, vectorised along anti-diagonals (the cells of one anti-diagonal are
    independent), one float32 add or subtract per candidate as the kernel does it, so its bits are the kernel's;
  * traceback: the state machine over dp's direction bytes.
"""
from typing import Tuple

import numpy as np
import torch

DIAG, E_SRC, F_SRC, ZERO = 1, 2, 3, 0
E_EXT, F_EXT = 4, 8


def sim_f64(q16: torch.Tensor, t16: torch.Tensor) -> torch.Tensor:
    return q16.double() @ t16.double().T


def sim_bound(q16: torch.Tensor, t16: torch.Tensor) -> torch.Tensor:
    """|fl32(sum) - sum| for D fp16 products (exact in fp32) accumulated in fp32 in any order."""
    D = q16.shape[1]
    return D * 2.0 ** -24 * (q16.double().abs() @ t16.double().abs().T) + 1e-30


def zscore_f64(s: torch.Tensor) -> torch.Tensor:
    mr, sr = s.mean(1, keepdim=True), s.std(1, unbiased=False, keepdim=True)
    mc, sc = s.mean(0, keepdim=True), s.std(0, unbiased=False, keepdim=True)
    tr = torch.where(sr > 0, (s - mr) / torch.where(sr > 0, sr, 1), torch.zeros_like(s))
    tc = torch.where(sc > 0, (s - mc) / torch.where(sc > 0, sc, 1), torch.zeros_like(s))
    return 0.5 * (tr + tc)


def dp(S, mode: str, o: float, e: float):
    """(H, E, F, dir) of the programme, float32 [La+1, Lb+1] and uint8 direction bytes as the kernel stores them."""
    S = np.asarray(S, dtype=np.float32)
    La, Lb = S.shape
    o, e = np.float32(o), np.float32(e)
    neg = np.float32(-np.inf)
    H = np.zeros((La + 1, Lb + 1), np.float32)
    E = np.full((La + 1, Lb + 1), neg, np.float32)
    F = np.full((La + 1, Lb + 1), neg, np.float32)
    D = np.zeros((La + 1, Lb + 1), np.uint8)
    local = mode == "local"
    with np.errstate(invalid="ignore", over="ignore"):
        if not local:
            for j in range(1, Lb + 1):
                op, ex = H[0, j - 1] - o, E[0, j - 1] - e
                E[0, j] = ex if ex > op else op
                H[0, j] = E[0, j]
            for i in range(1, La + 1):
                op, ex = H[i - 1, 0] - o, F[i - 1, 0] - e
                F[i, 0] = ex if ex > op else op
                H[i, 0] = F[i, 0]
        for d in range(2, La + Lb + 1):
            i = np.arange(max(1, d - Lb), min(La, d - 1) + 1)
            j = d - i
            eo, ex = H[i, j - 1] - o, E[i, j - 1] - e
            ev = np.where(ex > eo, ex, eo)
            fo, fx = H[i - 1, j] - o, F[i - 1, j] - e
            fv = np.where(fx > fo, fx, fo)
            h = H[i - 1, j - 1] + S[i - 1, j - 1]
            src = np.full(i.shape, DIAG, np.uint8)
            m = ev > h
            src[m], h = E_SRC, np.where(m, ev, h)
            m = fv > h
            src[m], h = F_SRC, np.where(m, fv, h)
            if local:
                m = np.float32(0) > h
                src[m], h = ZERO, np.where(m, np.float32(0), h)
            D[i, j] = src | np.where(ex > eo, E_EXT, 0).astype(np.uint8) | np.where(fx > fo, F_EXT, 0).astype(np.uint8)
            H[i, j], E[i, j], F[i, j] = h, ev, fv
    return H, E, F, D


def traceback(D, i: int, j: int, local: bool) -> Tuple[str, int, int]:
    """(ops in query->target order, start i, start j) from the end cell (i, j) in state H."""
    out, state = [], "H"
    while True:
        if i == 0 or j == 0:
            if local or (i == 0 and j == 0):
                break
            out.append("T" if i == 0 else "Q")
            if i == 0:
                j -= 1
            else:
                i -= 1
            continue
        d = int(D[i, j])
        if state == "H":
            src = d & 3
            if src == ZERO:
                break
            if src == DIAG:
                out.append("M")
                i, j = i - 1, j - 1
            else:
                state = "E" if src == E_SRC else "F"
        elif state == "E":
            out.append("T")
            j -= 1
            state = "E" if d & E_EXT else "H"
        else:
            out.append("Q")
            i -= 1
            state = "F" if d & F_EXT else "H"
    return "".join(reversed(out)), i, j


def align(S, mode: str = "local", o: float = 1.0, e: float = 0.1):
    """(score float32, (q0, q1), (t0, t1), ops) of one pair."""
    H, _, _, D = dp(S, mode, o, e)
    La, Lb = H.shape[0] - 1, H.shape[1] - 1
    if mode == "local":
        k = int(np.argmax(H))  # the first maximum in row-major order: smallest i, then smallest j
        i1, j1 = divmod(k, Lb + 1)
    else:
        i1, j1 = La, Lb
    ops, i0, j0 = traceback(D, i1, j1, mode == "local")
    return H[i1, j1], (i0, i1), (j0, j1), ops


def score_of(S, ops: str, q0: int, t0: int, o: float, e: float) -> float:
    """The alignment's score recomputed from its ops in float64 (a consistency check, not the kernel's bits)."""
    S = np.asarray(S, dtype=np.float64)
    i, j, total, prev = q0, t0, 0.0, None
    for op in ops:
        if op == "M":
            total += S[i, j]
            i, j = i + 1, j + 1
        else:
            total -= e if op == prev else o
            i, j = i + (op == "Q"), j + (op == "T")
        prev = op
    return total
