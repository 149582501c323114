"""Overlapping windows for proteins longer than a model's window: the one module that knows the rule.

ESM-1b / ESM-1v learn positions for at most 1024 tokens and ESM-2 was trained on crops of 1024 tokens, so a longer
protein runs as overlapping crops, each tokenised as a protein of its own, whose outputs are stitched back together.
With n residues (tokens other than <cls> / <eos>) and W residues per window:

  * n <= W: one window, the whole protein;
  * otherwise K = ceil((n - W) / (W // 2)) + 1 windows; window k covers residues [s_k, s_k + W) with
    s_k = k * (n - W) // (K - 1): every window is full, the last one ends at n, consecutive starts are at most W // 2
    apart;
  * a window's tokens are <cls> + its residues + <eos> (<eos> when the alphabet appends one), its positions restart at
    1, as when the crop is fed to the model alone;
  * residue p at offset o = p - s_k of window k has weight min(o + 1, W - o), normalised over the windows that cover
    p (a taper favouring the window where p sits most centrally); <cls> comes from window 0, <eos> from the last one;
  * every output row is the normalised-weight sum of its rows in the covering windows, in window order, in fp32
    (esmb200_window_merge). A row with one window is copied, so with n <= W every output is bit-identical to the
    unwindowed path. Logits are merged; log-probabilities are log_softmax of the merged logits.
"""
from __future__ import annotations

from typing import List, Tuple

import torch

from . import _lib
from .model import _ptr, _stream


def check_window(model, window) -> int:
    """The window as an int, or ValueError before anything runs: W >= 2, and W + 2 tokens must fit the learned
    position table of ESM-1b / ESM-1v."""
    if isinstance(window, bool) or int(window) != window:
        raise TypeError(f"window must be an integer, got {window!r}")
    W = int(window)
    if W < 2:
        raise ValueError(f"window must be at least 2 residues, got {W}")
    table = getattr(model, "embed_positions", None)
    if table is not None and W + 2 > table.max_positions:
        raise ValueError(f"window {W} + <cls> + <eos> exceeds the model's {table.max_positions} learned positions")
    return W


def starts(n: int, W: int) -> List[int]:
    """First residue of each window of a protein of n residues."""
    if n <= W:
        return [0]
    K = -(-(n - W) // (W // 2)) + 1
    return [k * (n - W) // (K - 1) for k in range(K)]


class Plan:
    """The windows of one protein of n residues: starts, their token rows, and the merge terms of each token."""

    def __init__(self, n: int, W: int, bos: int, eos: int):
        self.n, self.W, self.bos, self.eos = n, W, bos, eos
        self.starts = starts(n, W)
        self.K = len(self.starts)
        self.width = min(n, W)  # residues per window

    @property
    def tokens(self) -> int:
        """Tokens of one window."""
        return self.bos + self.width + self.eos

    def gather(self, T: int, Tw: int) -> torch.Tensor:
        """int64 [K, Tw]: window k's token j is row[gather[k, j]] of the protein's token row extended by one <pad> at
        index T (<cls> is row[0], the residues row[bos + s_k : bos + s_k + width], <eos> row[bos + n])."""
        assert Tw >= self.tokens
        g = torch.full((self.K, Tw), T, dtype=torch.int64)
        g[:, :self.bos] = torch.arange(self.bos)
        for k, s in enumerate(self.starts):
            g[k, self.bos:self.bos + self.width] = torch.arange(self.bos + s, self.bos + s + self.width)
        if self.eos:
            g[:, self.bos + self.width] = self.bos + self.n
        return g

    def residue_terms(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """(residue, window, offset, weight) of every window covering every residue, residue-major and in window order;
        weights fp32, normalised per residue (exactly 1.0 for a residue with one window)."""
        S = torch.tensor(self.starts, dtype=torch.int64)
        off = torch.arange(self.n)[:, None] - S[None, :]
        cov = (off >= 0) & (off < self.width)
        taper = torch.where(cov, torch.minimum(off + 1, self.W - off), 0).double()
        norm = taper / taper.sum(1, keepdim=True)
        res, win = cov.nonzero(as_tuple=True)
        return res, win, off[res, win], norm[res, win].float()

    def terms(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
        """(token position, window, token row in the window, weight) for every output token, ordered by position."""
        res, win, off, w = self.residue_terms()
        one = lambda v: torch.tensor([v], dtype=torch.int64)
        pos, wins, rows, ws = [res + self.bos], [win], [off + self.bos], [w]
        if self.bos:
            pos.insert(0, one(0)), wins.insert(0, one(0)), rows.insert(0, one(0)), ws.insert(0, torch.ones(1))
        if self.eos:
            pos.append(one(self.bos + self.n)), wins.append(one(self.K - 1)), rows.append(one(self.bos + self.width))
            ws.append(torch.ones(1))
        return torch.cat(pos), torch.cat(wins), torch.cat(rows), torch.cat(ws)


def segments(out_rows: torch.Tensor, rows: int) -> torch.Tensor:
    """int64 [rows + 1] segment offsets of terms sorted by their output row."""
    seg = torch.zeros(rows + 1, dtype=torch.int64)
    seg[1:] = torch.bincount(out_rows, minlength=rows).cumsum(0)
    return seg


def merge_rows(src: torch.Tensor, idx: torch.Tensor, w: torch.Tensor, seg: torch.Tensor) -> torch.Tensor:
    """esmb200_window_merge: out[r] = sum over j in [seg[r], seg[r+1]) of w[j] * src[idx[j]] in j order, fp32 [rows, C].
    src fp32 CUDA [R, C] with unit column stride; idx, w, seg host or device tensors."""
    if not src.is_cuda:
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
    if src.dtype != torch.float32 or src.dim() != 2 or src.stride(1) != 1:
        raise ValueError("src must be fp32 [R, C] with unit column stride")
    R, C = src.shape
    rows = seg.numel() - 1
    dev = src.device
    if idx.numel() and not (0 <= int(idx.min()) and int(idx.max()) < R):
        raise ValueError(f"merge indices must lie in [0, {R})")
    idx = idx.to(dev, torch.int64).contiguous()
    w = w.to(dev, torch.float32).contiguous()
    seg = seg.to(dev, torch.int64).contiguous()
    out = torch.empty((rows, C), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().esmb200_window_merge(_ptr(src), src.stride(0) if R else C, _ptr(idx), _ptr(w),
                                                     _ptr(seg), rows, C, _ptr(out), C, _stream()))
    return out
