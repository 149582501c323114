"""Exact k-nearest-neighbour search over protein embeddings, on the GPU.

extract_cli writes one `<label>.pt` per protein with its mean embedding per layer. An EmbeddingIndex holds those
vectors as one device tensor of fp16 rows and answers "which k proteins are closest to this one?" exactly:

    from esm_b200 import search
    index = search.EmbeddingIndex.from_extract_dir("out/", layer=33)       # or EmbeddingIndex(vectors, labels)
    index.save("db.pt"); index = search.EmbeddingIndex.load("db.pt")
    scores, idx = index.search(queries, k=10)     # fp32 [Q, k], int64 [Q, k] on the index's device
    scores, idx = index.search_all(k=10)          # every row against the index, its own row left out

Metrics. "cosine": rows are divided by their norm before rounding to fp16; scores are the cosine similarities,
descending. "l2": rows are rounded to fp16 as given; scores are Euclidean distances, ascending, computed as
sqrt(max(|q|^2 - s, 0)) from the kernel's s = 2 q.x - |x|^2 (|x|^2 in fp32 from the fp16 rows). Ties go to the
smaller index. Rows are zero-padded to a multiple of 64 columns, which changes no dot product.

One search is two kernel launches per batch of queries (esmb200_knn_search, include/esmb200.h): a wgmma GEMM whose
epilogue keeps each query's top k, and a merge of the database stripes' lists. The [Q, N] score matrix is never
stored, and a query's result does not depend on the other queries or on how the database is split.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from .model import _ptr, _stream

METRICS = ("cosine", "l2")
MAX_K = 128
MAX_SPLITS = 1024
FP16_MAX = 65504.0
QUERY_BATCH = 8192  # queries per launch pair: scratch is at most QUERY_BATCH * splits * k * 8 bytes
FORMAT = "esm_b200.search/1"


def _check_metric(metric: str) -> None:
    if metric not in METRICS:
        raise ValueError(f"metric must be 'cosine' or 'l2', got {metric!r}")


def padded_dim(E: int) -> int:
    """Columns of the stored fp16 rows: E rounded up to a multiple of 64."""
    return -(-E // 64) * 64


def prepare_rows(x: torch.Tensor, metric: str, what: str = "vectors") -> torch.Tensor:
    """fp16 [n, padded_dim(E)] rows for the kernel, on x's device: cosine rows divided by their norm (in float64)
    before rounding, l2 rows rounded as given; ValueError for non-finite values, a zero row under cosine or a value
    that fp16 cannot hold."""
    if not isinstance(x, torch.Tensor):
        raise TypeError(f"{what} must be a torch.Tensor, got {type(x).__name__}")
    if x.dim() != 2 or not x.dtype.is_floating_point:
        raise TypeError(f"{what} must be a 2-D floating-point tensor [n, E], got {tuple(x.shape)} {x.dtype}")
    n, E = x.shape
    if not bool(torch.isfinite(x).all()):
        raise ValueError(f"{what} hold non-finite values")
    y = x.double()
    if metric == "cosine":
        norm = y.norm(dim=1, keepdim=True)
        if bool((norm == 0).any()):
            raise ValueError(f"{what} hold a zero row, which has no cosine similarity")
        y = y / norm
    elif bool((y.abs() > FP16_MAX).any()):
        raise ValueError(f"{what} hold values beyond the fp16 range (|x| > {FP16_MAX:g})")
    rows = torch.zeros((n, padded_dim(E)), dtype=torch.float16, device=x.device)
    rows[:, :E] = y.to(torch.float16)
    return rows


def squared_norms(rows: torch.Tensor) -> torch.Tensor:
    """fp32 |x|^2 of fp16 rows, summed in float64 and rounded once."""
    return rows.double().pow(2).sum(1).float()


def choose_splits(Q: int, N: int, num_sms: int) -> int:
    """Database stripes for Q queries: enough CTAs (64-query blocks x stripes) to fill the GPU about twice, at most
    one stripe per 256-row tile."""
    blocks = -(-Q // 64)
    tiles = -(-N // 256)
    return max(1, min(MAX_SPLITS, tiles, -(-2 * num_sms // blocks)))


def knn(queries: torch.Tensor, base: torch.Tensor, k: int, beta: Optional[torch.Tensor] = None, alpha: float = 1.0,
        self_offset: int = -1, splits: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """The kernel pair on prepared operands: queries fp16 [Q, D] and base fp16 [N, D] on one CUDA device (D % 64 == 0,
    rows 16-byte aligned), beta fp32 [N] or None. Returns (s fp32 [Q, k], idx int64 [Q, k]) with s = alpha q.x + beta
    as esmb200_knn_search defines it. splits: database stripes (None: choose_splits)."""
    for name, t in (("queries", queries), ("base", base)):
        if t.dtype != torch.float16 or t.dim() != 2 or not t.is_cuda or t.stride(1) != 1:
            raise ValueError(f"{name} must be a CUDA fp16 tensor [n, D] with contiguous rows")
    if beta is not None and (beta.dtype != torch.float32 or not beta.is_contiguous() or beta.numel() != base.shape[0]
                             or beta.device != base.device):
        raise ValueError("beta must be a contiguous fp32 tensor [N] on the base's device")
    Q, N = queries.shape[0], base.shape[0]
    dev = base.device
    lib = _lib.load()
    with torch.cuda.device(dev):
        if splits is None:
            splits = choose_splits(Q, N, torch.cuda.get_device_properties(dev).multi_processor_count)
        nbytes = ctypes.c_size_t(0)
        _lib.check(lib.esmb200_knn_scratch_bytes(Q, k, splits, ctypes.byref(nbytes)))
        scratch = torch.empty(max(nbytes.value, 16), dtype=torch.uint8, device=dev)
        scores = torch.empty((Q, k), dtype=torch.float32, device=dev)
        idx = torch.empty((Q, k), dtype=torch.int64, device=dev)
        _lib.check(lib.esmb200_knn_search(_ptr(queries), queries.stride(0), Q, _ptr(base), base.stride(0), N,
                                          base.shape[1], _ptr(beta), float(alpha), self_offset, k, splits,
                                          _ptr(scratch), nbytes.value, _ptr(scores), _ptr(idx), _stream()))
    return scores, idx


def _read_extract_dir(path, layer: int) -> Tuple[List[str], torch.Tensor]:
    """(labels, fp32 [n, E]) from extract_cli's <label>.pt files under path (recursive: labels may contain '/'),
    ordered by the stored label. ValueError for a file without mean_representations[layer] or mixed widths."""
    files = []
    for root, _, names in os.walk(path):
        files += [os.path.join(root, f) for f in names if f.endswith(".pt")]
    if not files:
        raise ValueError(f"no .pt files under {path}")
    items, width = [], None
    for f in sorted(files):
        obj = torch.load(f, map_location="cpu", weights_only=True)
        mean = obj.get("mean_representations", {}) if isinstance(obj, dict) else {}
        if layer not in mean:
            raise ValueError(f"{f} has no mean_representations[{layer}] (extract_cli --include mean "
                             f"--repr_layers {layer})")
        v = mean[layer].reshape(-1).float()
        if width is None:
            width = (v.numel(), f)
        elif v.numel() != width[0]:
            raise ValueError(f"{f} has width {v.numel()}, {width[1]} has {width[0]}: one index holds one width")
        items.append((str(obj.get("label", os.path.splitext(os.path.relpath(f, path))[0])), v))
    items.sort(key=lambda t: t[0])
    return [l for l, _ in items], torch.stack([v for _, v in items])


class EmbeddingIndex:
    """fp16 rows [N, padded_dim(E)] on one device, their labels, the metric and (optionally) the layer they came from;
    l2 indexes also hold fp32 |x|^2. search() needs the index on a CUDA device."""

    def __init__(self, vectors: torch.Tensor, labels: Optional[Sequence[str]] = None, metric: str = "cosine",
                 layer: Optional[int] = None):
        _check_metric(metric)
        if isinstance(vectors, torch.Tensor) and vectors.dim() == 2 and vectors.shape[0] < 1:
            raise ValueError("an index needs at least one row")
        self._set(prepare_rows(vectors, metric), vectors.shape[1], labels, metric, layer)

    def _set(self, rows, dim, labels, metric, layer):
        N = rows.shape[0]
        labels = [str(i) for i in range(N)] if labels is None else [str(l) for l in labels]
        if len(labels) != N:
            raise ValueError(f"{len(labels)} labels for {N} rows")
        self.rows, self.dim, self.labels, self.metric, self.layer = rows, int(dim), labels, metric, layer
        self.sqnorm = squared_norms(rows) if metric == "l2" else None
        self._beta = -self.sqnorm if metric == "l2" else None

    @classmethod
    def _from_rows(cls, rows, dim, labels, metric, layer):
        self = cls.__new__(cls)
        self._set(rows, dim, labels, metric, layer)
        return self

    @classmethod
    def from_extract_dir(cls, path, layer: int, metric: str = "cosine", device=None) -> "EmbeddingIndex":
        """An index of the mean representations at `layer` of every extract_cli file under path, rows in label order."""
        _check_metric(metric)
        labels, x = _read_extract_dir(path, layer)
        return cls(x.to(device) if device is not None else x, labels, metric, layer)

    def __len__(self) -> int:
        return self.rows.shape[0]

    @property
    def device(self) -> torch.device:
        return self.rows.device

    def to(self, device) -> "EmbeddingIndex":
        return EmbeddingIndex._from_rows(self.rows.to(device), self.dim, self.labels, self.metric, self.layer)

    def save(self, path) -> None:
        torch.save({"format": FORMAT, "rows": self.rows.cpu(), "dim": self.dim, "labels": self.labels,
                    "metric": self.metric, "layer": self.layer}, path)

    @classmethod
    def load(cls, path, device=None) -> "EmbeddingIndex":
        """An index saved by save(), on `device` (default: the current CUDA device if there is one, else the CPU)."""
        obj = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(obj, dict) or obj.get("format") != FORMAT:
            raise ValueError(f"{path} is not a saved EmbeddingIndex")
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        _check_metric(obj["metric"])
        return cls._from_rows(obj["rows"].to(device), obj["dim"], obj["labels"], obj["metric"], obj["layer"])

    # ---- search ------------------------------------------------------------------------------------------------------
    def _check_k(self, k, candidates: int) -> int:
        if isinstance(k, bool) or not isinstance(k, int):
            raise TypeError(f"k must be an int, got {type(k).__name__}")
        hi = min(MAX_K, candidates)
        if not 1 <= k <= hi:
            raise ValueError(f"k must be in [1, {hi}] for this index, got {k}")
        return k

    def _check_device(self) -> None:
        if not self.rows.is_cuda:
            raise ValueError("the index is on the CPU: move it to a GPU with index.to('cuda') to search")

    def search(self, queries: torch.Tensor, k: int = 10) -> Tuple[torch.Tensor, torch.Tensor]:
        """The k nearest rows of each query (fp32/fp16 [Q, E] or [E], any device): (scores fp32 [Q, k], idx int64
        [Q, k]) on the index's device, cosine similarity descending or Euclidean distance ascending."""
        self._check_k(k, len(self))
        if isinstance(queries, torch.Tensor) and queries.dim() == 1:
            queries = queries[None]
        if isinstance(queries, torch.Tensor) and queries.dim() == 2 and queries.shape[1] != self.dim:
            raise ValueError(f"queries have width {queries.shape[1]}, the index {self.dim}")
        q = prepare_rows(queries, self.metric, "queries")
        self._check_device()
        return self._search_rows(q.to(self.device), k, self_rows=False)

    def search_all(self, k: int = 10) -> Tuple[torch.Tensor, torch.Tensor]:
        """Every row against the index with its own row left out: (scores, idx) [N, k] as search()."""
        self._check_k(k, len(self) - 1)
        self._check_device()
        return self._search_rows(self.rows, k, self_rows=True)

    def _search_rows(self, q: torch.Tensor, k: int, self_rows: bool):
        Q = q.shape[0]
        scores = torch.empty((Q, k), dtype=torch.float32, device=self.device)
        idx = torch.empty((Q, k), dtype=torch.int64, device=self.device)
        alpha = 2.0 if self.metric == "l2" else 1.0
        for b0 in range(0, Q, QUERY_BATCH):
            b1 = min(Q, b0 + QUERY_BATCH)
            s, i = knn(q[b0:b1], self.rows, k, self._beta, alpha, b0 if self_rows else -1)
            if self.metric == "l2":
                s = (squared_norms(q[b0:b1])[:, None] - s).clamp_min(0).sqrt()
            scores[b0:b1] = s
            idx[b0:b1] = i
        return scores, idx
