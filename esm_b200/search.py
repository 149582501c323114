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

Databases larger than the GPU: IndexWriter writes a sharded index directory, and ShardedIndex memory-maps it and
streams it through the GPU with the same results (see ShardedIndex).

Faster, approximate search: IVFIndex clusters the rows around nlist k-means centroids and scans only the nprobe lists
nearest each query, exactly over those lists, with the same scores and tie rule; nprobe == nlist gives EmbeddingIndex's
results bit for bit (see IVFIndex).

One search is two kernel launches per batch of queries (esmb200_knn_search, include/esmb200.h): a wgmma GEMM whose
epilogue keeps each query's top k, and a merge of the database stripes' lists. The [Q, N] score matrix is never
stored, and a query's result does not depend on the other queries or on how the database is split.
"""
from __future__ import annotations

import bisect
import ctypes
import json
import math
import numbers
import os
import pathlib
from concurrent.futures import ThreadPoolExecutor
from typing import List, Optional, Sequence, Tuple

import numpy as np
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


def _check_k(k, candidates: int) -> int:
    if isinstance(k, bool) or not isinstance(k, int):
        raise TypeError(f"k must be an int, got {type(k).__name__}")
    hi = min(MAX_K, candidates)
    if not 1 <= k <= hi:
        raise ValueError(f"k must be in [1, {hi}] for this index, got {k}")
    return k


def _read_extract_dir(path, layer: int) -> Tuple[List[str], torch.Tensor]:
    """(labels, fp32 [n, E]) from extract_cli's <label>.pt files under path (recursive: labels may contain '/'),
    ordered by the stored label. ValueError for a file without mean_representations[layer] or mixed widths."""
    items = _scan_extract_dir(path, layer, keep_vectors=True)
    return [l for l, _ in items], torch.stack([v for _, v in items])


def _scan_extract_dir(path, layer: int, keep_vectors: bool):
    """[(label, fp32 [E] vector or file path)] of every extract_cli file under path in label order, after the checks
    _read_extract_dir makes; with keep_vectors False only the paths are kept, so memory does not grow with the
    directory."""
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
        items.append((str(obj.get("label", os.path.splitext(os.path.relpath(f, path))[0])), v if keep_vectors else f))
    items.sort(key=lambda t: t[0])
    return items


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
        return cls._from_saved(torch.load(path, map_location="cpu", weights_only=True), path, device)

    @classmethod
    def _from_saved(cls, obj, path, device) -> "EmbeddingIndex":
        if not isinstance(obj, dict) or obj.get("format") != FORMAT:
            raise ValueError(f"{path} is not a saved EmbeddingIndex")
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        _check_metric(obj["metric"])
        return cls._from_rows(obj["rows"].to(device), obj["dim"], obj["labels"], obj["metric"], obj["layer"])

    # ---- search ------------------------------------------------------------------------------------------------------
    def _check_k(self, k, candidates: int) -> int:
        return _check_k(k, candidates)

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

    # ---- range search ------------------------------------------------------------------------------------------------
    def range_search(self, queries: torch.Tensor, *, min_score: Optional[float] = None,
                     max_distance: Optional[float] = None, max_hits: Optional[int] = None
                     ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every row within a threshold of each query (fp32/fp16 [Q, E] or [E], any device): cosine rows with
        similarity >= min_score, or l2 rows at distance <= max_distance (the threshold must match the metric). Returns
        CSR on the index's device: lims int64 [Q + 1], scores fp32 [nnz] and idx int64 [nnz]; query i's hits are
        scores[lims[i]:lims[i + 1]], ordered as search() orders them (its first k are search(k)'s, bit for bit).
        max_hits keeps each query's first max_hits hits. A query with more hits than the hit buffer holds
        (RANGE_HIT_BYTES / 12) is refused."""
        check_range_args(self.metric, min_score, max_distance, max_hits)
        if isinstance(queries, torch.Tensor) and queries.dim() == 1:
            queries = queries[None]
        if isinstance(queries, torch.Tensor) and queries.dim() == 2 and queries.shape[1] != self.dim:
            raise ValueError(f"queries have width {queries.shape[1]}, the index {self.dim}")
        q = prepare_rows(queries, self.metric, "queries")
        self._check_device()
        return self._range_rows(q.to(self.device), False, min_score, max_distance, max_hits)

    def range_search_all(self, *, min_score: Optional[float] = None, max_distance: Optional[float] = None,
                         max_hits: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every row against the index with its own row left out: (lims, scores, idx) as range_search()."""
        check_range_args(self.metric, min_score, max_distance, max_hits)
        self._check_device()
        return self._range_rows(self.rows, True, min_score, max_distance, max_hits)

    def _range_rows(self, q: torch.Tensor, self_rows: bool, min_score, max_distance, max_hits):
        Q, N, l2 = q.shape[0], len(self), self.metric == "l2"
        alpha = 2.0 if l2 else 1.0
        qn = squared_norms(q) if l2 else None
        tau = range_thresholds(self.metric, qn, Q, min_score, max_distance, self.device)
        parts = []
        for b0 in range(0, Q, QUERY_BATCH):
            b1 = min(Q, b0 + QUERY_BATCH)

            def run(c0, c1, cap_rows):  # queries [b0 + c0, b0 + c1) into a hit buffer of cap_rows hits
                hits = _HitBuffer(c1 - c0, cap_rows, self.device)
                knn_range(q[b0 + c0:b0 + c1], self.rows, 0, tau[b0 + c0:b0 + c1], *hits.tensors(), self._beta,
                          alpha, b0 + c0 if self_rows else -1)
                return hits

            for hits, c0, c1 in _range_passes(run, b1 - b0, min(range_hit_cap(), (b1 - b0) * N),
                                              _threshold_text(min_score, max_distance), b0):
                parts.append(_range_part(hits, max_hits, qn[b0 + c0:b0 + c1] if l2 else None))
        return _concat_csr(parts, self.device)


# ---- range search -----------------------------------------------------------------------------------------------------
RANGE_HIT_BYTES = 1 << 30  # device bytes of one range search's hit buffer (HIT_BYTES a hit): batches are sized to it
HIT_BYTES = 12             # a uint64 key and an int32 query row


def range_hit_cap() -> int:
    """Hits one hit buffer holds."""
    return RANGE_HIT_BYTES // HIT_BYTES


def check_range_args(metric: str, min_score, max_distance, max_hits) -> None:
    """ValueError unless exactly the metric's threshold is given (cosine: min_score, l2: max_distance >= 0), it is not
    NaN, and max_hits is None or an int >= 1."""
    if (min_score is None) == (max_distance is None):
        raise ValueError("pass exactly one threshold: min_score (cosine index) or max_distance (l2 index)")
    name, v = ("min_score", min_score) if min_score is not None else ("max_distance", max_distance)
    want = "min_score" if metric == "cosine" else "max_distance"
    if name != want:
        raise ValueError(f"a {metric} index takes {want}, not {name}")
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise ValueError(f"{name} must be a real number, got {v!r}")
    if math.isnan(float(v)):
        raise ValueError(f"{name} must not be NaN")
    if name == "max_distance" and float(v) < 0:
        raise ValueError(f"max_distance must be >= 0, got {v!r}")
    if max_hits is not None and (isinstance(max_hits, bool) or not isinstance(max_hits, int) or max_hits < 1):
        raise ValueError(f"max_hits must be None or an int >= 1, got {max_hits!r}")


def _threshold_text(min_score, max_distance) -> str:
    return f"min_score {min_score!r}" if min_score is not None else f"max_distance {max_distance!r}"


def fp32_at_or_above(x: float) -> float:
    """The smallest fp32 >= x (a real number): s >= x exactly when s >= it, for every fp32 s."""
    with np.errstate(over="ignore"):
        f = np.float32(x)
        if float(f) < x:
            f = np.nextafter(f, np.float32(np.inf))
    return float(f)


def fp32_at_or_below(x: float) -> float:
    """The largest fp32 <= x: d <= x exactly when d <= it, for every fp32 d."""
    with np.errstate(over="ignore"):
        f = np.float32(x)
        if float(f) > x:
            f = np.nextafter(f, np.float32(-np.inf))
    return float(f)


_ORD_NEG_INF = -0x7F800000 - 1  # ordinal of -inf: fp32 bits b >= 0 map to b, negative ones to -(b & 0x7FFFFFFF) - 1
_ORD_POS_INF = 0x7F800000


def _f32_of_ordinal(o: torch.Tensor) -> torch.Tensor:
    bits = torch.where(o >= 0, o, (-(o + 1)) - (1 << 31))  # int32 value of 0x80000000 | m is m - 2^31
    return bits.to(torch.int32).view(torch.float32)


def l2_distance(qn: torch.Tensor, s: torch.Tensor) -> torch.Tensor:
    """The reported l2 distance of kernel scores s: sqrt(max(|q|^2 - s, 0)) in fp32, as search() computes it."""
    return (qn - s).clamp_min(0).sqrt()


def l2_thresholds(qn: torch.Tensor, max_distance: float) -> torch.Tensor:
    """tau fp32 [Q]: per query (|q|^2 fp32 [Q]), the smallest fp32 s with l2_distance(|q|^2, s) <= max_distance.
    The distance is a chain of correctly rounded monotone operations, so it does not increase with s and the hits
    are exactly the candidates with s >= tau. Found by bisection over the ordered fp32 bit patterns, with the same
    operations on qn's device: 33 halvings cover [-inf, +inf], and +inf always qualifies (distance 0)."""
    r = fp32_at_or_below(float(max_distance))
    lo = torch.full(qn.shape, _ORD_NEG_INF, dtype=torch.int64, device=qn.device)
    hi = torch.full(qn.shape, _ORD_POS_INF, dtype=torch.int64, device=qn.device)
    for _ in range(33):
        mid = torch.div(lo + hi, 2, rounding_mode="floor")
        ok = l2_distance(qn, _f32_of_ordinal(mid)) <= r
        hi = torch.where(ok, mid, hi)
        lo = torch.where(ok, lo, mid + 1)
    return _f32_of_ordinal(hi) + 0.0  # -0 as +0, as the scores are


def range_thresholds(metric: str, qn: Optional[torch.Tensor], Q: int, min_score, max_distance,
                     device) -> torch.Tensor:
    """Each query's tau fp32 [Q] on device: its hits are the candidates with kernel score s >= tau."""
    if metric == "cosine":
        return torch.full((Q,), fp32_at_or_above(float(min_score)) + 0.0, dtype=torch.float32, device=device)
    return l2_thresholds(qn.to(device), max_distance)


def knn_range(queries: torch.Tensor, base: torch.Tensor, row0: int, tau: torch.Tensor, hit_keys: torch.Tensor,
              hit_rows: torch.Tensor, counts: torch.Tensor, total: torch.Tensor, beta: Optional[torch.Tensor] = None,
              alpha: float = 1.0, self_offset: int = -1, splits: Optional[int] = None) -> None:
    """esmb200_knn_range: append the hits of chunk base fp16 [n, D] (global rows row0 ..) for queries fp16 [Q, D]
    with thresholds tau fp32 [Q] to hit_keys int64 [cap] (uint64 keys) and hit_rows int32 [cap], adding to counts
    int64 [Q] and total int64 [1] (zeros before the first chunk), which count past cap."""
    for name, t in (("queries", queries), ("base", base)):
        if t.dtype != torch.float16 or t.dim() != 2 or not t.is_cuda or t.stride(1) != 1:
            raise ValueError(f"{name} must be a CUDA fp16 tensor [n, D] with contiguous rows")
    Q, n = queries.shape[0], base.shape[0]
    dev = base.device
    if queries.device != dev or queries.shape[1] != base.shape[1]:
        raise ValueError("queries and base must be on one device with one width")
    cap = hit_keys.numel() if isinstance(hit_keys, torch.Tensor) else -1
    want = [("tau", tau, torch.float32, (Q,)), ("hit_keys", hit_keys, torch.int64, (cap,)),
            ("hit_rows", hit_rows, torch.int32, (cap,)), ("counts", counts, torch.int64, (Q,)),
            ("total", total, torch.int64, (1,))]
    if beta is not None:
        want.append(("beta", beta, torch.float32, (n,)))
    for name, t, dtype, shape in want:
        if not (isinstance(t, torch.Tensor) and t.dtype == dtype and t.is_contiguous() and tuple(t.shape) == shape
                and t.device == dev):
            raise ValueError(f"{name} must be a contiguous {dtype} tensor {list(shape)} on the base's device")
    with torch.cuda.device(dev):
        if splits is None:
            splits = choose_splits(Q, n, torch.cuda.get_device_properties(dev).multi_processor_count)
        _lib.check(_lib.load().esmb200_knn_range(
            _ptr(queries), queries.stride(0), Q, _ptr(base), base.stride(0), n, row0, base.shape[1], _ptr(beta),
            float(alpha), self_offset, _ptr(tau), splits, _ptr(hit_keys) if cap else None,
            _ptr(hit_rows) if cap else None, cap, _ptr(counts), _ptr(total), _stream()))


_SIGN = -(1 << 63)


def knn_range_finish(hit_keys: torch.Tensor, hit_rows: torch.Tensor, counts: torch.Tensor,
                     max_hits: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """esmb200_knn_range_finish on the nnz = sum(counts) appended hits (hit_keys int64 [nnz], hit_rows int32 [nnz],
    counts int64 [Q], one CUDA device, in any order): (lims int64 [Q + 1], scores fp32, idx int64), each query's hits
    by key descending (score descending, index ascending), the first max_hits of each kept. The hits are sorted here
    with two stable torch sorts (keys are uint64: flipping the sign bit makes torch's signed order theirs)."""
    if not (isinstance(counts, torch.Tensor) and counts.dtype == torch.int64 and counts.dim() == 1
            and counts.is_contiguous() and counts.is_cuda):
        raise ValueError("counts must be a contiguous CUDA int64 tensor [Q]")
    dev, Q = counts.device, counts.numel()
    nnz = hit_keys.numel() if isinstance(hit_keys, torch.Tensor) else -1
    for name, t, dtype in (("hit_keys", hit_keys, torch.int64), ("hit_rows", hit_rows, torch.int32)):
        if not (isinstance(t, torch.Tensor) and t.dtype == dtype and t.dim() == 1 and t.numel() == nnz
                and t.device == dev):
            raise ValueError(f"{name} must be a {dtype} tensor [nnz] on the counts' device")
    if max_hits is not None and (isinstance(max_hits, bool) or not isinstance(max_hits, int) or max_hits < 1):
        raise ValueError(f"max_hits must be None or an int >= 1, got {max_hits!r}")
    order = torch.sort(hit_keys ^ _SIGN, descending=True, stable=True).indices
    order = order[torch.sort(hit_rows[order], stable=True).indices]
    keys, rows = hit_keys[order].contiguous(), hit_rows[order].contiguous()
    kept = counts if max_hits is None else counts.clamp(max=max_hits)
    n_out = int(kept.sum()) if Q else 0
    lims = torch.empty(Q + 1, dtype=torch.int64, device=dev)
    scores = torch.empty(n_out, dtype=torch.float32, device=dev)
    idx = torch.empty(n_out, dtype=torch.int64, device=dev)
    lib = _lib.load()
    with torch.cuda.device(dev):
        nbytes = ctypes.c_size_t(0)
        _lib.check(lib.esmb200_knn_range_finish_scratch_bytes(Q, ctypes.byref(nbytes)))
        scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        _lib.check(lib.esmb200_knn_range_finish(_ptr(keys), _ptr(rows), nnz, _ptr(counts), Q,
                                                -1 if max_hits is None else max_hits, _ptr(scratch), nbytes.value,
                                                _ptr(lims), _ptr(scores), _ptr(idx), _stream()))
    return lims, scores, idx


class _HitBuffer:
    """A range search pass's buffers: hit keys and rows [cap], counts [Q] and the total, counters zeroed."""

    def __init__(self, Q: int, cap: int, dev: torch.device):
        self.keys = torch.empty(cap, dtype=torch.int64, device=dev)
        self.rows = torch.empty(cap, dtype=torch.int32, device=dev)
        self.counts = torch.zeros(Q, dtype=torch.int64, device=dev)
        self.total = torch.zeros(1, dtype=torch.int64, device=dev)

    def tensors(self):
        return self.keys, self.rows, self.counts, self.total


def plan_range_reruns(counts: Sequence[int], cap: int, threshold: str, q_base: int = 0) -> List[Tuple[int, int]]:
    """After a pass overflowed a hit buffer of cap hits: consecutive query groups [c0, c1) whose exact counts sum to at
    most cap, each re-run with a buffer of exactly that many. ValueError naming the threshold and the count for a query
    whose hits alone exceed cap (q_base: the first query's number in the call)."""
    groups, c0, acc = [], 0, 0
    for i, c in enumerate(counts):
        if c > cap:
            raise ValueError(f"query {q_base + i} has {c} hits at {threshold}, more than the {cap} one hit buffer holds "
                             f"(search.RANGE_HIT_BYTES): use a tighter threshold")
        if acc + c > cap:
            groups.append((c0, i))
            c0, acc = i, 0
        acc += c
    if c0 < len(counts):
        groups.append((c0, len(counts)))
    return groups


def _range_passes(run, n: int, cap: int, threshold: str, q_base: int):
    """(hits, c0, c1) covering queries [0, n): one pass run(0, n, cap) into a buffer of cap hits, whose total is read
    once; after an overflow, the groups plan_range_reruns makes from its exact counts, each re-run into a buffer of
    exactly its hits."""
    hits = run(0, n, cap)
    total = int(hits.total.item())
    if total <= cap:
        yield hits, 0, n
        return
    counts = hits.counts.tolist()
    del hits
    for c0, c1 in plan_range_reruns(counts, cap, threshold, q_base):
        want = sum(counts[c0:c1])
        hits = run(c0, c1, want)
        if int(hits.total.item()) != want:
            raise RuntimeError(f"a range search re-run found {int(hits.total.item())} hits, its first pass {want}")
        yield hits, c0, c1


def _range_part(hits: _HitBuffer, max_hits, qn: Optional[torch.Tensor]):
    """The CSR of one pass; l2 scores become distances (l2_distance of each hit's query norm)."""
    nnz = min(int(hits.total.item()), hits.keys.numel())
    lims, s, i = knn_range_finish(hits.keys[:nnz], hits.rows[:nnz], hits.counts, max_hits)
    if qn is not None:
        s = l2_distance(qn.repeat_interleave(lims.diff(), output_size=s.numel()), s)
    return lims, s, i


def _concat_csr(parts, dev):
    lims, scores, idx, off = [torch.zeros(1, dtype=torch.int64, device=dev)], [], [], 0
    for l, s, i in parts:
        lims.append(l[1:] + off)
        scores.append(s)
        idx.append(i)
        off += s.numel()
    if not parts:
        return lims[0], torch.empty(0, dtype=torch.float32, device=dev), torch.empty(0, dtype=torch.int64, device=dev)
    return torch.cat(lims), torch.cat(scores), torch.cat(idx)


def plan_range_stream(N: int, Q: int, D: int, metric: str, cap: int) -> Tuple[int, int, int]:
    """(query block, chunk rows, hit buffer) of a streamed range search within cap device bytes: the hit buffer takes
    at most a quarter of cap (and RANGE_HIT_BYTES), the query block all Q rows if they fit beside a ring of one-tile
    slots, else the largest multiple of 64 within half of cap, and the ring's chunks the rest (whole tiles, at most
    MAX_SLOT_BYTES a slot). The results, whose size is the hit count, are not part of cap. ValueError when no block of
    64 queries or no one-tile chunk fits."""
    hit_cap = min(RANGE_HIT_BYTES, cap // 4) // HIT_BYTES
    if hit_cap < 1:
        raise ValueError(f"max_device_bytes = {cap} holds no hit buffer: pass more bytes")
    per_query = D * 2 + 4 + 8 + (4 if metric == "l2" else 0)  # rows, tau, counts, |q|^2
    fixed = lambda b: b * per_query + hit_cap * HIT_BYTES + 16 * 512  # noqa: E731  (512: the allocator's rounding)
    ring_tile = RING_SLOTS * TILE * _row_bytes(D, metric)
    block = Q
    if fixed(Q) + ring_tile > cap:
        block = max(0, cap // 2 - fixed(0)) // per_query // 64 * 64
        if block < 64:
            raise ValueError(f"max_device_bytes = {cap} holds no block of 64 query rows beside the hit buffer: "
                             f"pass more bytes")
    tiles = (cap - fixed(block)) // ring_tile
    if tiles < 1:
        raise ValueError(f"max_device_bytes = {cap} leaves no room for a {TILE}-row chunk: pass more bytes")
    chunk = int(min(tiles, max(1, MAX_SLOT_BYTES // (TILE * _row_bytes(D, metric))))) * TILE
    return max(block, 1), min(chunk, -(-N // TILE) * TILE), hit_cap


# ---- sharded indexes on disk ------------------------------------------------------------------------------------------
SHARD_FORMAT = "esm_b200.search-shards/1"
MANIFEST = "manifest.json"
SHARD_ROWS = 1 << 20          # rows per shard file the writer aims for
TILE = 256                    # database rows per kernel tile: chunks are whole tiles
RING_SLOTS = 2                # pinned host slots, and as many device slots
MAX_SLOT_BYTES = 256 << 20    # the most database bytes one ring slot holds
REFILL_THREADS = 16           # host threads copying one slot's rows out of the memory maps
DEVICE_SHARE = 0.5            # default max_device_bytes: this share of the device's free memory


def _read_manifest(path) -> dict:
    f = pathlib.Path(path) / MANIFEST
    try:
        man = json.loads(f.read_text())
    except (OSError, ValueError) as e:
        raise ValueError(f"{path} is not a sharded index: {e}") from None
    if not isinstance(man, dict) or man.get("format") != SHARD_FORMAT:
        raise ValueError(f"{f} is not a {SHARD_FORMAT} manifest")
    _check_metric(man["metric"])
    return man


def _write_durable(path: pathlib.Path, data) -> None:
    """Writes bytes (or a numpy array's raw bytes) to path and fsyncs the file."""
    with open(path, "wb") as f:
        f.write(data if isinstance(data, bytes) else memoryview(np.ascontiguousarray(data)).cast("B"))
        f.flush()
        os.fsync(f.fileno())


def _fsync_dir(path: pathlib.Path) -> None:
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _write_atomic(path: pathlib.Path, text: str) -> None:
    """Replaces path with text: written and fsynced under a temporary name, the directory fsynced (so the files the
    text names are durable first), renamed, and the directory fsynced again."""
    tmp = path.with_name(f".{path.name}.tmp{os.getpid()}")
    _write_durable(tmp, text.encode())
    _fsync_dir(path.parent)
    os.replace(tmp, path)
    _fsync_dir(path.parent)


class IndexWriter:
    """Writes a sharded index directory, or appends shards to an existing one.

        with search.IndexWriter("db/", dim=1280, metric="cosine", layer=33) as w:
            w.add(vectors, labels)       # any number of times; fp32/fp16 [n, dim], labels default to the row numbers
        index = search.ShardedIndex.open("db/")

    The directory holds manifest.json (format, metric, dim, padded_dim, layer and the ordered shards with their row
    counts) and per shard `<name>.f16` (raw little-endian fp16 rows [n, padded_dim], prepare_rows's rows),
    `<name>.labels.json` and, for l2, `<name>.norms` (little-endian fp32 |x|^2, squared_norms's values). add()
    prepares a batch at most one shard's rows at a time and buffers them until a shard is full, so memory stays
    within one shard whatever the batch size (the caller's batch aside). A batch that is refused leaves the writer as
    it was before the call. Shard files are fsynced as they are written; the manifest is written last, by close(),
    fsynced under a temporary name and renamed over the old one, so a writer that stops before close(), or a power
    loss at any point, leaves the previous index intact."""

    def __init__(self, path, dim: int, metric: str = "cosine", layer: Optional[int] = None,
                 shard_rows: int = SHARD_ROWS):
        _check_metric(metric)
        if isinstance(dim, bool) or not isinstance(dim, int) or dim < 1:
            raise ValueError(f"dim must be a positive int, got {dim!r}")
        if isinstance(shard_rows, bool) or not isinstance(shard_rows, int) or shard_rows < 1:
            raise ValueError(f"shard_rows must be a positive int, got {shard_rows!r}")
        self.path = pathlib.Path(path)
        self.dim, self.metric, self.layer, self.shard_rows = dim, metric, layer, shard_rows
        self._shards = []
        if (self.path / MANIFEST).exists():
            man = _read_manifest(self.path)
            for key, want in (("metric", metric), ("dim", dim), ("layer", layer)):
                if man[key] != want:
                    raise ValueError(f"{path} holds an index of {key} {man[key]!r}: cannot append {key} {want!r}")
            self._shards = list(man["shards"])
        self.path.mkdir(parents=True, exist_ok=True)
        self._pieces: List[Tuple[torch.Tensor, List[str]]] = []  # prepared rows and labels of the open shard
        self._buffered = 0
        self._closed = False

    def __len__(self) -> int:
        """Rows in the index once closed: the existing shards' and every row added."""
        return sum(s["rows"] for s in self._shards) + self._buffered

    def add(self, vectors: torch.Tensor, labels: Optional[Sequence[str]] = None) -> None:
        if self._closed:
            raise ValueError("the writer is closed")
        if not (isinstance(vectors, torch.Tensor) and vectors.dim() == 2):
            prepare_rows(vectors, self.metric)  # raises the TypeError
        if vectors.shape[1] != self.dim:
            raise ValueError(f"vectors have width {vectors.shape[1]}, the index {self.dim}")
        n, n0 = vectors.shape[0], len(self)
        labels = [str(n0 + i) for i in range(n)] if labels is None else [str(l) for l in labels]
        if len(labels) != n:
            raise ValueError(f"{len(labels)} labels for {n} rows")
        state = (list(self._pieces), self._buffered, len(self._shards))
        try:
            r0 = 0
            while r0 < n:  # fill the open shard, one slice at a time
                r1 = min(n, r0 + self.shard_rows - self._buffered)
                self._pieces.append((prepare_rows(vectors[r0:r1], self.metric).cpu(), labels[r0:r1]))
                self._buffered += r1 - r0
                if self._buffered == self.shard_rows:
                    self._flush()
                r0 = r1
        except BaseException:
            # the shards this call wrote are left out of the manifest; a later shard of the same name replaces them
            self._pieces, self._buffered = state[0], state[1]
            del self._shards[state[2]:]
            raise

    def _flush(self) -> None:
        rows = torch.cat([r for r, _ in self._pieces])
        labels = [l for _, ls in self._pieces for l in ls]
        name = f"shard-{len(self._shards):05d}"
        _write_durable(self.path / f"{name}.f16", rows.numpy().astype("<f2", copy=False))
        if self.metric == "l2":
            _write_durable(self.path / f"{name}.norms", squared_norms(rows).numpy().astype("<f4", copy=False))
        _write_durable(self.path / f"{name}.labels.json", json.dumps(labels).encode())
        self._shards.append({"name": name, "rows": rows.shape[0]})
        self._pieces, self._buffered = [], 0

    def close(self) -> None:
        """Writes the last shard and then the manifest."""
        if self._closed:
            return
        if len(self) < 1:
            raise ValueError("an index needs at least one row")
        if self._buffered:
            self._flush()
        man = {"format": SHARD_FORMAT, "metric": self.metric, "dim": self.dim, "padded_dim": padded_dim(self.dim),
               "layer": self.layer, "shards": self._shards}
        _write_atomic(self.path / MANIFEST, json.dumps(man, indent=1))
        self._closed = True

    def __enter__(self) -> "IndexWriter":
        return self

    def __exit__(self, exc_type, exc, tb) -> None:
        if exc_type is None:
            self.close()


class _ShardLabels(Sequence):
    """The labels of a sharded index by global row, each shard's file read the first time one of its rows is named."""

    def __init__(self, path: pathlib.Path, shards, starts):
        self._path, self._shards, self._starts = path, shards, starts
        self._cache = {}

    def __len__(self) -> int:
        return self._starts[-1]

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        i = int(i)
        if not 0 <= i < len(self):
            raise IndexError(i)
        s = bisect.bisect_right(self._starts, i) - 1
        if s not in self._cache:
            self._cache[s] = json.loads((self._path / f"{self._shards[s]['name']}.labels.json").read_text())
        return self._cache[s][i - self._starts[s]]


def _batch_sizes(q_rows: int, q_out: int) -> set:
    """The query-batch sizes a streamed search launches: q_out queries in blocks of q_rows (the last block shorter),
    each block in batches of QUERY_BATCH (the last batch shorter)."""
    sizes = set()
    for block in {min(q_rows, q_out), q_out % q_rows if q_rows else 0}:
        if block > 0:
            sizes.add(min(block, QUERY_BATCH))
            if block > QUERY_BATCH and block % QUERY_BATCH:
                sizes.add(block % QUERY_BATCH)
    return sizes


def scratch_bytes(q_rows: int, q_out: int, k: int, num_sms: int) -> int:
    """Scratch for every accumulate call of a streamed search (q_rows, q_out as _batch_sizes): the largest
    esmb200_knn_scratch_bytes over its batch sizes b at the most stripes choose_splits gives b (a short chunk only
    lowers that). Splits times b is not monotone in b, so a short last batch can need more than a full one."""
    most = lambda b: choose_splits(b, MAX_SPLITS * TILE, num_sms)  # noqa: E731  (no tile cap)
    return max([most(b) * b * k * 8 for b in _batch_sizes(q_rows, q_out)] + [16])


def _fixed_device_bytes(q_rows: int, q_out: int, k: int, D: int, metric: str, num_sms: int) -> int:
    """Device bytes of a streamed search besides the ring: q_rows resident query rows (and l2 norms) with their
    running lists, q_out rows of results, and the scratch (scratch_bytes)."""
    per_tensor = 512  # the caching allocator's rounding, for each of the call's tensors
    return (q_rows * D * 2 + (q_rows * 4 if metric == "l2" else 0) + q_rows * k * 8 + q_out * k * 12
            + scratch_bytes(q_rows, q_out, k, num_sms) + 16 * per_tensor)


def _row_bytes(D: int, metric: str) -> int:
    return D * 2 + (4 if metric == "l2" else 0)


def plan_chunk_rows(q_rows: int, q_out: int, k: int, D: int, metric: str, max_device_bytes: int,
                    num_sms: int) -> int:
    """Database rows per chunk of a streamed search: whole 256-row tiles, as many as let the ring's device slots and
    the fixed buffers (_fixed_device_bytes) fit in max_device_bytes, and at most MAX_SLOT_BYTES per slot.
    ValueError when not even one tile fits."""
    fixed = _fixed_device_bytes(q_rows, q_out, k, D, metric, num_sms)
    tile_bytes = RING_SLOTS * TILE * _row_bytes(D, metric)
    tiles = (max_device_bytes - fixed) // tile_bytes
    if tiles < 1:
        raise ValueError(f"max_device_bytes = {max_device_bytes} leaves no room for a {TILE}-row chunk beside "
                         f"{fixed} bytes of queries, lists, results and scratch: pass fewer queries or more bytes")
    return int(min(tiles, max(1, MAX_SLOT_BYTES // (TILE * _row_bytes(D, metric))))) * TILE


def device_bytes(q_rows: int, q_out: int, k: int, D: int, metric: str, chunk_rows: int, num_sms: int) -> int:
    """The device bytes plan_chunk_rows budgets for a chunk of chunk_rows rows."""
    return _fixed_device_bytes(q_rows, q_out, k, D, metric, num_sms) + RING_SLOTS * chunk_rows * _row_bytes(D, metric)


def knn_accumulate(queries: torch.Tensor, base: torch.Tensor, row0: int, k: int, keys: torch.Tensor, scratch,
                   beta: Optional[torch.Tensor] = None, alpha: float = 1.0, self_offset: int = -1,
                   splits: Optional[int] = None) -> None:
    """esmb200_knn_search_accumulate: fold the chunk base fp16 [n, D] (global rows row0 ..) into the running keys
    [Q, k] (int64 storage of the uint64 keys, zeros before the first chunk). scratch: a contiguous CUDA uint8 tensor
    of at least esmb200_knn_scratch_bytes(Q, k, splits) bytes, or None to allocate one."""
    for name, t in (("queries", queries), ("base", base)):
        if t.dtype != torch.float16 or t.dim() != 2 or not t.is_cuda or t.stride(1) != 1:
            raise ValueError(f"{name} must be a CUDA fp16 tensor [n, D] with contiguous rows")
    Q, n = queries.shape[0], base.shape[0]
    dev = base.device
    if queries.device != dev or queries.shape[1] != base.shape[1]:
        raise ValueError("queries and base must be on one device with one width")
    _check_keys(keys, Q, k, dev)
    if beta is not None and (beta.dtype != torch.float32 or not beta.is_contiguous() or beta.numel() != n
                             or beta.device != dev):
        raise ValueError("beta must be a contiguous fp32 tensor [n] on the base's device")
    if scratch is not None and (scratch.dtype != torch.uint8 or not scratch.is_contiguous() or scratch.device != dev):
        raise ValueError("scratch must be a contiguous uint8 tensor on the base's device")
    lib = _lib.load()
    with torch.cuda.device(dev):
        if splits is None:
            splits = choose_splits(Q, n, torch.cuda.get_device_properties(base.device).multi_processor_count)
        nbytes = ctypes.c_size_t(0)
        _lib.check(lib.esmb200_knn_scratch_bytes(Q, k, splits, ctypes.byref(nbytes)))
        if scratch is None:
            scratch = torch.empty(max(nbytes.value, 16), dtype=torch.uint8, device=base.device)
        _lib.check(lib.esmb200_knn_search_accumulate(
            _ptr(queries), queries.stride(0), Q, _ptr(base), base.stride(0), n, row0, base.shape[1], _ptr(beta),
            float(alpha), self_offset, k, splits, _ptr(scratch), scratch.numel(), _ptr(keys), _stream()))


def _check_keys(keys: torch.Tensor, Q: int, k: int, dev: torch.device) -> None:
    if not (isinstance(keys, torch.Tensor) and keys.dtype == torch.int64 and keys.is_contiguous()
            and tuple(keys.shape) == (Q, k) and keys.device == dev):
        raise ValueError(f"keys must be a contiguous int64 tensor [{Q}, {k}] on {dev}")


def knn_decode(keys: torch.Tensor, scores: torch.Tensor, idx: torch.Tensor) -> None:
    """esmb200_knn_decode: running keys [Q, k] to scores fp32 [Q, k] and idx int64 [Q, k] (dense, on keys' device)."""
    if not (isinstance(keys, torch.Tensor) and keys.dim() == 2 and keys.is_cuda):
        raise ValueError("keys must be a CUDA tensor [Q, k]")
    Q, k = keys.shape
    _check_keys(keys, Q, k, keys.device)
    for name, t, dtype in (("scores", scores, torch.float32), ("idx", idx, torch.int64)):
        if not (t.dtype == dtype and t.is_contiguous() and tuple(t.shape) == (Q, k) and t.device == keys.device):
            raise ValueError(f"{name} must be a contiguous {dtype} tensor [{Q}, {k}] on the keys' device")
    with torch.cuda.device(keys.device):
        _lib.check(_lib.load().esmb200_knn_decode(_ptr(keys), Q, k, _ptr(scores), _ptr(idx), _stream()))


def _cuda_device(device) -> torch.device:
    if not torch.cuda.is_available():
        raise ValueError("searching a sharded index needs a CUDA device")
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"results go to a CUDA device, got {dev}")
    return torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())


class _HostRing:
    """RING_SLOTS page-locked host slots of `rows` database rows (and l2 betas): plain host memory registered with
    CUDA, the only host memory a streamed search pins (never the database)."""

    def __init__(self, rows: int, D: int, l2: bool):
        self.rows = [torch.empty((rows, D), dtype=torch.float16) for _ in range(RING_SLOTS)]
        self.beta = [torch.empty(rows, dtype=torch.float32) for _ in range(RING_SLOTS)] if l2 else None
        self._registered = []
        cudart = torch.cuda.cudart()
        for t in self.rows + (self.beta or []):
            rc = cudart.cudaHostRegister(t.data_ptr(), t.numel() * t.element_size(), 0)
            if int(rc) != 0:
                self.release()
                raise RuntimeError(f"cudaHostRegister failed ({int(rc)}) for a {t.nbytes}-byte ring slot")
            self._registered.append(t)

    def fits(self, rows: int, D: int, l2: bool) -> bool:
        return self.rows[0].shape[0] >= rows and self.rows[0].shape[1] == D and (self.beta is not None or not l2)

    def release(self) -> None:
        cudart = torch.cuda.cudart()
        for t in self._registered:
            cudart.cudaHostUnregister(t.data_ptr())
        self._registered = []


_host_rings: dict = {}


def _host_ring(rows: int, D: int, l2: bool, device: torch.device) -> _HostRing:
    """The page-locked ring of the streamed searches on (device, current CUDA stream), kept registered between calls:
    allocating and registering 2 x 268 MB costs about half a second, as much as streaming several GB. A larger or
    different ring replaces it (the calls before it have synchronised). release_host_memory() unregisters them."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    ring = _host_rings.get(key)
    if ring is None or not ring.fits(rows, D, l2):
        if ring is not None:
            ring.release()
            del _host_rings[key]
        ring = _host_rings[key] = _HostRing(rows, D, l2)
    return ring


def release_host_memory() -> None:
    """Unregisters and frees the page-locked rings ShardedIndex searches keep between calls."""
    for ring in _host_rings.values():
        ring.release()
    _host_rings.clear()


class ShardedIndex:
    """A sharded index directory (IndexWriter), memory-mapped and searched by streaming its rows through the GPU, so
    the database may be larger than the device. Same rows, labels, metric conventions and results as an EmbeddingIndex
    of the same vectors:

        index = search.ShardedIndex.open("db/")
        scores, idx = index.search(queries, k=10)      # fp32 / int64 [Q, k] on the current CUDA device
        scores, idx = index.search_all(k=10)           # every row against the index, its own row left out
        index.labels[idx[0, 0]]                        # labels are read per shard, when a hit is named

    Each call streams the database through a ring of RING_SLOTS page-locked host slots and as many device slots, one
    chunk of whole 256-row tiles per slot: host threads refill a slot from the memory maps, a copy stream moves it to
    the device, and the fused top-k kernel folds it into each query's running top-k list on the compute stream. The
    database crosses the host link once per call (once per query block for search_all when its queries do not fit
    beside the ring). max_device_bytes caps the device memory of the call and sets the chunk size; it does not change
    the results. The page-locked host slots (at most 2 x 256 MB) stay registered for the next call, since registering
    them costs about half a second; search.release_host_memory() frees them."""

    def __init__(self, path, man: dict):
        self.path = pathlib.Path(path)
        self.metric, self.dim, self.layer = man["metric"], int(man["dim"]), man["layer"]
        self.padded_dim = int(man["padded_dim"])
        if self.padded_dim != padded_dim(self.dim):
            raise ValueError(f"{path}: padded_dim {self.padded_dim} does not match dim {self.dim}")
        self.shards = list(man["shards"])
        self._starts = [0]
        for s in self.shards:
            self._starts.append(self._starts[-1] + int(s["rows"]))
        if self._starts[-1] >= 1 << 31:
            raise ValueError(f"{path} holds {self._starts[-1]} rows: a search takes fewer than 2^31")
        self._rows, self._norms = [], []
        for s in self.shards:
            n = int(s["rows"])
            self._rows.append(np.memmap(self.path / f"{s['name']}.f16", dtype="<f2", mode="r",
                                        shape=(n, self.padded_dim)))
            if self.metric == "l2":
                self._norms.append(np.memmap(self.path / f"{s['name']}.norms", dtype="<f4", mode="r", shape=(n,)))
        self.labels = _ShardLabels(self.path, self.shards, self._starts)

    @classmethod
    def open(cls, path) -> "ShardedIndex":
        return cls(path, _read_manifest(path))

    def __len__(self) -> int:
        return self._starts[-1]

    def read_rows(self, g0: int, g1: int, rows_out: np.ndarray, beta_out: Optional[np.ndarray] = None) -> None:
        """Global rows [g0, g1) into rows_out fp16 [g1 - g0, padded_dim] and, for l2, -|x|^2 into beta_out."""
        s, o = bisect.bisect_right(self._starts, g0) - 1, 0
        while g0 + o < g1:
            a = g0 + o - self._starts[s]
            b = min(g1, self._starts[s + 1]) - self._starts[s]
            np.copyto(rows_out[o:o + b - a], self._rows[s][a:b])
            if beta_out is not None:
                np.negative(self._norms[s][a:b], out=beta_out[o:o + b - a])
            o += b - a
            s += 1

    def _read_parallel(self, pool, g0: int, g1: int, rows_out: np.ndarray, beta_out: Optional[np.ndarray]) -> None:
        """read_rows split into REFILL_THREADS pieces run on the pool's threads (numpy copies release the GIL)."""
        step = -(-(g1 - g0) // REFILL_THREADS)
        jobs = [pool.submit(self.read_rows, p, min(g1, p + step), rows_out[p - g0:min(g1, p + step) - g0],
                            None if beta_out is None else beta_out[p - g0:min(g1, p + step) - g0])
                for p in range(g0, g1, step)]
        for j in jobs:
            j.result()

    # ---- search ------------------------------------------------------------------------------------------------------
    def search(self, queries: torch.Tensor, k: int = 10, device=None,
               max_device_bytes: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """The k nearest rows of each query (fp32/fp16 [Q, E] or [E], any device): (scores fp32 [Q, k], idx int64
        [Q, k]) on `device` (default: the current CUDA device), as EmbeddingIndex.search returns them."""
        _check_k(k, len(self))
        if isinstance(queries, torch.Tensor) and queries.dim() == 1:
            queries = queries[None]
        if isinstance(queries, torch.Tensor) and queries.dim() == 2 and queries.shape[1] != self.dim:
            raise ValueError(f"queries have width {queries.shape[1]}, the index {self.dim}")
        q = prepare_rows(queries, self.metric, "queries")
        dev = _cuda_device(device)
        qn = squared_norms(q) if self.metric == "l2" else None
        return self._stream(q, qn, k, dev, max_device_bytes)

    def search_all(self, k: int = 10, device=None,
                   max_device_bytes: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Every row against the index with its own row left out: (scores, idx) [N, k] as search()."""
        _check_k(k, len(self) - 1)
        dev = _cuda_device(device)
        return self._stream(None, None, k, dev, max_device_bytes)

    def _query_block(self, k: int, cap: int, num_sms: int) -> int:
        """Rows of the database held on the device as queries at once by search_all: all of them if they fit beside
        a ring of one-tile slots (the database then crosses the host link once), else the largest multiple of 64
        that fits in half the cap."""
        N, D = len(self), self.padded_dim
        if _fixed_device_bytes(N, N, k, D, self.metric, num_sms) + RING_SLOTS * TILE * _row_bytes(D, self.metric) <= cap:
            return N
        fits = lambda b: _fixed_device_bytes(b, N, k, D, self.metric, num_sms) <= cap // 2  # noqa: E731
        lo, hi = 0, N // 64
        while lo < hi:
            mid = (lo + hi + 1) // 2
            lo, hi = (mid, hi) if fits(64 * mid) else (lo, mid - 1)
        if lo == 0:
            raise ValueError(f"max_device_bytes = {cap} holds no block of 64 query rows beside the results of "
                             f"{N} queries: pass more bytes")
        return 64 * lo

    def _block_queries(self, pool, q, qn, a0: int, a1: int, dev: torch.device):
        """The query rows [a0, a1) on the device and, for l2, their |x|^2: q's, or the database's own rows (q None,
        read from the maps; |x|^2 read as -|x|^2 and negated exactly)."""
        l2 = self.metric == "l2"
        if q is not None:
            return q[a0:a1].to(dev), (qn[a0:a1].to(dev) if l2 else None)
        buf = torch.empty((a1 - a0, self.padded_dim), dtype=torch.float16)
        nbuf = torch.empty(a1 - a0, dtype=torch.float32) if l2 else None
        self._read_parallel(pool, a0, a1, buf.numpy(), nbuf.numpy() if l2 else None)
        return buf.to(dev), ((-nbuf).to(dev) if l2 else None)

    def _stream(self, q: Optional[torch.Tensor], qn: Optional[torch.Tensor], k: int, dev: torch.device,
                max_device_bytes: Optional[int]):
        N, D, l2 = len(self), self.padded_dim, self.metric == "l2"
        self_rows = q is None
        Q = N if self_rows else q.shape[0]
        alpha = 2.0 if l2 else 1.0
        with torch.cuda.device(dev):
            num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
            cap = int(DEVICE_SHARE * torch.cuda.mem_get_info(dev)[0]) if max_device_bytes is None \
                else int(max_device_bytes)
            block = self._query_block(k, cap, num_sms) if self_rows else Q
            chunk = plan_chunk_rows(block, Q, k, D, self.metric, cap, num_sms)
            chunk = min(chunk, -(-N // TILE) * TILE)
            scores = torch.empty((Q, k), dtype=torch.float32, device=dev)
            idx = torch.empty((Q, k), dtype=torch.int64, device=dev)
            if Q == 0:
                return scores, idx
            scratch = torch.empty(scratch_bytes(block, Q, k, num_sms), dtype=torch.uint8, device=dev)
            ring = _ChunkRing(self, chunk, dev)
            try:
                with ThreadPoolExecutor(REFILL_THREADS) as pool:
                    for a0 in range(0, Q, block):
                        a1 = min(Q, a0 + block)
                        qrows, qnorm = self._block_queries(pool, q, qn, a0, a1, dev)
                        keys = torch.zeros((a1 - a0, k), dtype=torch.int64, device=dev)

                        def consume(rows, beta, g0, g1):
                            for b0 in range(0, a1 - a0, QUERY_BATCH):
                                b1 = min(a1 - a0, b0 + QUERY_BATCH)
                                splits = choose_splits(b1 - b0, g1 - g0, num_sms)
                                knn_accumulate(qrows[b0:b1], rows, g0, k, keys[b0:b1], scratch, beta, alpha,
                                               a0 + b0 if self_rows else -1, splits)

                        ring.run(pool, consume)
                        knn_decode(keys, scores[a0:a1], idx[a0:a1])
                        if l2:
                            sc = scores[a0:a1]
                            torch.sub(qnorm[:, None], sc, out=sc)
                            sc.clamp_min_(0).sqrt_()
                        del keys, qrows
            finally:  # the host ring is reused by the next call: nothing may still read it
                ring.synchronize()
        return scores, idx

    # ---- range search ------------------------------------------------------------------------------------------------
    def range_search(self, queries: torch.Tensor, *, min_score: Optional[float] = None,
                     max_distance: Optional[float] = None, max_hits: Optional[int] = None, device=None,
                     max_device_bytes: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every row within the threshold of each query, as EmbeddingIndex.range_search returns them (lims, scores,
        idx on `device`, default the current CUDA device), streamed through the GPU as search() streams it."""
        check_range_args(self.metric, min_score, max_distance, max_hits)
        if isinstance(queries, torch.Tensor) and queries.dim() == 1:
            queries = queries[None]
        if isinstance(queries, torch.Tensor) and queries.dim() == 2 and queries.shape[1] != self.dim:
            raise ValueError(f"queries have width {queries.shape[1]}, the index {self.dim}")
        q = prepare_rows(queries, self.metric, "queries")
        dev = _cuda_device(device)
        qn = squared_norms(q) if self.metric == "l2" else None
        return self._range_stream(q, qn, min_score, max_distance, max_hits, dev, max_device_bytes)

    def range_search_all(self, *, min_score: Optional[float] = None, max_distance: Optional[float] = None,
                         max_hits: Optional[int] = None, device=None,
                         max_device_bytes: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """Every row against the index with its own row left out: (lims, scores, idx) as range_search()."""
        check_range_args(self.metric, min_score, max_distance, max_hits)
        dev = _cuda_device(device)
        return self._range_stream(None, None, min_score, max_distance, max_hits, dev, max_device_bytes)

    def _range_stream(self, q, qn, min_score, max_distance, max_hits, dev, max_device_bytes):
        N, D, l2 = len(self), self.padded_dim, self.metric == "l2"
        self_rows = q is None
        Q = N if self_rows else q.shape[0]
        alpha = 2.0 if l2 else 1.0
        with torch.cuda.device(dev):
            num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
            cap = int(DEVICE_SHARE * torch.cuda.mem_get_info(dev)[0]) if max_device_bytes is None \
                else int(max_device_bytes)
            block, chunk, hit_cap = plan_range_stream(N, Q, D, self.metric, cap)
            parts = []
            ring = _ChunkRing(self, chunk, dev)
            try:
                with ThreadPoolExecutor(REFILL_THREADS) as pool:
                    for a0 in range(0, Q, block):
                        a1 = min(Q, a0 + block)
                        qrows, qnorm = self._block_queries(pool, q, qn, a0, a1, dev)
                        tau = range_thresholds(self.metric, qnorm, a1 - a0, min_score, max_distance, dev)

                        def run(c0, c1, cap_rows):  # query rows [c0, c1) of the block: one pass over the database
                            hits = _HitBuffer(c1 - c0, cap_rows, dev)

                            def consume(rows, beta, g0, g1):
                                knn_range(qrows[c0:c1], rows, g0, tau[c0:c1], *hits.tensors(), beta, alpha,
                                          a0 + c0 if self_rows else -1, choose_splits(c1 - c0, g1 - g0, num_sms))

                            ring.run(pool, consume)
                            return hits

                        for hits, c0, c1 in _range_passes(run, a1 - a0, min(hit_cap, (a1 - a0) * N),
                                                          _threshold_text(min_score, max_distance), a0):
                            parts.append(_range_part(hits, max_hits, qnorm[c0:c1] if l2 else None))
                        del qrows
            finally:
                ring.synchronize()
        return _concat_csr(parts, dev)


class _ChunkRing:
    """One streamed call's ring: RING_SLOTS device slots of `chunk` rows (and l2 betas), the page-locked host ring,
    a copy stream and the events that order them. run() passes the whole database through it once."""

    def __init__(self, index: "ShardedIndex", chunk: int, dev: torch.device):
        self.index, self.l2 = index, index.metric == "l2"
        N, D = len(index), index.padded_dim
        self.rows = [torch.empty((chunk, D), dtype=torch.float16, device=dev) for _ in range(RING_SLOTS)]
        self.beta = [torch.empty(chunk, dtype=torch.float32, device=dev) for _ in range(RING_SLOTS)] if self.l2 \
            else None
        self.host = _host_ring(chunk, D, self.l2, dev)
        self.compute, self.copy = torch.cuda.current_stream(dev), torch.cuda.Stream(device=dev)
        self.copied = [torch.cuda.Event() for _ in range(RING_SLOTS)]
        self.consumed = [torch.cuda.Event() for _ in range(RING_SLOTS)]
        self.bounds = [(g, min(N, g + chunk)) for g in range(0, N, chunk)]

    def _fill(self, pool, c: int) -> None:
        """host slot c % RING_SLOTS <- chunk c, once the slot's last copy has finished"""
        s, (g0, g1) = c % RING_SLOTS, self.bounds[c]
        host = self.host
        self.copied[s].synchronize()
        self.index._read_parallel(pool, g0, g1, host.rows[s].numpy(), host.beta[s].numpy() if self.l2 else None)
        with torch.cuda.stream(self.copy):  # device slot s is free once chunk c - RING_SLOTS is done
            self.copy.wait_event(self.consumed[s])
            n = g1 - g0
            self.rows[s][:n].copy_(host.rows[s][:n], non_blocking=True)
            if self.l2:
                self.beta[s][:n].copy_(host.beta[s][:n], non_blocking=True)
            self.copied[s].record(self.copy)

    def run(self, pool, consume) -> None:
        """consume(rows fp16 [n, D], beta fp32 [n] or None, g0, g1) enqueues the work on chunk [g0, g1) on the
        compute stream; chunks come in order."""
        self._fill(pool, 0)
        for c, (g0, g1) in enumerate(self.bounds):
            s = c % RING_SLOTS
            self.compute.wait_event(self.copied[s])
            consume(self.rows[s][:g1 - g0], self.beta[s][:g1 - g0] if self.l2 else None, g0, g1)
            self.consumed[s].record(self.compute)
            if c + 1 < len(self.bounds):
                self._fill(pool, c + 1)  # the host refills the next slot while the GPU works on this one

    def synchronize(self) -> None:
        self.compute.synchronize()
        self.copy.synchronize()


# ---- inverted-file index ----------------------------------------------------------------------------------------------
IVF_FORMAT = "esm_b200.search-ivf/1"
MAX_NPROBE = 128
DEFAULT_NPROBE = 8
IVF_SCRATCH_CAP = 1 << 30   # device bytes of one esmb200_ivf_search call's scratch: query batches are sized to it
ASSIGN_BATCH = 1 << 20      # rows assigned to their lists per knn launch pair
MEAN_ROWS = 1 << 23         # rows per esmb200_kmeans_means call, its limit: no column sum of one call can overflow


def ivf_scratch_bytes(Q: int, nprobe: int, nlist: int, N: int, D: int, k: int) -> int:
    """esmb200_ivf_scratch_bytes: pure host arithmetic; ValueError (the library's message) for arguments it refuses."""
    nbytes = ctypes.c_size_t(0)
    _lib.check(_lib.load().esmb200_ivf_scratch_bytes(Q, nprobe, nlist, N, D, k, ctypes.byref(nbytes)))
    return nbytes.value


def ivf_query_batch(nprobe: int, nlist: int, N: int, D: int, k: int, cap: Optional[int] = None) -> int:
    """Queries per esmb200_ivf_search call: the most (up to QUERY_BATCH) whose scratch stays within cap (default
    IVF_SCRATCH_CAP), at least 1."""
    cap = IVF_SCRATCH_CAP if cap is None else cap
    lo, hi = 1, QUERY_BATCH
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if ivf_scratch_bytes(mid, nprobe, nlist, N, D, k) <= cap else (lo, mid - 1)
    return lo


def ivf_search(queries: torch.Tensor, rows: torch.Tensor, ids: torch.Tensor, offsets: torch.Tensor, k: int,
               beta: Optional[torch.Tensor] = None, alpha: float = 1.0, probes: Optional[torch.Tensor] = None,
               self_ids: Optional[torch.Tensor] = None, scratch: Optional[torch.Tensor] = None
               ) -> Tuple[torch.Tensor, torch.Tensor]:
    """esmb200_ivf_search on prepared operands, all on one CUDA device: queries fp16 [Q, D], rows fp16 [N, D] in list
    order, ids int64 [N], offsets int64 [nlist + 1], beta fp32 [N] or None, probes int32 [Q, nprobe] (None: every
    list), self_ids int64 [Q] or None. Returns (s fp32 [Q, k], idx int64 [Q, k]), NaN / -1 past the candidates."""
    for name, t in (("queries", queries), ("rows", rows)):
        if t.dtype != torch.float16 or t.dim() != 2 or not t.is_cuda or t.stride(1) != 1:
            raise ValueError(f"{name} must be a CUDA fp16 tensor [n, D] with contiguous rows")
    dev = rows.device
    Q, N, D = queries.shape[0], rows.shape[0], rows.shape[1]
    nlist = offsets.numel() - 1
    want = [("ids", ids, torch.int64, (N,)), ("offsets", offsets, torch.int64, (nlist + 1,))]
    if beta is not None:
        want.append(("beta", beta, torch.float32, (N,)))
    if probes is not None:
        want.append(("probes", probes, torch.int32, (Q, probes.shape[-1] if probes.dim() == 2 else -1)))
    if self_ids is not None:
        want.append(("self_ids", self_ids, torch.int64, (Q,)))
    for name, t, dtype, shape in want:
        if not (t.dtype == dtype and t.is_contiguous() and tuple(t.shape) == shape and t.device == dev):
            raise ValueError(f"{name} must be a contiguous {dtype} tensor {list(shape)} on the rows' device")
    if queries.device != dev or queries.shape[1] != D:
        raise ValueError("queries and rows must be on one device with one width")
    nprobe = nlist if probes is None else probes.shape[1]
    lib = _lib.load()
    with torch.cuda.device(dev):
        nbytes = ivf_scratch_bytes(Q, nprobe, nlist, N, D, k)
        if scratch is None or scratch.numel() < nbytes:
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        scores = torch.empty((Q, k), dtype=torch.float32, device=dev)
        idx = torch.empty((Q, k), dtype=torch.int64, device=dev)
        _lib.check(lib.esmb200_ivf_search(_ptr(queries), queries.stride(0), Q, _ptr(rows), rows.stride(0), N,
                                          _ptr(ids), _ptr(offsets), nlist, D, _ptr(beta), float(alpha), _ptr(probes),
                                          nprobe, _ptr(self_ids), k, _ptr(scratch), scratch.numel(), _ptr(scores),
                                          _ptr(idx), _stream()))
    return scores, idx


def kmeans_means(rows: torch.Tensor, assign: torch.Tensor, nlist: int
                 ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """esmb200_kmeans_means: (sums int64 [nlist, D], means fp32 [nlist, D], counts int64 [nlist]) of rows fp16 [n, D]
    under assign int64 [n], on the rows' CUDA device; means = fp32((sums / counts) * 2^-24), exactly."""
    if rows.dtype != torch.float16 or rows.dim() != 2 or not rows.is_cuda or rows.stride(1) != 1:
        raise ValueError("rows must be a CUDA fp16 tensor [n, D] with contiguous rows")
    n, D = rows.shape
    if not (assign.dtype == torch.int64 and assign.is_contiguous() and tuple(assign.shape) == (n,)
            and assign.device == rows.device):
        raise ValueError(f"assign must be a contiguous int64 tensor [{n}] on the rows' device")
    dev = rows.device
    sums = torch.empty((nlist, D), dtype=torch.int64, device=dev)
    means = torch.empty((nlist, D), dtype=torch.float32, device=dev)
    counts = torch.empty(nlist, dtype=torch.int64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().esmb200_kmeans_means(_ptr(rows), rows.stride(0), n, D, _ptr(assign), nlist,
                                                    _ptr(sums), _ptr(means), _ptr(counts), _stream()))
    return sums, means, counts


def check_sum_bound(counts: torch.Tensor, max_abs: float) -> None:
    """ValueError when a cluster's exact column sum could pass int64: count * max|x| * 2^24 >= 2^63 (cosine rows,
    |x| <= 1, never can; l2 rows up to 65504 can past 2^23 members)."""
    most = int(counts.max()) if counts.numel() else 0
    if most * int(max_abs * 2 ** 24) >= 2 ** 63:
        raise ValueError(f"a cluster of {most} rows with values up to {max_abs:g} could overflow its int64 column sums: "
                         f"train on fewer rows")


def exact_means(rows: torch.Tensor, assign: torch.Tensor, nlist: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(means fp32 [nlist, D], counts int64 [nlist]) as kmeans_means defines them, for any number of rows: more than
    MEAN_ROWS rows go through kmeans_means in slices whose int64 sums are added exactly, and the means are formed as
    the kernel forms them, fp32(((double)S / count) * 2^-24), bit for bit; check_sum_bound refuses a cluster whose sum
    could overflow."""
    n = rows.shape[0]
    if n <= MEAN_ROWS:
        _, means, counts = kmeans_means(rows, assign, nlist)
        return means, counts
    sums = counts = None
    for r0 in range(0, n, MEAN_ROWS):
        s, _, c = kmeans_means(rows[r0:r0 + MEAN_ROWS], assign[r0:r0 + MEAN_ROWS], nlist)
        sums, counts = (s, c) if sums is None else (sums + s, counts + c)
    # each slice's sums and the total are bounded by count * max|x| * 2^24, so no addition wrapped if this holds
    check_sum_bound(counts, float(rows.abs().max()))
    means = ((sums.double() / counts[:, None].double()) * 2.0 ** -24).float()
    means[counts == 0] = 0
    return means, counts


def training_sample(N: int, train_rows: int, seed: int) -> torch.Tensor:
    """The k-means training sample: the first train_rows entries of a seeded permutation of the N rows, drawn on the CPU
    so that every device trains on the same rows. Its first nlist rows are the initial centroids."""
    return torch.randperm(N, generator=torch.Generator().manual_seed(seed))[:train_rows]


def worst_served(s: torch.Tensor, x_sqnorm: Optional[torch.Tensor], metric: str) -> torch.Tensor:
    """Sample positions from worst to best served by their centroid: the lowest cosine similarity s, or the largest
    l2 distance |x|^2 - s (fp32, s = 2 x.c - |c|^2), ties to the smaller position."""
    bad = -s if metric == "cosine" else x_sqnorm - s
    return torch.sort(-bad, stable=True).indices


def fill_empty(centroids: torch.Tensor, empty: torch.Tensor, x: torch.Tensor, s: torch.Tensor,
               x_sqnorm: Optional[torch.Tensor], metric: str) -> torch.Tensor:
    """The empty-cluster rule: the empty centroids (bool [nlist]), in ascending index order, each take the next
    worst-served sample row (worst_served); the row becomes the centroid as it is. Returns the new centroid rows."""
    e = empty.nonzero().flatten()
    if e.numel() == 0:
        return centroids
    out = centroids.clone()
    out[e] = x[worst_served(s, x_sqnorm, metric)[:e.numel()]]
    return out


def _check_int(name, v, lo, hi=None):
    if isinstance(v, bool) or not isinstance(v, int) or v < lo or (hi is not None and v > hi):
        raise ValueError(f"{name} must be an int in [{lo}, {hi if hi is not None else 'inf'}], got {v!r}")
    return v


def _assign(rows: torch.Tensor, centroids: torch.Tensor, metric: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """(s fp32 [n], list int64 [n]): each row's best centroid under the search score, ties to the smaller index."""
    l2 = metric == "l2"
    beta = -squared_norms(centroids) if l2 else None
    s_out, a_out = [], []
    for r0 in range(0, rows.shape[0], ASSIGN_BATCH):
        s, a = knn(rows[r0:r0 + ASSIGN_BATCH], centroids, 1, beta, 2.0 if l2 else 1.0)
        s_out.append(s[:, 0])
        a_out.append(a[:, 0])
    return torch.cat(s_out), torch.cat(a_out)


def train_kmeans(rows: torch.Tensor, dim: int, metric: str, nlist: int, train_rows: int, iters: int,
                 seed: int) -> torch.Tensor:
    """Lloyd's k-means on the prepared rows (fp16 [N, D], CUDA): the centroid rows fp16 [nlist, D] (IVFIndex)."""
    x = rows[training_sample(rows.shape[0], train_rows, seed).to(rows.device)]
    x_sqnorm = squared_norms(x) if metric == "l2" else None
    cent = x[:nlist].clone()
    for _ in range(iters):
        s, a = _assign(x, cent, metric)
        means, counts = exact_means(x, a, nlist)
        empty = counts == 0
        if metric == "cosine":  # a mean of zero has no direction: the cluster is refilled as an empty one
            empty |= (means != 0).sum(1) == 0
        new = torch.empty_like(cent)
        keep = (~empty).nonzero().flatten()
        new[keep] = prepare_rows(means[keep][:, :dim], metric, "centroids")
        cent = fill_empty(new, empty, x, s, x_sqnorm, metric)
    return cent


class IVFIndex:
    """An inverted-file index: the rows of an EmbeddingIndex grouped into nlist lists around k-means centroids.

        index = search.IVFIndex.from_extract_dir("out/", layer=33, nlist=1024)   # or IVFIndex(vectors, nlist=...)
        index = search.IVFIndex.from_index(embedding_index, nlist=1024)
        scores, idx = index.search(queries, k=10, nprobe=8)    # idx: original row numbers, -1 for a missing hit
        scores, idx = index.search_all(k=10, nprobe=8)         # every row against the index, its own row left out

    Rows, metrics and scores are EmbeddingIndex's. A query's result is the exact top k, by (score descending, original
    index ascending), over the rows of the nprobe lists whose centroids score highest for it (the same score, ties to
    the smaller list); with fewer than k rows in them the missing slots are NaN and -1. nprobe == nlist scans every
    list and gives EmbeddingIndex's results bit for bit.

    Training (Lloyd's k-means on the GPU, deterministic for given rows and seed): the sample is training_sample(N,
    train_rows, seed) (train_rows defaults to min(N, 256 nlist)) and its first nlist rows are the initial centroids.
    Each of `iters` iterations assigns every sample row to its best centroid (esmb200_knn_search with k = 1), takes each
    centroid's exact mean (exact_means) and prepares it as a row (prepare_rows: cosine centroids are unit fp16 rows);
    a cluster left empty (or, for cosine, with a zero mean) takes the worst-served sample row instead (fill_empty).
    Every row then goes to its best centroid's list; a list holds its rows in ascending original index."""

    def __init__(self, vectors: torch.Tensor, labels: Optional[Sequence[str]] = None, metric: str = "cosine",
                 layer: Optional[int] = None, *, nlist: int, train_rows: Optional[int] = None, iters: int = 20,
                 seed: int = 0):
        _check_metric(metric)
        if isinstance(vectors, torch.Tensor) and vectors.dim() == 2 and vectors.shape[0] < 1:
            raise ValueError("an index needs at least one row")
        rows = prepare_rows(vectors, metric)
        self._build(rows, vectors.shape[1], labels, metric, layer, nlist, train_rows, iters, seed)

    def _build(self, rows, dim, labels, metric, layer, nlist, train_rows, iters, seed):
        N = rows.shape[0]
        _check_int("nlist", nlist, 1, N)
        train_rows = min(N, 256 * nlist) if train_rows is None else train_rows
        _check_int("train_rows", train_rows, nlist, N)
        _check_int("iters", iters, 0)
        _check_int("seed", seed, 0)
        labels = [str(i) for i in range(N)] if labels is None else [str(l) for l in labels]
        if len(labels) != N:
            raise ValueError(f"{len(labels)} labels for {N} rows")
        if not rows.is_cuda:
            if not torch.cuda.is_available():
                raise ValueError("training an IVFIndex needs a CUDA device")
            rows = rows.to(torch.device("cuda", torch.cuda.current_device()))
        cent = train_kmeans(rows, dim, metric, nlist, train_rows, iters, seed)
        _, a = _assign(rows, cent, metric)
        ids = torch.sort(a, stable=True).indices
        offsets = torch.zeros(nlist + 1, dtype=torch.int64, device=rows.device)
        offsets[1:] = torch.cumsum(torch.bincount(a, minlength=nlist), 0)
        params = {"nlist": nlist, "train_rows": train_rows, "iters": iters, "seed": seed}
        self._set(rows[ids], ids, offsets, cent, dim, labels, metric, layer, params)

    def _set(self, rows, ids, offsets, centroids, dim, labels, metric, layer, params):
        self.rows, self.ids, self.offsets, self.centroids = rows, ids, offsets, centroids
        self.dim, self.labels, self.metric, self.layer, self.params = int(dim), list(labels), metric, layer, dict(params)
        self.nlist = offsets.numel() - 1
        self.sqnorm = squared_norms(rows) if metric == "l2" else None
        self._beta = -self.sqnorm if metric == "l2" else None
        self._cbeta = -squared_norms(centroids) if metric == "l2" else None
        self._pos = torch.empty_like(ids)  # the stored position of each original row
        self._pos[ids] = torch.arange(ids.numel(), device=ids.device)

    @classmethod
    def _from_parts(cls, rows, ids, offsets, centroids, dim, labels, metric, layer, params) -> "IVFIndex":
        self = cls.__new__(cls)
        self._set(rows, ids, offsets, centroids, dim, labels, metric, layer, params)
        return self

    @classmethod
    def from_index(cls, index: EmbeddingIndex, *, nlist: int, train_rows: Optional[int] = None, iters: int = 20,
                   seed: int = 0) -> "IVFIndex":
        """An IVF index of an EmbeddingIndex's rows, labels, metric and layer (its rows are used as they are)."""
        self = cls.__new__(cls)
        self._build(index.rows, index.dim, index.labels, index.metric, index.layer, nlist, train_rows, iters, seed)
        return self

    @classmethod
    def from_extract_dir(cls, path, layer: int, metric: str = "cosine", *, nlist: int, train_rows: Optional[int] = None,
                         iters: int = 20, seed: int = 0, device=None) -> "IVFIndex":
        """An IVF index of the mean representations at `layer` of every extract_cli file under path (label order)."""
        _check_metric(metric)
        labels, x = _read_extract_dir(path, layer)
        return cls(x.to(device) if device is not None else x, labels, metric, layer, nlist=nlist,
                   train_rows=train_rows, iters=iters, seed=seed)

    def __len__(self) -> int:
        return self.rows.shape[0]

    @property
    def device(self) -> torch.device:
        return self.rows.device

    def to(self, device) -> "IVFIndex":
        return IVFIndex._from_parts(self.rows.to(device), self.ids.to(device), self.offsets.to(device),
                                    self.centroids.to(device), self.dim, self.labels, self.metric, self.layer,
                                    self.params)

    def save(self, path) -> None:
        torch.save({"format": IVF_FORMAT, "rows": self.rows.cpu(), "ids": self.ids.cpu(),
                    "offsets": self.offsets.cpu(), "centroids": self.centroids.cpu(), "labels": self.labels,
                    "metric": self.metric, "layer": self.layer, "dim": self.dim, "params": self.params}, path)

    @classmethod
    def _from_saved(cls, obj, path, device) -> "IVFIndex":
        if not isinstance(obj, dict) or obj.get("format") != IVF_FORMAT:
            raise ValueError(f"{path} is not a saved IVFIndex")
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        _check_metric(obj["metric"])
        return cls._from_parts(obj["rows"].to(device), obj["ids"].to(device), obj["offsets"].to(device),
                               obj["centroids"].to(device), obj["dim"], obj["labels"], obj["metric"], obj["layer"],
                               obj["params"])

    @classmethod
    def load(cls, path, device=None) -> "IVFIndex":
        """An index saved by save(), on `device` (default: the current CUDA device if there is one, else the CPU)."""
        return cls._from_saved(torch.load(path, map_location="cpu", weights_only=True), path, device)

    # ---- search ------------------------------------------------------------------------------------------------------
    def check_nprobe(self, nprobe) -> int:
        """nprobe, or the default min(DEFAULT_NPROBE, nlist) for None; ValueError outside [1, min(nlist, 128)] unless
        it is nlist."""
        if nprobe is None:
            return min(DEFAULT_NPROBE, self.nlist)
        if isinstance(nprobe, bool) or not isinstance(nprobe, int) or not (
                nprobe == self.nlist or 1 <= nprobe <= min(self.nlist, MAX_NPROBE)):
            raise ValueError(f"nprobe must be in [1, {min(self.nlist, MAX_NPROBE)}] or nlist = {self.nlist}, "
                             f"got {nprobe!r}")
        return nprobe

    def probes(self, q: torch.Tensor, nprobe: int) -> torch.Tensor:
        """The coarse step on prepared query rows: int32 [Q, nprobe], each query's top-nprobe lists by the search
        score against the centroid rows, ties to the smaller list."""
        _, lists = knn(q, self.centroids, nprobe, self._cbeta, 2.0 if self.metric == "l2" else 1.0)
        return lists.int()

    def search(self, queries: torch.Tensor, k: int = 10, nprobe: Optional[int] = None
               ) -> Tuple[torch.Tensor, torch.Tensor]:
        """The k nearest rows of each query among its nprobe lists (default min(8, nlist)), as EmbeddingIndex.search
        returns them, with original row numbers; NaN / -1 past the probed lists' rows."""
        _check_k(k, len(self))
        nprobe = self.check_nprobe(nprobe)
        if isinstance(queries, torch.Tensor) and queries.dim() == 1:
            queries = queries[None]
        if isinstance(queries, torch.Tensor) and queries.dim() == 2 and queries.shape[1] != self.dim:
            raise ValueError(f"queries have width {queries.shape[1]}, the index {self.dim}")
        q = prepare_rows(queries, self.metric, "queries")
        self._check_device()
        return self._search_rows(q.to(self.device), k, nprobe, self_rows=False)

    def search_all(self, k: int = 10, nprobe: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Every row (in original order) against the index with its own row left out: (scores, idx) [N, k]."""
        _check_k(k, len(self) - 1)
        nprobe = self.check_nprobe(nprobe)
        self._check_device()
        return self._search_rows(None, k, nprobe, self_rows=True)

    def _check_device(self) -> None:
        if not self.rows.is_cuda:
            raise ValueError("the index is on the CPU: move it to a GPU with index.to('cuda') to search")

    def _search_rows(self, q: Optional[torch.Tensor], k: int, nprobe: int, self_rows: bool):
        Q = len(self) if self_rows else q.shape[0]
        N, D, l2 = len(self), self.rows.shape[1], self.metric == "l2"
        scores = torch.empty((Q, k), dtype=torch.float32, device=self.device)
        idx = torch.empty((Q, k), dtype=torch.int64, device=self.device)
        batch = ivf_query_batch(nprobe, self.nlist, N, D, k)
        scratch = None
        for b0 in range(0, Q, batch):
            b1 = min(Q, b0 + batch)
            qb = self.rows[self._pos[b0:b1]] if self_rows else q[b0:b1]
            probes = None if nprobe == self.nlist else self.probes(qb, nprobe)
            self_ids = torch.arange(b0, b1, device=self.device) if self_rows else None
            if scratch is None:
                scratch = torch.empty(ivf_scratch_bytes(b1 - b0, nprobe, self.nlist, N, D, k), dtype=torch.uint8,
                                      device=self.device)
            s, i = ivf_search(qb, self.rows, self.ids, self.offsets, k, self._beta, 2.0 if l2 else 1.0, probes,
                              self_ids, scratch)
            if l2:
                s = (squared_norms(qb)[:, None] - s).clamp_min(0).sqrt()
            scores[b0:b1] = s
            idx[b0:b1] = i
        return scores, idx


def load_file_index(path, device=None):
    """The EmbeddingIndex or IVFIndex saved in one .pt file, by its format (read once)."""
    obj = torch.load(path, map_location="cpu", weights_only=True)
    ivf = isinstance(obj, dict) and obj.get("format") == IVF_FORMAT
    return (IVFIndex if ivf else EmbeddingIndex)._from_saved(obj, path, device)
