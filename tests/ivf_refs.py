"""References for the inverted-file index (esm_b200.search.IVFIndex): the exact k-means mean, the probed rows of a
query, and the exact top k over them, restated without the list-scan kernel."""
import numpy as np
import torch


def exact_means(x: torch.Tensor, assign: torch.Tensor, nlist: int):
    """(sums int64 [nlist, D], means fp32 [nlist, D], counts int64 [nlist]) of fp16 rows x under assign, as
    esmb200_kmeans_means defines them: sums of x * 2^24 as exact integers, means fp32((S / count) * 2^-24)."""
    xi = (x.cpu().numpy().astype(np.float64) * 2.0 ** 24).astype(np.int64)
    a = assign.cpu().numpy()
    D = xi.shape[1]
    sums = np.zeros((nlist, D), dtype=np.int64)
    ok = (a >= 0) & (a < nlist)
    np.add.at(sums, a[ok], xi[ok])
    counts = np.bincount(a[ok], minlength=nlist).astype(np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        means = ((sums.astype(np.float64) / counts[:, None]) * 2.0 ** -24).astype(np.float32)
    means[counts == 0] = 0
    return torch.from_numpy(sums), torch.from_numpy(means), torch.from_numpy(counts)


def probed_rows(ids: torch.Tensor, offsets: torch.Tensor, lists) -> torch.Tensor:
    """The stored positions of the rows of the given lists (each list once, however often it is named), in ascending
    original index."""
    off = offsets.tolist()
    pos = [p for l in set(lists) if 0 <= l < len(off) - 1 for p in range(off[l], off[l + 1])]
    pos = torch.tensor(sorted(pos, key=lambda p: int(ids[p])), dtype=torch.int64)
    return pos


def topk_over(search, q: torch.Tensor, rows: torch.Tensor, ids: torch.Tensor, beta, alpha: float, pos: torch.Tensor,
              k: int, self_id: int = -1):
    """The exact search kernel (esmb200_knn_search) over the stored rows at pos only (ascending original index, so its
    ties are the original index's), for one prepared query row q [1, D]: (s fp32 [k], idx int64 [k]) with NaN / -1
    past the candidates."""
    if self_id >= 0:
        pos = pos[ids[pos].cpu() != self_id]
    s_out = torch.full((k,), float("nan"), dtype=torch.float32)
    i_out = torch.full((k,), -1, dtype=torch.int64)
    kk = min(k, pos.numel())
    if kk > 0:
        p = pos.to(rows.device)
        s, i = search.knn(q, rows[p].contiguous(), kk, None if beta is None else beta[p].contiguous(), alpha)
        s_out[:kk] = s[0].cpu()
        i_out[:kk] = ids[pos][i[0].cpu()]
    return s_out, i_out
