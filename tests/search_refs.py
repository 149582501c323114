"""float64 restatement of esmb200_knn_search (esm_b200/search.py) and the check its results are held to.

For fp16 operands A [Q, D], X [N, D], the exact score is s(i, j) = alpha (A_i . X_j) + beta_j in float64. The kernel's
fp32 score differs from it by at most
    tol(i, j) = alpha gemm_acc_bound(|A_i| . |X_j|, D, A_i . X_j) + 2^-23 |s(i, j)|
(the tensor-core accumulation, then one fma rounding). So if the kernel returns the set R for query i, every returned
j and every left-out candidate j' satisfy s(i, j) + tol(i, j) >= s(i, j') - tol(i, j'): the returned indices equal the
exact top k except inside the ambiguity band at the k-th score, where rounding may swap candidates.
"""
from __future__ import annotations

import numpy as np
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


# ---- designed exact scores ---------------------------------------------------------------------------------------
# A designed score matrix has no rounding anywhere: query q is one-hot (or two-hot) and column j of the database carries
# the score, so every wgmma sum has one or two nonzero exact products, and alpha, beta are chosen so that
# fmaf(alpha, acc, beta) is exact too. The kernel must then return exactly the top k under (score descending, index
# ascending), bit for bit. Candidates are compared through the kernel's own ranking key, stored biased as int64
# (key - 2^63) so that torch and numpy order it: I64_MIN is key 0, an empty slot.
I64_MIN = -(1 << 63)
QCAP, CHUNK, TILE, BLOCK_M = 64, 32, 256, 64  # the kernel's queue, chunk, tile and query block (csrc/knn.cuh)
FLT_MAX = 3.4028234663852886e38


def biased_keys(s: torch.Tensor, mask: torch.Tensor, row0: int = 0) -> torch.Tensor:
    """int64 [Q, N]: the kernel's key of each candidate (float64 scores that fp32 holds exactly, global index row0 + j)
    minus 2^63; I64_MIN where mask is False."""
    s32 = s.float()
    assert torch.equal(s32.double()[mask], s[mask]), "a designed score is not exact in fp32"
    u = (s32 + 0.0).view(torch.int32).long() & 0xFFFFFFFF  # + 0: -0 becomes +0, as in the kernel
    o = torch.where(u >= 1 << 31, (~u) & 0xFFFFFFFF, u | (1 << 31))
    j = torch.arange(s.shape[1], device=s.device, dtype=torch.int64) + row0
    return ((o - (1 << 31)) * (1 << 32) + (0xFFFFFFFF - j)).masked_fill(~mask, I64_MIN)


def raw_keys(b: torch.Tensor) -> torch.Tensor:
    """Biased keys to the int64 storage of the uint64 keys (the running list of esmb200_knn_search_accumulate)."""
    return b ^ I64_MIN


def decode(b: torch.Tensor):
    """Biased keys to (scores fp32, idx int64) as knn_decode_key writes them: key 0 is NaN (0xFFFFFFFF) and 2^32 - 1."""
    hi = torch.div(b, 1 << 32, rounding_mode="floor")
    low = b - hi * (1 << 32)
    o = hi + (1 << 31)
    u = torch.where(o >= 1 << 31, o & 0x7FFFFFFF, (~o) & 0xFFFFFFFF)
    u = torch.where(u >= 1 << 31, u - (1 << 32), u)
    return u.to(torch.int32).view(torch.float32), 0xFFFFFFFF - low


def top_keys(b: torch.Tensor, k: int) -> torch.Tensor:
    """The k largest biased keys per row, descending (I64_MIN past the candidates)."""
    if b.shape[1] < k:
        b = torch.cat([b, torch.full((b.shape[0], k - b.shape[1]), I64_MIN, dtype=b.dtype, device=b.device)], 1)
    return torch.topk(b, k, dim=1).values


def designed_topk(s: torch.Tensor, k: int, mask: torch.Tensor, row0: int = 0):
    """(scores fp32, idx int64) [Q, k]: the exact answer for designed scores s float64 [Q, N], empty slots decoded."""
    return decode(top_keys(biased_keys(s, mask, row0), k))


def materialize(hi: torch.Tensor, lo, D: int, Q: int):
    """fp16 operands of a design: R design rows of scores hi + lo [R, N] (lo None: one-hot, R <= D). Query q uses row
    q % R: it is 1 at column r and, with lo, at column D/2 + r, and X[j, r] = hi[r, j], X[j, D/2 + r] = lo[r, j]. With
    D >= 128 the two slots lie in different 64-wide K blocks. Returns (A16 [Q, D], X16 [N, D], s float64 [Q, N])."""
    R, N = hi.shape
    half = D if lo is None else D // 2
    assert R <= half
    X = torch.zeros(N, D, dtype=torch.float64)
    X[:, :R] = hi.T
    if lo is not None:
        X[:, half:half + R] = lo.T
    X16 = X.half()
    assert torch.equal(X16.double(), X), "a designed slot is not exact in fp16"
    A = torch.zeros(Q, D, dtype=torch.float16)
    r = torch.arange(Q) % R
    A[torch.arange(Q), r] = 1
    if lo is not None:
        A[torch.arange(Q), half + r] = 1
    s = hi if lo is None else hi + lo
    return A, X16, s[r]


# ---- the kernel's queue protocol, restated for the ordering only --------------------------------------------------
class Trace:
    """What queue_protocol saw: per chunk the queue counts before it and the pushes in it, merges, skipped tiles, and the
    epilogue slots (hr, column in the tile) that held a survivor."""

    def __init__(self):
        self.chunks = []    # dicts: block, stripe, tile, chunk, before [rows], pushed [rows], merge
        self.skipped = []   # (block, stripe, tile)
        self.busy = []      # (block, stripe, tile)
        self.slots = np.zeros((2, TILE), dtype=bool)


def queue_protocol(b: np.ndarray, k: int, splits: int = 1, seed=None, trace: Trace = None) -> np.ndarray:
    """knn_topk_kernel's ordering on biased keys b int64 [Q, N] (I64_MIN: not a candidate), then the stripe merge:
    per 64-row block and stripe, tiles of 256 columns; a tile where no row has a key above its threshold is skipped
    (the warpgroup OR); otherwise 32-column chunks push every key above the row's threshold (read before the chunk) to
    its queue, and when any row's queue passed 32, every row with a queue is merged into its k-list and its threshold
    becomes the list's k-th key (never lower than a seed). Returns the final biased lists [Q, k]."""
    Q, N = b.shape
    tiles = -(-N // TILE)
    tps = -(-tiles // splits)
    out = []
    for b0 in range(0, Q, BLOCK_M):
        kb = b[b0:b0 + BLOCK_M]
        rows = kb.shape[0]
        hr = (np.arange(rows) % 16) >= 8
        stripe_lists = [] if seed is None else [seed[b0:b0 + BLOCK_M]]
        for s in range(splits):
            lst = np.full((rows, k), I64_MIN, dtype=np.int64)
            th = np.full(rows, I64_MIN, dtype=np.int64) if seed is None else seed[b0:b0 + BLOCK_M, k - 1].copy()
            queue = np.full((rows, QCAP), I64_MIN, dtype=np.int64)
            cnt = np.zeros(rows, dtype=np.int64)

            def merge_all():
                for r in np.nonzero(cnt)[0]:
                    lst[r] = np.sort(np.concatenate([lst[r], queue[r, :cnt[r]]]))[::-1][:k]
                    th[r] = max(th[r], lst[r, k - 1])
                    cnt[r] = 0

            for t in range(s * tps, min(tiles, (s + 1) * tps)):
                cols = kb[:, t * TILE:min(N, (t + 1) * TILE)]
                if not (cols > th[:, None]).any():
                    if trace is not None:
                        trace.skipped.append((b0 // BLOCK_M, s, t))
                    continue
                if trace is not None:
                    trace.busy.append((b0 // BLOCK_M, s, t))
                for ch in range(TILE // CHUNK):
                    sub = cols[:, ch * CHUNK:(ch + 1) * CHUNK]
                    surv = sub > th[:, None]
                    before = cnt.copy()
                    for r in np.nonzero(surv.any(1))[0]:
                        v = sub[r, surv[r]]
                        queue[r, cnt[r]:cnt[r] + v.size] = v
                        cnt[r] += v.size
                    assert int(cnt.max()) <= QCAP, "a queue overflowed its 64 entries"
                    full = bool((cnt > QCAP - CHUNK).any())
                    if trace is not None:
                        trace.chunks.append(dict(block=b0 // BLOCK_M, stripe=s, tile=t, chunk=ch, before=before,
                                                 pushed=cnt - before, merge=full))
                        for h in (0, 1):
                            trace.slots[h, ch * CHUNK:ch * CHUNK + sub.shape[1]] |= surv[hr == bool(h)].any(0)
                    if full:
                        merge_all()
            merge_all()
            stripe_lists.append(lst)
        out.append(np.sort(np.concatenate(stripe_lists, 1), 1)[:, ::-1][:, :k])
    return np.concatenate(out, 0)


# ---- designs ----------------------------------------------------------------------------------------------------
def _frac(n):
    return n * 2.0 ** -10


SCHEDULE_TILES = 7  # tile 0 warm-up, tiles 1 ... 6 records, then a partial tile
SCHEDULE_N = SCHEDULE_TILES * TILE + 100
SCHEDULE_ROWS = 128  # two 64-row blocks: two-slot design rows at D = 256


def schedule_records(seed: int = 0):
    """{row: {global chunk: [positions in the chunk]}}: where each design row's records sit. Chunk c covers columns
    [32 c, 32 c + 32); chunks 0-7 are the warm-up tile. Block 0 (rows 0-63) follows a written plan (below), block 1
    and the last, partial tile a seeded random one."""
    g = np.random.default_rng(seed)
    rec = {r: {} for r in range(SCHEDULE_ROWS)}
    full = list(range(CHUNK))
    # tile 1 (chunks 8-15)
    rec[0][8], rec[0][9] = list(range(31)), full         # 31 queued, then a full chunk: 63
    rec[8][8], rec[8][9] = full, full                    # 32 queued, then a full chunk: a queue of exactly 64
    rec[9][8], rec[9][9] = [5], full                     # 1 + 32 = 33
    rec[1][9] = [17]                                     # one survivor, merged because other rows overflowed
    rec[2][10], rec[2][11] = [0], full                   # 33, the only row past 32: it alone forces the merge
    rec[10][11] = [3, 9, 14, 20, 31]                     # merged with row 2
    rec[5][13] = full                                    # 32 queued ...
    rec[13][12], rec[13][15] = list(range(0, 30, 3)), list(range(1, 31, 3))
    # tile 2 (chunks 16-23): a full chunk in every chunk for an hr = 0 row and an hr = 1 row: every register slot
    # (i, c, e) of both halves holds a survivor, and the queues overflow every second chunk, mid-tile; row 5's 32
    # (from tile 1) are merged when row 3 first overflows
    for c in range(16, 24):
        rec[3][c] = full
        rec[11][c] = full
    # tile 3: nothing (skipped); tile 4 (chunks 32-39): scattered records, row 6 past 32 after seven chunks
    for c in range(32, 40):
        for r in range(4, 64, 8):
            rec[r][c] = sorted({(r + 5 * c + d) % CHUNK for d in (0, 11, 23)})
        rec[6][c] = sorted({(7 * c + d) % CHUNK for d in (0, 6, 13, 19, 26)})
    # tile 5: nothing; tile 6 (chunks 48-55): a lone record at each end of the tile
    rec[63][48] = [0]
    rec[62][55] = [31]
    # the partial tile (chunks 56-59, 100 columns) for block 0, and every record tile for block 1
    sizes = [0, 0, 0, 1, 2, 3, 5, 9, 16, 31, 32]
    for r in range(SCHEDULE_ROWS):
        chunks = range(56, 60) if r < 64 else range(8, 60)
        for c in chunks:
            width = min(CHUNK, SCHEDULE_N - CHUNK * c)
            n = min(int(g.choice(sizes)), width)
            if n:
                rec[r][c] = sorted(g.choice(width, n, replace=False).tolist())
    return rec


def schedule_design(seed: int = 0):
    """(hi, lo) float64 [128, SCHEDULE_N] of the queue-schedule database. Tile 0 is a warm-up whose scores fall with
    the column (-1000 - j + a fraction), so after its merges every row holds a full list (k <= 128) and nothing later
    in the tile survives. Past it, a row's records (schedule_records) rise strictly: record m scores -900 + m (1/4 +
    2^-10), above everything before it, so each one survives and each chunk pushes exactly the records placed in it.
    Every other column scores about -2000 and never survives."""
    rec = schedule_records(seed)
    R, N = SCHEDULE_ROWS, SCHEDULE_N
    j = np.arange(N)
    s = np.empty((R, N))
    for r in range(R):
        s[r] = -2000.0 + _frac((j * 7 + r) % 1024)
        s[r, :TILE] = -1000.0 - j[:TILE] + _frac((r * 37 + j[:TILE]) % 1024)
        m = 0
        for c in sorted(rec[r]):
            for pos in rec[r][c]:
                s[r, CHUNK * c + pos] = -900.0 + m * (0.25 + 2.0 ** -10)
                m += 1
    hi = np.floor(s)
    return torch.from_numpy(hi), torch.from_numpy(s - hi)


def tie_design(N: int = 2000, seed: int = 1):
    """(hi, lo) [128, N]: scores from {-1, -0.5, 0, 0.5, 1, 1.5} (ties everywhere), and for each row a top score 5 at
    the columns on either side of chunk, tile and stripe boundaries, so a cut through them ties to the smaller index."""
    g = torch.Generator().manual_seed(seed)
    hi = torch.randint(-1, 2, (128, N), generator=g).double()
    lo = 0.5 * torch.randint(0, 2, (128, N), generator=g).double()
    hi[:, TIE_COLUMNS] = 5.0
    lo[:, TIE_COLUMNS] = 0.0
    return hi, lo


TIE_COLUMNS = [31, 32, 63, 64, 255, 256, 257, 511, 512, 767, 768, 1023, 1024, 1535, 1536, 1999]
