"""GPU: esmb200_knn_search and esmb200_knn_search_accumulate / esmb200_knn_decode on designed exact scores
(tests/search_refs.py): every score is exact in fp32, so the kernels must return the exact top k under (score
descending, index ascending), compared bit for bit on scores and indices, with no ambiguity band. Scratch and outputs
are filled with 0xFF bytes before every call, so a list that was never written would decode as the largest key.

  1. the queue schedules (search_refs.schedule_design; the host tests show which queue counts, merges and skips each
     reaches), ties across chunk, tile and stripe boundaries, signed zeros and extreme betas, Q in {1, 64, 65, 200};
  2. the stripe merge at every list slot: 1024 tiles with the winners in the last stripes, splits from 1 to 1024 and
     more stripes than tiles;
  3. the streamed pair on ragged chunks fed forward, reversed and shuffled, per-chunk splits up to 1024 (the running
     list as list 1024), the partial lists after every chunk (empty slots NaN and 2^32 - 1), self_offset across chunk
     edges, and indices at the top of the 2^31 range;
  4. strided query and database rows, alpha and beta of either sign.
"""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # search_refs, kernel_refs

import search_refs as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
KS = [1, 31, 32, 33, 64, 127, 128]
QS = [1, 64, 65, 200]


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _poisoned(nbytes):
    return torch.full((max(nbytes, 16),), 0xFF, dtype=torch.uint8, device=DEV)


def _search(A, X, k, beta=None, alpha=1.0, self_offset=-1, splits=1):
    """esmb200_knn_search into 0xFF-filled scratch and outputs. A, X: fp16 [*, D] with unit column stride."""
    from esm_b200 import _lib
    lib = _lib.load()
    Q, N, D = A.shape[0], X.shape[0], A.shape[1]
    scratch = _poisoned(splits * Q * k * 8)
    scores = torch.full((Q, k), -1, dtype=torch.int32, device=DEV).view(torch.float32)
    idx = torch.full((Q, k), -1, dtype=torch.int64, device=DEV)
    rc = lib.esmb200_knn_search(_p(A), A.stride(0), Q, _p(X), X.stride(0), N, D, _p(beta), float(alpha), self_offset,
                                k, splits, _p(scratch), scratch.numel(), _p(scores), _p(idx), None)
    assert rc == 0, lib.esmb200_last_error()
    return scores, idx


def _accumulate(A, X, row0, k, keys, beta=None, alpha=1.0, self_offset=-1, splits=1):
    from esm_b200 import _lib
    lib = _lib.load()
    Q, n, D = A.shape[0], X.shape[0], A.shape[1]
    scratch = _poisoned(splits * Q * k * 8)
    rc = lib.esmb200_knn_search_accumulate(_p(A), A.stride(0), Q, _p(X), X.stride(0), n, row0, D, _p(beta),
                                           float(alpha), self_offset, k, splits, _p(scratch), scratch.numel(),
                                           _p(keys), None)
    assert rc == 0, lib.esmb200_last_error()


def _decode(keys):
    from esm_b200 import search
    Q, k = keys.shape
    scores = torch.full((Q, k), -1, dtype=torch.int32, device=DEV).view(torch.float32)
    idx = torch.full((Q, k), -1, dtype=torch.int64, device=DEV)
    search.knn_decode(keys, scores, idx)
    return scores, idx


def _assert_same(got, want, what=""):
    gs, gi = got
    ws, wi = want
    gs, gi, ws, wi = gs.cpu(), gi.cpu(), ws.cpu(), wi.cpu()
    bad = (gs.view(torch.int32) != ws.view(torch.int32)) | (gi != wi)
    if bool(bad.any()):
        q, r = [int(v) for v in torch.nonzero(bad)[0]]
        raise AssertionError(f"{what}: {int(bad.sum())} entries differ; first at query {q} rank {r}: got "
                             f"({float(gs[q, r])!r}, {int(gi[q, r])}), want ({float(ws[q, r])!r}, {int(wi[q, r])})")


def _on(A, X, *rest):
    return (A.to(DEV), X.to(DEV)) + tuple(r.to(DEV) if isinstance(r, torch.Tensor) else r for r in rest)


def _all(s):
    return torch.ones_like(s, dtype=torch.bool)


# ---- 1. schedules, ties, signed zeros, extremes --------------------------------------------------------------------
@pytest.fixture(scope="module")
def schedule():
    return ref.schedule_design()


@pytest.mark.parametrize("Q", QS)
@pytest.mark.parametrize("k", KS)
def test_queue_schedules(schedule, k, Q):
    A, X, s = ref.materialize(*schedule, 256, Q)
    A, X = _on(A, X)
    want = ref.designed_topk(s, k, _all(s))
    _assert_same(_search(A, X, k), want, "splits 1")
    _assert_same(_search(A, X, k, splits=3), want, "splits 3")


@pytest.mark.parametrize("splits", [1, 2, 3, 7, 8, 13])
def test_ties_across_chunk_tile_and_stripe_boundaries(splits):
    hi, lo = ref.tie_design()
    for Q, k in ((200, 11), (65, 128), (1, 16)):
        A, X, s = ref.materialize(hi, lo, 256, Q)
        A, X = _on(A, X)
        _assert_same(_search(A, X, k, splits=splits), ref.designed_topk(s, k, _all(s)), f"Q {Q} k {k}")


@pytest.mark.parametrize("Q", QS)
@pytest.mark.parametrize("k", [1, 64, 128])
def test_signed_zeros_rank_as_plus_zero(k, Q):
    """A database of zero rows: acc = +0, and with alpha = -1 and beta_j = -0 on odd j, +0 on even j, half the fmaf
    results are -0. Every score must come back +0, the indices 0 ... k-1."""
    N = 1000
    A = torch.zeros(Q, 64, dtype=torch.float16, device=DEV)
    A[:, 0] = 1
    X = torch.zeros(N, 64, dtype=torch.float16, device=DEV)
    beta = torch.zeros(N, device=DEV)
    beta[1::2] = -0.0
    assert int(beta.view(torch.int32)[1]) == -(1 << 31)
    want = (torch.zeros(Q, k), torch.arange(k).expand(Q, k))
    for splits in (1, 4):
        _assert_same(_search(A, X, k, beta, -1.0, splits=splits), want, f"splits {splits}")
    # and the same zeros among nonzero scores: the +0 group ranks by index between the positives and negatives
    beta[:300:3] = 2.0 ** -20
    beta[600::5] = -(2.0 ** -20)
    s = beta.double().cpu().expand(Q, N).clone()
    _assert_same(_search(A, X, k, beta, -1.0, splits=2), ref.designed_topk(s, k, _all(s)), "mixed")


def _extreme_beta(N, seed):
    vals = [float("inf"), -float("inf"), ref.FLT_MAX, -ref.FLT_MAX, 2.0 ** -149, -(2.0 ** -149), 2.0 ** -126,
            2.0 ** -126 - 2.0 ** -149, -(2.0 ** -126 - 2.0 ** -149), 0.0, -0.0, 1.0, -1.0, 3.0e38]
    g = torch.Generator().manual_seed(seed)
    return torch.tensor(vals).float().double()[torch.randint(0, len(vals), (N,), generator=g)]


@pytest.mark.parametrize("Q", QS)
@pytest.mark.parametrize("alpha", [1.0, -1.0])
def test_extreme_betas_with_k_equal_to_n(alpha, Q):
    """beta of +-inf, +-FLT_MAX, subnormals and signed zeros over zero rows (s = beta exactly), k = N = 128: every
    candidate comes back, the -inf ones ahead of any empty slot. Then over designed rows: acc + inf = inf exactly."""
    N = 128
    beta = _extreme_beta(N, int(alpha > 0) + Q)
    A = torch.zeros(Q, 64, dtype=torch.float16)
    A[:, 1] = 1
    X = torch.zeros(N, 64, dtype=torch.float16)
    s = beta.expand(Q, N).clone()
    A, X, b = _on(A, X, beta.float())
    for splits in (1, 2):
        _assert_same(_search(A, X, N, b, alpha, splits=splits), ref.designed_topk(s, N, _all(s)), f"splits {splits}")
    # designed acc in [-2048, 2048] beside +-inf betas and finite exact ones
    g = torch.Generator().manual_seed(Q)
    hi = torch.randint(-2048, 2049, (64, 700), generator=g).double()
    beta = torch.randint(-4, 5, (700,), generator=g).double() * 0.5
    beta[::7] = float("inf")
    beta[3::11] = -float("inf")
    A, X, acc = ref.materialize(hi, None, 64, Q)
    s = alpha * acc + beta[None]
    A, X, b = _on(A, X, beta.float())
    for k in (1, 100, 128):
        _assert_same(_search(A, X, k, b, alpha, splits=2), ref.designed_topk(s, k, _all(s)), f"k {k}")


# ---- 2. the stripe merge's list slots ------------------------------------------------------------------------------
MERGE_TILES = 1024
MERGE_N = MERGE_TILES * ref.TILE


@pytest.fixture(scope="module")
def merge_db():
    """D = 64, one-hot queries: background scores 1 ... 8 (ties), 160 winners per query column (scores 100 ...)
    placed in tiles 768 ... 1023 and always in the last tile, so for splits = 1024 they sit in stripes >= 768, the
    merge kernel's fourth list slot (stripes t + 256 m, m = 3)."""
    g = torch.Generator().manual_seed(7)
    X = (torch.arange(MERGE_N) % 8 + 1).double()[:, None].repeat(1, 64)
    for c in range(64):
        rows = torch.cat([MERGE_N - 1 - torch.arange(8) * 37,
                          768 * ref.TILE + torch.randperm(256 * ref.TILE - 1000, generator=g)[:152]])
        X[rows, c] = 100.0 + torch.randperm(1900, generator=g)[:160].double()
    A = torch.eye(64, dtype=torch.float16)
    s = X.T.contiguous().to(DEV)  # query c scores column c
    return A.to(DEV), X.half().to(DEV), s


def _slots_reached(splits, tiles):
    """The merge kernel's list slots m (list t + 256 m) that hold a nonempty stripe."""
    tps = -(-tiles // splits)
    stripes = -(-tiles // tps)
    return sorted({s // 256 for s in range(stripes)})


@pytest.mark.parametrize("splits", [1, 31, 32, 33, 255, 256, 257, 511, 512, 513, 767, 768, 769, 1023, 1024])
def test_merge_slots(merge_db, splits):
    A, X, s = merge_db
    k = 128
    want = ref.designed_topk(s, k, _all(s))
    assert int(want[1].min()) >= 768 * ref.TILE  # every winner lies in the last quarter of the tiles
    _assert_same(_search(A, X, k, splits=splits), want, f"splits {splits}, slots {_slots_reached(splits, 1024)}")


@pytest.mark.parametrize("tiles,splits", [(1, 2), (3, 64), (12, 1024), (300, 1024), (767, 1024)])
def test_more_stripes_than_tiles(merge_db, tiles, splits):
    """Stripes past the last tile still write their (empty) lists: the 0xFF scratch would otherwise win."""
    A, X, s = merge_db
    n = tiles * ref.TILE - 5
    Xs, ss = X[MERGE_N - n:], s[:, MERGE_N - n:]
    for k in (1, 128):
        _assert_same(_search(A, Xs, k, splits=splits), ref.designed_topk(ss, k, _all(ss)), f"k {k}")


# ---- 3. the streamed pair --------------------------------------------------------------------------------------------
SIZES = [1, 7, 255, 256, 257, 1000, 3, 64, 49]  # sums to SCHEDULE_N = 1892
SPLITS = [1, 1024, 3, 257, 1, 1024, 64, 1024, 2]


def _chunks():
    assert sum(SIZES) == ref.SCHEDULE_N
    edges = torch.tensor([0] + SIZES).cumsum(0).tolist()
    return list(zip(edges[:-1], edges[1:]))


@pytest.mark.parametrize("order", ["forward", "reversed", "shuffled"])
@pytest.mark.parametrize("Q,k", [(65, 128), (200, 33), (1, 1)])
def test_accumulate_ragged_chunks_in_any_order(schedule, order, Q, k):
    A, X, s = ref.materialize(*schedule, 256, Q)
    A, X = _on(A, X)
    chunks = _chunks()
    if order == "reversed":
        chunks = chunks[::-1]
    elif order == "shuffled":
        chunks = [chunks[i] for i in torch.randperm(len(chunks), generator=torch.Generator().manual_seed(Q + k))]
    keys = torch.zeros(Q, k, dtype=torch.int64, device=DEV)
    seen = torch.zeros(ref.SCHEDULE_N, dtype=torch.bool)
    for step, ((a, b), sp) in enumerate(zip(chunks, SPLITS)):
        _accumulate(A, X[a:b], a, k, keys, splits=sp)
        seen[a:b] = True
        mask = seen.expand(Q, -1)
        want = ref.top_keys(ref.biased_keys(s, mask), k)
        got = ref.raw_keys(keys.cpu())  # the stored uint64 keys, biased as search_refs orders them
        assert torch.equal(got, want), f"running list after chunk {step} ({a}, {b}), splits {sp}"
        _assert_same(_decode(keys), ref.decode(want), f"decoded after chunk {step}")  # empty: NaN, 2^32 - 1
    final = ref.designed_topk(s, k, _all(s))
    _assert_same(_decode(keys), final, "final")
    _assert_same(_search(A, X, k), final, "resident")


@pytest.mark.parametrize("offset", [0, 1, 255, 300])
def test_accumulate_self_offset_across_ragged_chunks(schedule, offset):
    """Query q's own row q + offset is made its best candidate, so leaving it out is visible; chunk edges fall on
    and beside those rows."""
    hi, lo = schedule
    Q, k = 200, 64
    hi = hi.clone()
    # query q's design row is q % 128: boost column q + offset for the first 128 queries (shared by q + 128)
    for q in range(min(Q, 128)):
        hi[q, q + offset] = 2000.0
    A, X, s = ref.materialize(hi, lo, 256, Q)
    mask = ref.candidates_mask(Q, ref.SCHEDULE_N, offset, "cpu")
    A, X = _on(A, X)
    keys = torch.zeros(Q, k, dtype=torch.int64, device=DEV)
    for (a, b), sp in zip(_chunks(), SPLITS):
        _accumulate(A, X[a:b], a, k, keys, self_offset=offset, splits=sp)
    want = ref.designed_topk(s, k, mask)
    _assert_same(_decode(keys), want, "streamed")
    _assert_same(_search(A, X, k, self_offset=offset), want, "resident")


def test_accumulate_indices_at_the_top_of_the_range(schedule):
    """row0 = 2^31 - 1 - n: the last global row is 2^31 - 2, and indices decode exactly there."""
    Q, k = 65, 128
    A, X, s = ref.materialize(*schedule, 256, Q)
    A, X = _on(A, X)
    n = ref.SCHEDULE_N
    top = (1 << 31) - 1 - n
    want = ref.designed_topk(s, k, _all(s), row0=top)
    assert int(want[1].min()) >= top and int(want[1].max()) >= (1 << 31) - 2 - 50
    for cuts in ([(0, n)], [(0, 700), (700, n)], [(1000, n), (0, 1000)]):
        keys = torch.zeros(Q, k, dtype=torch.int64, device=DEV)
        for (a, b), sp in zip(cuts, (1024, 2)):
            _accumulate(A, X[a:b], top + a, k, keys, splits=sp)
        _assert_same(_decode(keys), want, f"cuts {cuts}")


# ---- 4. strides, alpha and beta ------------------------------------------------------------------------------------
def test_strided_rows_equal_the_contiguous_call(schedule):
    Q, k = 65, 64
    A, X, s = ref.materialize(*schedule, 256, Q)
    A, X = _on(A, X)
    Aw = torch.full((Q, 256 + 72), float("nan"), dtype=torch.float16, device=DEV)
    Xw = torch.full((X.shape[0], 256 + 136), float("nan"), dtype=torch.float16, device=DEV)
    Aw[:, 64:320], Xw[:, 128:384] = A, X
    As, Xs = Aw[:, 64:320], Xw[:, 128:384]
    assert As.stride(0) == 328 and Xs.stride(0) == 392 and not As.is_contiguous()
    want = ref.designed_topk(s, k, _all(s))
    _assert_same(_search(As, Xs, k), want, "strided")
    _assert_same(_search(A, X, k), want, "contiguous")
    keys = torch.zeros(Q, k, dtype=torch.int64, device=DEV)
    for (a, b), sp in zip(_chunks(), SPLITS):
        _accumulate(As, Xs[a:b], a, k, keys, splits=sp)
    _assert_same(_decode(keys), want, "strided, streamed")


@pytest.mark.parametrize("alpha", [-1.0, 0.5, -0.375, 3.0, -2.0 ** -6])
def test_alpha_and_beta_of_either_sign(alpha):
    """s = alpha acc + beta_j with acc in [-64, 64) in steps of 2^-10 and beta a multiple of 2^-12 in [-64, 64]: the
    fma is exact, so a negative alpha must rank the smallest acc first."""
    g = torch.Generator().manual_seed(int(abs(alpha) * 1000))
    R, N, Q = 100, 3000, 200
    hi = torch.randint(-64, 64, (R, N), generator=g).double()
    lo = torch.randint(0, 1024, (R, N), generator=g).double() * 2.0 ** -10
    beta = torch.randint(-(1 << 18), (1 << 18) + 1, (N,), generator=g).double() * 2.0 ** -12
    A, X, acc = ref.materialize(hi, lo, 256, Q)
    s = alpha * acc + beta[None]
    A, X, b = _on(A, X, beta.float())
    for k in (1, 77, 128):
        want = ref.designed_topk(s, k, _all(s))
        _assert_same(_search(A, X, k, b, alpha, splits=5), want, f"k {k}")
        keys = torch.zeros(Q, k, dtype=torch.int64, device=DEV)
        for a in range(0, N, 1100):
            e = min(N, a + 1100)
            _accumulate(A, X[a:e], a, k, keys, b[a:e], alpha, splits=7)
        _assert_same(_decode(keys), want, f"streamed, k {k}")
