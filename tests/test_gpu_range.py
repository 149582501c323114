"""GPU: range search (esmb200_knn_range, esm_b200.search range_search). Designed exact scores through the kernel's
fixed thresholds and flushes (a score at tau is a hit, one ulp above it is not; ties across chunk, tile and stripe
edges; signed zeros; -inf and FLT_MAX thresholds), random rows against search() bit for bit and against a float64
restatement, independence of Q, batching, splits, the hit-buffer capacity and max_hits, the sharded index against the
resident one, and the CLI end to end. Outputs and buffers are filled with 0xFF or NaN first."""

import numpy as np
import pytest
import torch

from range_refs import range_expected
from search_refs import FLT_MAX, TIE_COLUMNS, candidates_mask, exact, materialize, tie_design

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _hits(Q, cap):
    return (torch.full((cap,), -1, dtype=torch.int64, device=DEV), torch.full((cap,), -1, dtype=torch.int32, device=DEV),
            torch.zeros(Q, dtype=torch.int64, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV))


def _kernel_csr(A, X, tau, alpha=1.0, beta=None, self_offset=-1, splits=None, chunks=None, max_hits=None, cap=None):
    """The kernel's CSR through knn_range (chunks: row bounds appended one after another) and knn_range_finish."""
    from esm_b200 import search
    Q, N = A.shape[0], X.shape[0]
    cap = Q * N if cap is None else cap
    hk, hr, counts, total = _hits(Q, cap)
    for g0, g1 in chunks or [(0, N)]:
        search.knn_range(A, X[g0:g1], g0, tau, hk, hr, counts, total, None if beta is None else beta[g0:g1], alpha,
                         self_offset, splits)
    t = int(total)
    assert t == int(counts.sum())
    return search.knn_range_finish(hk[:t], hr[:t], counts, max_hits), t


def _assert_csr(got, want):
    lims, s, i = got
    wl, ws, wi = want
    assert torch.equal(lims.cpu(), wl), "lims"
    assert torch.equal(s.cpu().view(torch.int32), ws.view(torch.int32)), "scores"
    assert torch.equal(i.cpu(), wi), "indices"


# ---- designed exact scores ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alpha", [1.0, -1.0])
@pytest.mark.parametrize("t", [1.0, "ulp_above_1", 0.0, -0.0, 5.0, float("-inf"), FLT_MAX, -FLT_MAX])
def test_designed_thresholds_are_exact(alpha, t):
    hi, lo = tie_design()
    A, X, s = materialize(hi, lo, 256, 130)
    s = alpha * s
    t = float(np.nextafter(np.float32(1.0), np.float32(2.0))) if t == "ulp_above_1" else t
    Q, N = A.shape[0], X.shape[0]
    tau = torch.full((Q,), t, dtype=torch.float32)
    mask = candidates_mask(Q, N, -1, "cpu")
    want = range_expected(s, mask, tau + 0.0)
    A, X = A.to(DEV), X.to(DEV)
    for splits in (1, 3, None):
        got, nnz = _kernel_csr(A, X, tau.to(DEV), alpha, splits=splits)
        _assert_csr(got, want)
    if t == float("-inf"):
        assert nnz == Q * N
    if t == FLT_MAX:
        assert nnz == 0


def test_designed_ties_self_and_chunks():
    """Ties at the tie columns cut by chunk, tile and stripe edges; the self column left out at chunk edges; chunks
    appended in any order and max_hits cutting through ties."""
    hi, lo = tie_design()
    A, X, s = materialize(hi, lo, 256, 200)
    Q, N = A.shape[0], X.shape[0]
    tau = torch.full((Q,), 1.5, dtype=torch.float32)
    for self_offset in (-1, 0, 700):
        mask = candidates_mask(Q, N, self_offset, "cpu")
        want = range_expected(s, mask, tau)
        for chunks in ([(0, N)], [(0, 256), (256, 768), (768, N)], [(1536, N), (0, 1), (1, 1536)]):
            got, _ = _kernel_csr(A.to(DEV), X.to(DEV), tau.to(DEV), self_offset=self_offset, chunks=chunks)
            _assert_csr(got, want)
        for M in (1, 7, 16):
            got, _ = _kernel_csr(A.to(DEV), X.to(DEV), tau.to(DEV), self_offset=self_offset, max_hits=M)
            _assert_csr(got, range_expected(s, mask, tau, max_hits=M))
    assert len(TIE_COLUMNS) == 16


def test_counting_past_capacity_is_exact():
    hi, lo = tie_design()
    A, X, s = materialize(hi, lo, 256, 70)
    Q, N = A.shape[0], X.shape[0]
    tau = torch.full((Q,), 0.5, dtype=torch.float32, device=DEV)
    want = (s >= 0.5).sum(1)
    from esm_b200 import search
    for cap in (0, 1, 100, int(want.sum()) - 1):
        hk, hr, counts, total = _hits(Q, cap)
        search.knn_range(A.to(DEV), X.to(DEV), 0, tau, hk, hr, counts, total)
        assert torch.equal(counts.cpu(), want) and int(total) == int(want.sum())
        assert bool((hr[:cap] >= 0).all())


# ---- random rows -------------------------------------------------------------------------------------------------------
def _index(metric, N=3000, E=320, seed=0):
    from esm_b200 import search
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn(20, E, generator=g)
    x = centres[torch.randint(0, 20, (N,), generator=g)] + 0.6 * torch.randn(N, E, generator=g)
    return search.EmbeddingIndex(x.to(DEV), metric=metric), x


def _thr(metric, v):
    return {"min_score": v} if metric == "cosine" else {"max_distance": v}


@pytest.mark.parametrize("metric,v", [("cosine", 0.6), ("cosine", 0.3), ("l2", 14.0), ("l2", 16.0)])
def test_random_rows_agree_with_search(metric, v):
    index, x = _index(metric)
    q = x[:150] + 0.1
    lims, sc, ix = index.range_search(q, **_thr(metric, v))
    la, sa, ia = index.range_search_all(**_thr(metric, v))
    assert int(lims[-1]) > 0 and int(la[-1]) > 0, "the thresholds should give hits"
    for (L, S, I), tops in (((lims, sc, ix), [index.search(q, k) for k in (1, 10, 128)]),
                            ((la, sa, ia), [index.search_all(k) for k in (1, 10, 128)])):
        for ts, ti in tops:
            k = ts.shape[1]
            for i in range(ts.shape[0]):
                a, b = int(L[i]), int(L[i + 1])
                c = min(b - a, k)
                assert torch.equal(S[a:a + c].view(torch.int32), ts[i, :c].view(torch.int32)) and \
                    torch.equal(I[a:a + c], ti[i, :c]), f"query {i}: range and search(k={k}) differ"
                if b - a < k:  # the next neighbour fails the threshold
                    nxt = float(ts[i, b - a])
                    assert (nxt < v) if metric == "cosine" else (nxt > v)
    # float64 restatement outside the ambiguity band (cosine)
    if metric == "cosine":
        from esm_b200 import search as S_
        A16 = S_.prepare_rows(q.to(DEV), metric)
        s64, tol = exact(A16, index.rows)
        got = torch.zeros_like(s64, dtype=torch.bool)
        rows = torch.repeat_interleave(torch.arange(q.shape[0], device=DEV), lims.diff())
        got[rows, ix] = True
        assert not bool((got & (s64 + tol < v)).any()), "a hit below the threshold past the band"
        assert not bool((~got & (s64 - tol > v)).any()), "a missed hit above the threshold past the band"


@pytest.mark.parametrize("metric,v", [("cosine", 0.5), ("l2", 15.0)])
def test_independence_of_batching_capacity_and_max_hits(monkeypatch, metric, v):
    from esm_b200 import search
    index, x = _index(metric, N=2000)
    q = x[:300] * 1.01
    ref = index.range_search(q, **_thr(metric, v))
    full = ref[0]
    for Q in (1, 63, 64, 65):
        got = index.range_search(q[:Q], **_thr(metric, v))
        assert torch.equal(got[0], full[:Q + 1])
        n = int(full[Q])
        assert torch.equal(got[1], ref[1][:n]) and torch.equal(got[2], ref[2][:n])
    monkeypatch.setattr(search, "QUERY_BATCH", 70)  # past one batch
    for r, g in zip(ref, index.range_search(q, **_thr(metric, v))):
        assert torch.equal(r, g)
    biggest = int(full.diff().max())
    monkeypatch.setattr(search, "RANGE_HIT_BYTES", search.HIT_BYTES * (biggest + 5))  # overflow and re-run
    for r, g in zip(ref, index.range_search(q, **_thr(metric, v))):
        assert torch.equal(r, g)
    all_ref = index.range_search_all(**_thr(metric, v))
    monkeypatch.setattr(search, "RANGE_HIT_BYTES", 1 << 30)
    for r, g in zip(all_ref, index.range_search_all(**_thr(metric, v))):
        assert torch.equal(r, g)
    for M in (1, 5, 200):
        L, S, I = index.range_search(q, **_thr(metric, v), max_hits=M)
        for i in range(q.shape[0]):
            a, b = int(full[i]), int(full[i + 1])
            c = min(M, b - a)
            assert int(L[i + 1] - L[i]) == c
            assert torch.equal(S[int(L[i]):int(L[i]) + c], ref[1][a:a + c])
            assert torch.equal(I[int(L[i]):int(L[i]) + c], ref[2][a:a + c])
    monkeypatch.setattr(search, "RANGE_HIT_BYTES", search.HIT_BYTES * (biggest - 1))
    with pytest.raises(ValueError, match=f"{biggest} hits at"):
        index.range_search(q, **_thr(metric, v))


def test_everything_and_nothing():
    index, x = _index("cosine", N=700)
    L, S, I = index.range_search_all(min_score=float("-inf"))
    assert int(L[-1]) == 700 * 699 and bool((I.view(700, 699) != torch.arange(700, device=DEV)[:, None]).all())
    L, S, I = index.range_search(x[:5], min_score=float("-inf"))
    assert int(L[-1]) == 5 * 700
    L, S, I = index.range_search(x[:5], min_score=1.5)
    assert torch.equal(L, torch.zeros(6, dtype=torch.int64, device=DEV)) and S.numel() == 0


# ---- sharded ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric,v", [("cosine", 0.5), ("l2", 15.0)])
def test_sharded_equals_resident(tmp_path, monkeypatch, metric, v):
    from esm_b200 import search
    index, x = _index(metric, N=2500, seed=4)
    with search.IndexWriter(tmp_path / "db", x.shape[1], metric, shard_rows=700) as w:
        w.add(x)
    sh = search.ShardedIndex.open(tmp_path / "db")
    q = x[:90] + 0.05
    ref, ref_all = index.range_search(q, **_thr(metric, v)), index.range_search_all(**_thr(metric, v))
    row = search._row_bytes(index.rows.shape[1], metric)
    for tiles in (1, 3, 100):
        monkeypatch.setattr(search, "MAX_SLOT_BYTES", tiles * search.TILE * row)
        for r, g in zip(ref, sh.range_search(q, **_thr(metric, v))):
            assert torch.equal(r, g)
        for r, g in zip(ref_all, sh.range_search_all(**_thr(metric, v))):
            assert torch.equal(r, g)
    # a small device budget: query blocks and a small hit buffer, so blocks overflow and are re-streamed
    monkeypatch.setattr(search, "MAX_SLOT_BYTES", 256 << 20)
    biggest = int(ref_all[0].diff().max())
    monkeypatch.setattr(search, "RANGE_HIT_BYTES", search.HIT_BYTES * (biggest + 10))
    for r, g in zip(ref_all, sh.range_search_all(**_thr(metric, v), max_device_bytes=4 << 20)):
        assert torch.equal(r, g)


# ---- the CLI end to end -------------------------------------------------------------------------------------------------
def test_cli_range_end_to_end(tmp_path):
    from esm_b200 import search_cli
    g = torch.Generator().manual_seed(7)
    E, layer = 128, 6
    centre = torch.randn(E, generator=g)
    d = tmp_path / "extract"
    d.mkdir()
    for i in range(400):
        v = centre + (0.3 if i < 300 else 3.0) * torch.randn(E, generator=g)
        torch.save({"label": f"p{i:03d}", "mean_representations": {layer: v}}, d / f"p{i:03d}.pt")
    p = search_cli.create_parser()
    search_cli.run(p.parse_args(["build", str(d), "--layer", str(layer), "--out", str(tmp_path / "db.pt")]))
    search_cli.run(p.parse_args(["build", str(d), "--layer", str(layer), "--out", str(tmp_path / "db")]))
    outs = []
    for db in ("db.pt", "db"):
        out = tmp_path / f"{db}.tsv"
        n = search_cli.run(p.parse_args(["range", str(tmp_path / db), "--all", "--min-score", "0.8", "--out",
                                         str(out)]))
        lines = out.read_text().splitlines()[1:]
        assert n == len(lines) > 0
        outs.append(lines)
    assert outs[0] == outs[1]
    per_query = {}
    for line in outs[0]:
        per_query[line.split("\t")[0]] = per_query.get(line.split("\t")[0], 0) + 1
    assert max(per_query.values()) > 128
