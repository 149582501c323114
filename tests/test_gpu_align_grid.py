"""GPU: the similarity kernels of the embedding alignment past one pass of their grid-stride loops, through the C ABI
(esmb200_align_similarity) with the output filled with NaN and the scratch with 0xFF bytes before every call.

A launch has at most 64 CTAs per pair (align_splits), so one pass of align_sim_kernel covers 64 tiles of 64 x 64,
and one pass of align_stats_kernel covers 512 rows (64 CTAs x 8 warps) and 16,384 columns (64 x 256 threads):

  1. S and the z-scored S' against float64 (tests/align_refs.py) with the bounds of tests/test_gpu_align.py: 2000 x 1500
     at E = 1280 (768 tiles, 2000 rows), 20,000 x 3 and 3 x 20,000 at D = 64 (rows, columns and tiles past a pass),
     alone and in batches of 3 and 4 pairs beside small ones;
  2. one-hot rows, where every S entry is one exact product or zero: S bit for bit;
  3. the programme on the 2000 x 1500 pair bit for bit against align_refs.align, local and global.
"""
import ctypes
import os
import struct
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # align_refs

import align_refs as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _similarity(qs, ts, zscore):
    """esmb200_align_similarity on fp16 rows qs[p] [La, D], ts[p] [Lb, D]: the S' of each pair, [La, Lb] fp32."""
    from esm_b200 import _lib
    lib = _lib.load()
    P, D = len(qs), qs[0].shape[1]
    La, Lb = [q.shape[0] for q in qs], [t.shape[0] for t in ts]
    off = lambda v: torch.tensor([0] + v, dtype=torch.int64).cumsum(0).to(DEV)  # noqa: E731
    q_off, t_off, s_off = off(La), off(Lb), off([a * b for a, b in zip(La, Lb)])
    n_q, n_t, n_cells = sum(La), sum(Lb), sum(a * b for a, b in zip(La, Lb))
    need = lib.esmb200_align_scratch_bytes(P, n_q, n_t, n_cells)
    scratch = torch.full((need,), 0xFF, dtype=torch.uint8, device=DEV)
    out = torch.full((n_cells,), float("nan"), device=DEV)
    q = torch.cat(qs).to(DEV).contiguous()
    t = torch.cat(ts).to(DEV).contiguous()
    rc = lib.esmb200_align_similarity(_p(q), _p(t), D, _p(q_off), _p(t_off), _p(s_off), P, n_q, n_t, n_cells,
                                      int(zscore), _p(out), _p(scratch), need, None)
    assert rc == 0, lib.esmb200_last_error()
    edges = s_off.tolist()
    return [out[edges[p]:edges[p + 1]].view(La[p], Lb[p]) for p in range(P)]


def _rows(L, D, seed):
    from esm_b200 import search
    g = torch.Generator().manual_seed(seed)
    return search.prepare_rows(torch.randn(L, D, generator=g).to(DEV), "cosine")


def _check(q16, t16, s, zscore):
    """The bounds of tests/test_gpu_align.py::test_similarity_against_float64, on the device in float64."""
    q, t = q16.to(DEV), t16.to(DEV)
    s64, bound = ref.sim_f64(q, t), ref.sim_bound(q, t)
    got = s.double()
    assert not bool(torch.isnan(got).any()), f"{int(torch.isnan(got).sum())} entries never written"
    if not zscore:
        err = (got - s64).abs() / bound
        assert bool((err <= 1).all()), float(err.max())
        return float(err.max())
    want = ref.zscore_f64(s64)
    sr = s64.std(1, unbiased=False, keepdim=True)
    sc = s64.std(0, unbiased=False, keepdim=True)
    b = bound.max()
    tol = 4 * 0.5 * (torch.where(sr > 0, b / sr.clamp_min(1e-300), 0 * sr) +
                     torch.where(sc > 0, b / sc.clamp_min(1e-300), 0 * sc)) + 1e-5 * (1 + want.abs())
    err = (got - want).abs() / tol
    assert bool((err <= 1).all()), float(err.max())
    return float(err.max())


SHAPES = [(2000, 1500, 1280), (20_000, 3, 64), (3, 20_000, 64)]


@pytest.mark.parametrize("zscore", [False, True])
@pytest.mark.parametrize("La,Lb,D", SHAPES)
def test_past_one_pass_of_the_grid(La, Lb, D, zscore):
    q, t = _rows(La, D, La), _rows(Lb, D, Lb + 1)
    (s,) = _similarity([q], [t], zscore)
    _check(q, t, s, zscore)


@pytest.mark.parametrize("zscore", [False, True])
@pytest.mark.parametrize("D", [64, 1280])
def test_past_one_pass_in_a_batch(D, zscore):
    """The long pairs of the D beside pairs of one row and of one tile edge: each pair's grid is its own."""
    pairs = [(20_000, 3), (1, 1), (3, 20_000), (65, 64)] if D == 64 else [(1, 1), (2000, 1500), (64, 65)]
    qs = [_rows(a, D, 10 + i) for i, (a, _) in enumerate(pairs)]
    ts = [_rows(b, D, 20 + i) for i, (_, b) in enumerate(pairs)]
    for q, t, s in zip(qs, ts, _similarity(qs, ts, zscore)):
        _check(q, t, s, zscore)


def _one_hot(L, D, seed):
    """Rows with one nonzero entry, a signed value k/8 (k in 1 ... 16), in a random column."""
    g = torch.Generator().manual_seed(seed)
    r = torch.zeros(L, D, dtype=torch.float16)
    col = torch.randint(0, D, (L,), generator=g)
    val = torch.randint(1, 17, (L,), generator=g).half() / 8 * (torch.randint(0, 2, (L,), generator=g) * 2 - 1).half()
    r[torch.arange(L), col] = val
    return r.to(DEV)


@pytest.mark.parametrize("La,Lb,D", [(2000, 1500, 1280), (20_000, 3, 64), (3, 20_000, 64)])
def test_one_hot_rows_are_exact(La, Lb, D):
    q, t = _one_hot(La, D, 1), _one_hot(Lb, D, 2)
    (s,) = _similarity([q], [t], False)
    want = (q.double() @ t.double().T).float()
    assert torch.equal(s, want)  # NaN (never written) fails too
    assert int((s != 0).sum()) > La * Lb // (4 * D)  # enough nonzero products to see a tile go missing


def _bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


@pytest.mark.parametrize("mode", ["local", "global"])
def test_the_programme_on_the_large_pair(mode):
    from esm_b200 import align
    q, t = _rows(2000, 1280, 2000), _rows(1500, 1280, 1501)
    t[200:900] = q[1000:1700]  # a long diagonal to find
    (s,) = _similarity([q], [t], True)
    a = align.align_matrices([s.cpu()], mode, 1.0, 0.1)[0]
    want = ref.align(s.cpu().numpy(), mode, 1.0, 0.1)
    assert _bits(a.score) == _bits(float(want[0])) and (a.query_span, a.target_span, a.ops) == tuple(want[1:])
    if mode == "local":
        assert a.query_span[1] - a.query_span[0] >= 700
