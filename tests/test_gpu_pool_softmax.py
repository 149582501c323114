"""GPU (-m gpu): mean_pool_kernel and log_softmax_rows_kernel against float64 (kernel_refs.mean_pool64 / log_softmax64).

  * mean pool: lengths 0, negative and past T - 1 (clamped; 0 gives NaN), lengths around the 8-row and 32-row unroll
    edges, E that is not a multiple of the 128 columns of a block; the <cls> row, every row past a sequence's length and
    a whole guard sequence behind the batch are NaN, so a row read that should not be shows in the result.
  * log-softmax rows: V on both sides of the lane / lane + 32 split, n around the 8 rows of a block, -inf entries, a row
    of -inf only (NaN, as torch), a dominant logit in the last column, the columns V .. ld of the pitched buffer NaN,
    targets at 0, 31, 32 and V - 1.

Both kernels are deterministic: a second run gives the same bits."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu


def _lib():
    from esm_b200 import _lib
    return _lib


def S():
    return torch.cuda.current_stream().cuda_stream


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def same_bits(a, b):
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(nan=0.0), b.nan_to_num(nan=0.0))


@pytest.mark.parametrize("E", [4, 132, 320, 1280])
@pytest.mark.parametrize("T", [80, 34])
def test_mean_pool_against_float64(T, E):
    L = _lib(); lib = L.load()
    lens = [n for n in (0, -5, 1, 2, 7, 8, 9, 15, 16, 17, 24, 25, 31, 32, 33, 39, 40, 41, 56, 57, 63, 64, 65)
            if n < T - 1] + [T - 2, T - 1, T, T + 100]
    B = len(lens)
    g = torch.Generator().manual_seed(T * E)
    buf = (torch.randn(B + 1, T, E, generator=g) * 2 + 0.7).cuda()
    buf[B] = float("nan")  # behind the batch
    x = buf[:B]
    x[:, 0] = float("nan")  # <cls>
    for b, n in enumerate(lens):
        x[b, 1 + max(n, 0):] = float("nan")
    lengths = torch.tensor(lens, dtype=torch.int32, device="cuda")
    obuf = torch.full((B + 1, E), float("nan"), device="cuda")
    out = obuf[:B]
    L.check(lib.esmb200_mean_pool(x.data_ptr(), lengths.data_ptr(), out.data_ptr(), B, T, E, S()))
    want = kr.mean_pool64(x, lengths)
    empty = torch.tensor([n <= 0 for n in lens], device="cuda")
    assert torch.equal(out.isnan().all(-1), empty) and torch.equal(out.isnan().any(-1), empty)
    assert torch.equal(want.isnan().all(-1), empty)
    assert bool(obuf[B].isnan().all())
    err = (out.double() - want).abs()[~empty]
    r = float((err / kr.mean_pool_bound(x, lengths)[~empty]).max())
    report(f"mean_pool T={T} E={E} B={B}", err_over_bound=r, max_abs=float(err.max()))
    assert r <= 1.0
    out2 = torch.full_like(out, float("nan"))
    L.check(lib.esmb200_mean_pool(x.data_ptr(), lengths.data_ptr(), out2.data_ptr(), B, T, E, S()))
    assert same_bits(out, out2)


def test_mean_pool_argument_checks():
    L = _lib(); lib = L.load()
    x, out = torch.zeros(2, 4, 8, device="cuda"), torch.zeros(2, 8, device="cuda")
    n = torch.ones(2, dtype=torch.int32, device="cuda")
    before = lib.esmb200_launch_count()
    assert lib.esmb200_mean_pool(x.data_ptr(), n.data_ptr(), out.data_ptr(), 2, 1, 8, S()) == -1   # no residue row
    assert lib.esmb200_mean_pool(x.data_ptr(), n.data_ptr(), out.data_ptr(), 2, 4, 6, S()) == -1   # E % 4
    assert b"E % 4" in lib.esmb200_last_error()
    assert lib.esmb200_mean_pool(x.data_ptr(), n.data_ptr(), out.data_ptr(), 0, 4, 8, S()) == -1
    assert lib.esmb200_mean_pool(x.data_ptr(), None, out.data_ptr(), 2, 4, 8, S()) == -1
    assert lib.esmb200_launch_count() == before


def softmax_rows(n, V, ld, seed):
    """[n, ld] logits, NaN in the columns >= V. Row i takes pattern i % 5: 0 a dominant logit in column V - 1 (lse ~ 0);
    1 uniform in [-80, 80]; 2 -inf entries among them; 3 -inf only; 4 nearly equal logits."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, ld, generator=g) * 160 - 80
    for i in range(n):
        k = i % 5
        if k == 0:
            x[i, V - 1] = 200.0
        elif k == 2:
            x[i, 0:V:3] = float("-inf")
        elif k == 3:
            x[i] = float("-inf")
        elif k == 4:
            x[i] = 3.0 + 1e-3 * torch.rand(ld, generator=g)
    x[:, V:] = float("nan")
    return x


@pytest.mark.parametrize("n", [1, 7, 8, 9, 1000])
@pytest.mark.parametrize("V", [1, 2, 31, 32, 33, 63, 64])
def test_log_softmax_rows_against_float64(V, n):
    L = _lib(); lib = L.load()
    ld = V + 3
    buf = torch.full((n + 1, ld), float("nan"))
    buf[:n] = softmax_rows(n, V, ld, seed=64 * n + V)
    buf = buf.cuda()
    x = buf[:n]
    obuf = torch.full((n + 1, V), float("nan"), device="cuda")
    out = obuf[:n]
    L.check(lib.esmb200_log_softmax_rows(x.data_ptr(), ld, n, V, None, out.data_ptr(), S()))
    want = kr.log_softmax64(x[:, :V])
    bound = kr.log_softmax_bound(x[:, :V])
    assert torch.equal(out.isnan(), want.isnan()) and torch.equal(out.isinf(), want.isinf())
    assert bool(obuf[n].isnan().all())
    assert bool(out[3::5].isnan().all()) and not bool(out[0::5].isnan().any())
    live = want.isfinite()
    assert torch.equal(out[want.isinf()].double(), want[want.isinf()])  # -inf stays -inf
    r = float(((out.double() - want).abs()[live] / bound[live]).max())
    assert float(out[0, V - 1]) == 0.0 or V == 1  # the dominant logit: log-probability 0
    # the target gather: columns 0, 31, 32 and V - 1 in turn
    tgt = torch.tensor([min(c, V - 1) for c in (0, 31, 32, V - 1)] * (n // 4 + 1), device="cuda")[:n]
    tbuf = torch.full((n + 1,), float("nan"), device="cuda")
    L.check(lib.esmb200_log_softmax_rows(x.data_ptr(), ld, n, V, tgt.data_ptr(), tbuf.data_ptr(), S()))
    assert same_bits(tbuf[:n], out.gather(1, tgt[:, None])[:, 0]) and bool(tbuf[n].isnan())
    out2 = torch.full_like(out, float("nan"))
    L.check(lib.esmb200_log_softmax_rows(x.data_ptr(), ld, n, V, None, out2.data_ptr(), S()))
    assert same_bits(out, out2)
    report(f"log_softmax_rows V={V} n={n}", err_over_bound=r, finite=float(live.sum()))
    assert r <= 1.0
