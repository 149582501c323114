"""GPU (-m gpu): the standalone contact pass, esmb200_contact_accumulate + esmb200_contact_finalize (the path of the
fp32x3 layers, the MSA row maps and caller-supplied attentions), against float64 at the kernels' own outputs.

  * accumulate: maps that are real softmaxes of random logits at a flat and a sharp gain, padded query rows and key
    columns zero, read as one layer's slice of a stacked [B,L,H,T,T] tensor (batch_stride); S at the edges of the
    16-row stripes, the 32-column lane groups and both instantiations (S <= 512, S > 512); crops (1, T-1), (0, T) and
    (3, T-2); keep NULL or with <eos> mid-sequence; two layers added into an accumulator that starts non-zero; row_sum
    and every col_part stripe, the partial last one included, compared on their own (kernel_refs.contact_stripes).
  * finalize: C = layers * heads around the 16-channel slabs and at 660, bias NULL or given, logits out to |z| ~ 90
    (__expf saturates: the output must stay in [0, 1]); the logit is rebuilt from the output where |z| < 10 and held
    to the bound of its fp32 evaluation; two runs give the same bits.
  * both together give the contacts of kernel_refs.contacts_from_partials."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

U = kr.U32


def _lib():
    from esm_b200 import _lib
    return _lib


def S_():
    return torch.cuda.current_stream().cuda_stream


def P(t):
    return t.data_ptr() if t is not None else None


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def make_maps(B, L, H, T, gains, valid, seed):
    """[B,L,H,T,T] fp32: softmax over the first valid[b] keys of gain * N(0,1) logits (head h takes gains[h % 2]); the
    rows of the other queries and the columns of the other keys are zero, as the stack writes them."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(B, L, H, T, T, device="cuda", generator=g)
    a *= torch.tensor([gains[h % 2] for h in range(H)], device="cuda")[None, None, :, None, None]
    pos = torch.arange(T, device="cuda")
    for b in range(B):
        a[b, ..., pos >= valid[b]] = float("-inf")
    a = torch.softmax(a, -1)
    for b in range(B):
        a[b, :, :, pos >= valid[b]] = 0.0
    return a


CROPS = {"cls_eos": (1, -1, 2), "whole": (0, 0, 0), "inner": (3, -2, 5)}  # lo, hi - T, T - S

# (S, H, crop, keep given)
ACC_CASES = [(1, 5, "cls_eos", True), (15, 1, "whole", False), (16, 20, "inner", True), (17, 5, "cls_eos", True),
             (63, 40, "cls_eos", False), (64, 5, "whole", True), (65, 20, "inner", True), (511, 5, "cls_eos", True),
             (512, 40, "cls_eos", True), (513, 5, "whole", False), (1022, 5, "cls_eos", True),
             (1024, 20, "whole", True), (1024, 1, "inner", False)]


def accumulate(attn, l, w, keep8, acc, lo, hi):
    """esmb200_contact_accumulate on layer l of the stacked attn [B,L,H,T,T]; row_sum and col_part start as NaN"""
    L_ = _lib()
    B, L, H, T, _ = attn.shape
    S = hi - lo
    row = torch.full((B, H, S), float("nan"), device="cuda")
    col = torch.full((B, H, (S + 15) // 16, S), float("nan"), device="cuda")
    L_.check(L_.load().esmb200_contact_accumulate(attn.data_ptr() + l * H * T * T * 4, L * H * T * T,
                                                  w.data_ptr() + l * H * 4, P(keep8), P(acc), P(row), P(col), B, H, T,
                                                  lo, hi, S_()))
    return row, col


def finalize(acc, u, a1, bias):
    L_ = _lib()
    B, C, S = a1.shape
    out = torch.full((B, S, S), float("nan"), device="cuda")
    L_.check(L_.load().esmb200_contact_finalize(P(acc), P(u), P(a1), P(bias), P(out), B, C, S, S_()))
    return out


@pytest.mark.parametrize("S,H,crop,with_keep", ACC_CASES)
def test_accumulate_against_float64(S, H, crop, with_keep):
    B, L = 2, 2
    lo, dhi, dT = CROPS[crop]
    T = S + dT
    hi = T + dhi
    valid = [T, max(1, 2 * T // 3)]
    attn = make_maps(B, L, H, T, (0.5, 6.0), valid, seed=S + H)
    keep = None
    if with_keep:  # <eos> is each sequence's last valid token: the end of the first, mid-way in the second
        keep = torch.ones(B, T, dtype=torch.bool, device="cuda")
        for b in range(B):
            keep[b, valid[b] - 1] = False
    keep8 = keep.to(torch.uint8) if with_keep else None
    g = torch.Generator().manual_seed(S * H)
    w = torch.randn(L, H, generator=g).cuda()
    acc0 = torch.randn(B, S, S, generator=g).cuda()
    acc = acc0.clone()
    acc_ref, acc_abs = acc0.double(), acc0.double().abs()
    worst = {"row": 0.0, "col": 0.0}
    rows, cols, rows64, cols64 = [], [], [], []
    for l in range(L):
        row, col = accumulate(attn, l, w, keep8, acc, lo, hi)
        a_l, row_ref, col_ref = kr.contact_stripes(attn[:, l], w[l], keep, lo, hi)
        acc_ref = acc_ref + a_l
        acc_abs = acc_abs + kr.contact_stripes(attn[:, l], w[l].abs(), keep, lo, hi)[0]
        assert not bool(row.isnan().any()) and not bool(col.isnan().any()), f"layer {l}: unwritten sums"
        # sums of probabilities (all >= 0): S terms per row, 16 per stripe column
        for name, got, ref, n in (("row", row, row_ref, S), ("col", col, col_ref, 16)):
            err = (got.double() - ref).abs()
            bound = kr.sum_bound(ref, max(n, 2)) + 1e-30
            worst[name] = max(worst[name], float((err / bound).max()))
        rows.append(row); cols.append(col); rows64.append(row_ref); cols64.append(col_ref)
    # one fma per head in each launch, then one add into the running sum per launch
    err = (acc.double() - acc_ref).abs()
    acc_ratio = float((err / ((L * H + L) * U * acc_abs + 1e-30)).max())
    assert float(cols64[0][0, :, -1].sum()) > 0  # the last, partial stripe holds weight
    # both kernels together: a1 and u as ContactPredictionHead prepares them, contacts against float64
    c_abs = 0.0
    if S >= 15:
        a1 = torch.stack([r + c.sum(2) for r, c in zip(rows, cols)], 1).view(B, L * H, S)
        u = (a1 * (w.reshape(1, L * H, 1) / a1.sum(-1, keepdim=True))).contiguous()
        bias = torch.tensor([-0.3], device="cuda")
        got = finalize(acc, u, a1, bias)
        want = kr.contacts_from_partials(acc_ref, torch.stack([r[:, :, None] for r in rows64]), torch.stack(cols64), w,
                                         -0.3)
        assert not bool(got.isnan().any()) and not bool(want.isnan().any())
        c_abs = float((got.double() - want).abs().max())
    report(f"contact_accumulate S={S} H={H} T={T} crop={crop} keep={int(with_keep)}", row_err_over_bound=worst["row"],
           col_err_over_bound=worst["col"], acc_err_over_bound=acc_ratio, contacts_max_abs=c_abs)
    assert worst["row"] <= 1.0 and worst["col"] <= 1.0 and acc_ratio <= 1.0
    assert c_abs <= 1e-5  # O(1) logits evaluated in fp32, halved by the sigmoid


def test_accumulate_is_deterministic_and_checks_its_arguments():
    L_ = _lib(); lib = L_.load()
    B, L, H, T = 2, 1, 5, 200
    attn = make_maps(B, L, H, T, (0.5, 6.0), [T, 120], seed=1)
    w = torch.randn(L, H, generator=torch.Generator().manual_seed(2)).cuda()
    outs = []
    for _ in range(2):
        acc = torch.zeros(B, T - 2, T - 2, device="cuda")
        row, col = accumulate(attn, 0, w, None, acc, 1, T - 1)
        outs.append((acc, row, col))
    assert all(torch.equal(a, b) for a, b in zip(*outs))
    acc, row, col = outs[0]
    before = lib.esmb200_launch_count()

    def call(T=T, lo=1, hi=T - 1, B=B, H=H, attn_p=attn.data_ptr()):
        return lib.esmb200_contact_accumulate(attn_p, 0, P(w), None, P(acc), P(row), P(col), B, H, T, lo, hi, S_())

    assert call(T=1025, lo=0, hi=1025) == -1 and b"at most 1024 positions" in lib.esmb200_last_error()
    assert call(lo=-1) == -1 and call(hi=T + 1) == -1 and call(lo=5, hi=5) == -1 and call(B=0) == -1 and call(H=0) == -1
    assert call(attn_p=None) == -1
    assert lib.esmb200_launch_count() == before


@pytest.mark.parametrize("C,S,with_bias", [(1, 65, True), (15, 130, False), (16, 64, True), (17, 130, True),
                                           (660, 130, False), (660, 1024, True)])
def test_finalize_against_float64(C, S, with_bias):
    check_finalize(C, S, with_bias)


def check_finalize(C, S, with_bias, B=2):
    """esmb200_contact_finalize on random acc, u and a1 against float64, gated on the logit rebuilt from the output;
    returns the worst logit error over its bound"""
    g = torch.Generator().manual_seed(C + S)
    acc = torch.randn(B, S, S, generator=g) * 2
    acc[:, :8] *= 20   # logits out to |z| ~ 90 and beyond
    acc = acc.cuda()
    a1 = (torch.rand(B, C, S, generator=g) + 0.05).cuda()  # row sum + column sum of a map: positive
    w = (torch.randn(C, generator=g) * 40).cuda()
    u = (a1.double() * (w.double()[None, :, None] / a1.double().sum(-1, keepdim=True))).float().contiguous()
    bias = torch.tensor([0.7], device="cuda") if with_bias else None
    out = finalize(acc, u, a1, bias)
    assert torch.equal(out, finalize(acc, u, a1, bias))
    assert not bool(out.isnan().any()) and float(out.min()) >= 0.0 and float(out.max()) <= 1.0
    b64 = 0.7 if with_bias else 0.0
    corr = torch.einsum("bci,bcj->bij", u.double(), a1.double())
    z = acc.double() + acc.double().transpose(-1, -2) - corr + b64
    mag = acc.double().abs() + acc.double().abs().transpose(-1, -2) + abs(b64) + \
        torch.einsum("bci,bcj->bij", u.double().abs(), a1.double().abs())
    assert float(z.abs().max()) > 88 and float((z.abs() < 10).double().mean()) > 0.3
    assert bool((out[z > 30] == 1.0).all()) and bool((out[z < -104] == 0.0).all())
    # C fmas, the two adds of acc and the bias: (C + 3) u of the absolute sum; then exp(-z) (ex2.approx of a rounded
    # product: 2^-21 + 2^-22 |z| relative, which is the same absolute change of z), and 1 + e, the quotient and the
    # stored fp32 output (4 u of the output, magnified by 1 / (1 - out) on the way back through logit)
    mid = z.abs() < 10
    sig = torch.sigmoid(z)
    bound = (C + 3) * U * mag + 2.0 ** -21 + 2.0 ** -22 * z.abs() + 4 * U / (1 - sig)
    zgot = torch.logit(out.double())
    r = float(((zgot - z).abs()[mid] / bound[mid]).max())
    asym = float((zgot - zgot.transpose(-1, -2)).abs()[mid & mid.transpose(-1, -2)].max())
    report(f"contact_finalize C={C} S={S} bias={int(with_bias)}", logit_err_over_bound=r, logit_asymmetry=asym,
           probs_max_abs=float((out.double() - sig).abs().max()), z_absmax=float(z.abs().max()))
    assert r <= 1.0
    assert bool(((zgot - zgot.transpose(-1, -2)).abs() <= bound + bound.transpose(-1, -2))[mid & mid.transpose(-1, -2)].all())
    return r
