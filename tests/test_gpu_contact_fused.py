"""GPU (-m gpu): the fused probability + contact pass (csrc/attention_contact.cuh, attention_probs_contact_kernel<DS>)
that every fp16 `return_contacts=True` forward of ESM-2 / ESM-1b runs, checked at the kernel's own outputs:

  * the probabilities it writes are bit-identical to those of the separate probability kernel (the forward without
    contacts), which test_gpu_kernels.py ties to an fp32 softmax;
  * every row / column partial (one per 32-key or 32-query quarter of a 128-wide tile) and the accumulator
    sum_l sum_h w[l,h] A against float64 sums of the returned probabilities (kernel_refs.contact_partials);
  * the contacts of finish_job against the contact head evaluated in float64 on the returned maps, and against the
    non-fused accumulation kernel.

DS = 1 (head_dim 64 and 16) and DS = 2 (head_dim 128 and 96); T around the 128-wide tile edges and at 1024; ragged
batches with <eos> at different positions, padded query rows and a sequence shorter than 128 (its later key tiles take
the kernel's `live == false` branch). Two layers, so the accumulator is read-modified-written across launches."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

U = kr.U32


def build_model(L, E, H, seed):
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict
    model = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    model.load_state_dict(make_state_dict(L, E, H, seed=seed), strict=True)
    return model.eval().cuda()


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def fused_stack(model, tokens):
    """model._stack with contacts; the job's partial buffers start as NaN so that an unwritten entry fails."""
    head = model.contact_head
    begin = head.begin_job

    def begin_nan(*args, **kw):
        st = begin(*args, **kw)
        st["row"].fill_(float("nan"))
        st["col"].fill_(float("nan"))
        return st

    head.begin_job = begin_nan
    try:
        _, _, _, attn_t, cjob = model._stack(tokens, need_head_weights=True, return_contacts=True)
    finally:
        del head.begin_job
    return attn_t["stacked"], cjob


# (L, E, H, T, residue lengths): eos at position length + 1; the last sequence is padded
CASES = [
    (2, 128, 2, 40, [38, 20]),           # DS = 1, one tile
    (2, 320, 20, 127, [125, 60]),        # DS = 1, 16-wide heads in 64-wide slots (8M width)
    (2, 128, 2, 128, [126, 90]),         # one full tile
    (2, 128, 2, 129, [127, 100]),        # one column past the tile
    (2, 256, 2, 129, [127, 100]),        # DS = 2, head_dim 128 (15B head width)
    (2, 192, 2, 300, [298, 100, 40]),    # DS = 2, head_dim 96; later key tiles of two sequences are not live
    (2, 128, 2, 300, [298, 250, 20]),
    (2, 128, 2, 1024, [1022, 517]),
    (2, 256, 2, 1024, [1022, 90]),       # DS = 2 at T = 1024
]


def check_partials(probs, st, keep, lo, hi):
    """A contact job's row / column partials and accumulator against float64 sums of the maps probs [B,L,H,T,T]
    (kernel_refs.contact_partials with the job's own weights st["w"]); returns the worst error / bound ratios."""
    B, L, H, T, _ = probs.shape
    S = hi - lo
    nt = (T + 127) // 128
    assert st["row"].shape == st["col"].shape == (L, B, H, 4 * nt, S)
    acc_ref = torch.zeros(B, S, S, dtype=torch.float64, device="cuda")
    acc_abs = torch.zeros_like(acc_ref)
    worst = {"row": 0.0, "col": 0.0}
    w = st["w"]
    for l in range(L):
        acc_l, row, col = kr.contact_partials(probs[:, l], w[l], keep, lo, hi)
        acc_ref += acc_l
        acc_abs += kr.contact_partials(probs[:, l], w[l].abs(), keep, lo, hi)[0]
        for name, ref in (("row", row), ("col", col)):
            got = st[name][l].double()
            assert not bool(got.isnan().any()), f"layer {l}: unwritten {name} partial"
            # 32 fp32 additions of probabilities (the kernel's exact operands, all >= 0): |err| <= 31 u sum
            err = (got - ref).abs()
            bound = kr.sum_bound(ref, 32) + 1e-30
            worst[name] = max(worst[name], float((err / bound).max()))
            assert bool((err <= bound).all()), (l, name, float((err - bound).max()))
        del acc_l, row, col
    # acc: one fma per head in each layer's launch, then one add into the running sum per layer:
    # |err| <= (L * H + L) u sum_l sum_h |w| A
    err = (st["acc"].double() - acc_ref).abs()
    bound = (L * H + L) * U * acc_abs + 1e-30
    acc_ratio = float((err / bound).max())
    assert bool((err <= bound).all())
    return dict(row_err_over_bound=worst["row"], col_err_over_bound=worst["col"], acc_err_over_bound=acc_ratio)


def check_fused(L, E, H, T, lengths):
    """The fused pass of a 2-layer model on make_tokens(lengths, T) against float64 (check_partials), its
    probabilities against the separate probability kernel's bit for bit, and its contacts against the head in float64
    on the same maps (and, up to T = 1024, against the non-fused accumulation kernel).  Returns (model, tokens, probs,
    ratios)."""
    from oracle.weights import make_tokens
    model = build_model(L, E, H, seed=T + E)
    tokens = make_tokens(lengths, T, seed=T, n_mask=1).cuda()
    with torch.no_grad():
        probs, st = fused_stack(model, tokens)
        # the separate probability kernel (no contact job) must write the same bits
        _, _, _, attn_sep, _ = model._stack(tokens, need_head_weights=True, return_contacts=False)
    assert torch.equal(probs, attn_sep["stacked"])
    del attn_sep

    head = model.contact_head
    lo, hi = 1, T - 1
    keep = tokens.ne(head.eos_idx)
    out = check_partials(probs, st, keep, lo, hi)

    # contacts: finish_job (fp32 APC + finalize kernel) against the head in float64 on the same maps; the logits are
    # O(1) sums whose fp32 evaluation is good to ~1e-6, the sigmoid halves that
    with torch.no_grad():
        got = head.finish_job(st)
        want = head._forward_torch(tokens, probs.double(), st["w"].double(), lo, hi)
    out["contacts_max_abs"] = float((got.double() - want).abs().max())
    if T <= 1024:  # esmb200_contact_accumulate's limit
        with torch.no_grad():
            nonfused = head(tokens, probs)
        out["nonfused_contacts_max_abs"] = float((nonfused.double() - want).abs().max())
    report(f"contact_fused L{L}_E{E}_H{H}_T{T}", **out)
    assert out["contacts_max_abs"] <= 1e-5
    if T <= 1024:
        assert out["nonfused_contacts_max_abs"] <= 1e-5
        # and both paths' contacts against each other
        torch.testing.assert_close(got, nonfused, atol=1e-5, rtol=0)
    return model, tokens, probs, out


@pytest.mark.parametrize("L,E,H,T,lengths", CASES)
def test_fused_contact_pass_against_float64(L, E, H, T, lengths):
    check_fused(L, E, H, T, lengths)


def test_row_partials_are_per_quarter_not_only_per_row():
    """A partial-index mistake that keeps each row's total (e.g. quarters stored in reverse) must not pass: the
    per-row totals agree, each partial is still compared on its own above; here the partials of one row are shown to
    differ between quarters, so a permutation changes them."""
    from oracle.weights import make_tokens
    model = build_model(2, 128, 2, seed=3)
    tokens = make_tokens([298, 250], 300, seed=3).cuda()
    with torch.no_grad():
        _, st = fused_stack(model, tokens)
    row = st["row"][0, 0, 0]  # [4 nt, S] of layer 0, sequence 0, head 0
    assert float((row[0:4] - row[0:4].flip(0)).abs().max()) > 1e-3
    assert float((st["col"][0, 0, 0, 0:4] - st["col"][0, 0, 0, 0:4].flip(0)).abs().max()) > 1e-3
