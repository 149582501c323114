"""GPU (-m gpu): the kernels whose work grows with the sequence length, past the 1024 tokens where the other
kernel-level files stop, against the same float64 references and bounds.  ESM-2 has no length limit, and
predict_contacts exists so that long proteins fit; above 1024 tokens the key blocks per row (the running-maximum
rescale chain, P V and the row sum), the key-mask words, the persistent work-item walk, the fused contact partials'
quarters, the finalize tile grid, the probability grids and the rope table rows all run past anything shorter
sequences reach.

  * fp16 attention, both head widths (attention_wg_kernel at D = 64, the two-slot attention_fwd_kernel<false, 2> at
    D = 128), T from 1025 to 16384 (up to 128 key blocks per row), diffuse and sharp logits, one sequence padded at
    about half its length (the last live key block partial, every later one dead): test_gpu_attention_f16.check16 with
    the reference sliced by query rows; probabilities, row sums and saved statistics wherever the fp32 [B,H,T,T] output
    stays near 1 GB; the 15B head shape (40 heads of 128) at T = 4096; a maximum rising every 64 keys across all 64
    blocks; the neighbour-leak case at T = 4097;
  * fp32x3 attention (test_gpu_attention_split.check) at T = 1025, 2049 and 4096 with probabilities and statistics;
  * the fused and the store-free contact passes at T = 2049 and 4097, both head widths (acc, row and column partials
    against kernel_refs.contact_partials: test_gpu_contact_fused.check_partials);
  * esmb200_contact_finalize at S = 2047 and 4094 with the 15B shape's 48 x 40 channels and with 20;
  * the QKV RoPE epilogue with the models' own tables at T = 4097 and 16384 (fp16 and split GEMM), and the two-slot
    rotation of 128-wide heads through one layer at T = 2049;
  * one layer at T = 4096 against layer64 (fp16 at d = 64 and 128, fp32x3 at d = 64), and predict_contacts of a
    2-layer model at T = 4097 against the float64 contact head on the library's own attention maps.

Every case prints a PARITY line; DESIGN.md section 4 records the measured ratios."""
import pytest
import torch

import kernel_refs as kr
import test_gpu_attention_f16 as f16
import test_gpu_attention_split as split
import test_gpu_contact_fused as fused
import test_gpu_contact_standalone as standalone
import test_gpu_contacts_only as conly
import test_gpu_gemm_shapes as gemm
import test_gpu_gemm_split as gemm_split
import test_gpu_layer_head_widths as widths
from test_gpu_layer_split import LAYER_DELTA_RELFRO, LAYER_PROBS_MAX_ABS

pytestmark = pytest.mark.gpu

PROBS_BYTES = 1.1e9  # largest fp32 [B,H,T,T] probability output a case writes, but for the 15B head shape


def half_length(T):
    """a length near T / 2 that is not a multiple of 64: the sequence's last live key block is partial"""
    return T // 2 - 37


# ---- fp16 attention -------------------------------------------------------------------------------------------------
LONG_T = [1025, 1151, 1152, 1153, 2047, 2048, 2049, 4095, 4096, 4097, 8193, 16384]


@pytest.mark.parametrize("std", [1.0, 8.0], ids=["diffuse", "sharp"])
@pytest.mark.parametrize("T", LONG_T)
@pytest.mark.parametrize("D", [64, 128])
def test_attention_f16_long(D, T, std):
    B, H = 2, 2
    lengths = [T, half_length(T)]
    probs = 4 * B * H * T * T <= PROBS_BYTES
    qkv = f16.make_qkv(B, T, H, D, 1000 * D + T + int(std), std)
    f16.check16(f"long lengths={lengths} std={std}", qkv, f16.pad_of(B, T, lengths), B, T, H, D, probs=probs)


def test_attention_f16_15b_head_shape():
    """40 heads of 128 at T = 4096, B = 1: 32 query tiles per head, 1280 work items"""
    B, T, H, D = 1, 4096, 40, 128
    qkv = f16.make_qkv(B, T, H, D, 15, 1.0)
    f16.check16("15B heads", qkv, f16.pad_of(B, T, [4000]), B, T, H, D)


@pytest.mark.parametrize("D", [64, 128])
def test_attention_f16_maximum_rises_every_64_keys(D):
    """every one of the 64 64-key steps of T = 4096 raises each row's maximum by ~3.2: every block rescales O and l"""
    B, H, T = 2, 2, 4096
    f16.check16("long rising maximum per 64 keys", f16.rising_qkv(B, T, H, D, 6), None, B, T, H, D)


@pytest.mark.parametrize("masked", [False, True], ids=["no_mask", "mask"])
@pytest.mark.parametrize("D", [64, 128])
def test_attention_f16_neighbour_rows_do_not_leak(D, masked):
    """T = 4097: the last key box of each sequence holds one key of its own and reads 127 rows of the next sequence"""
    f16.check_neighbour_isolation(D, 4097, masked)


# ---- fp32x3 attention -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("std", [2.0, 8.0], ids=["std2", "sharp"])
@pytest.mark.parametrize("T", [1025, 2049, 4096])
def test_attention_split_long(T, std):
    B = 2
    H = 2 if T < 4096 else 1
    lengths = [T, half_length(T)]
    x = split.make_qkv(B, T, H, 100 + T, std)
    split.check(f"long lengths={lengths} std={std}", x, split.pad_of(B, T, lengths), B, T, H, lengths)


# ---- contact passes -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [2049, 4097])
@pytest.mark.parametrize("E", [128, 256], ids=["d64", "d128"])
def test_fused_and_store_free_contact_passes_long(E, T):
    """<cls> / <eos> crop and <eos> masking, the second sequence padded at about half its length; the store-free pass
    (esmb200_stack_contacts' pass) on its own weights against float64 on the storing pass's maps, and bit for bit
    against the storing pass"""
    L, H = 2, 2
    lengths = [T - 2, half_length(T)]
    model, tokens, probs, _ = fused.check_fused(L, E, H, T, lengths)
    lo, hi = 1, T - 1
    keep = tokens.ne(model.contact_head.eos_idx)
    (xa, a), (xb, b) = conly.storing_and_store_free(model, tokens, lo, hi, keep.to(torch.uint8).contiguous())
    out = fused.check_partials(probs, b, keep, lo, hi)
    fused.report(f"contact_store_free L{L}_E{E}_H{H}_T{T}", **out)
    for name in ("row", "col", "acc"):
        assert torch.equal(a[name], b[name]), name
    assert torch.equal(xa, xb)


@pytest.mark.parametrize("S", [2047, 4094])
@pytest.mark.parametrize("C", [1920, 20], ids=["15B_channels", "C20"])
def test_contact_finalize_long(C, S):
    """(S / 64)^2 tiles per sequence: 1024 and 4096 CTAs"""
    standalone.check_finalize(C, S, True, B=1)


# ---- QKV RoPE epilogue ----------------------------------------------------------------------------------------------
def model_tables(E, H, T):
    from esm_b200.model import rope_tables
    d = E // H
    return rope_tables((1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))).cuda(), T)


@pytest.mark.parametrize("E,H,T", [(128, 2, 4097), (128, 2, 16384), (320, 20, 4097)])
def test_qkv_rope_f16_long(E, H, T):
    """The QKV epilogue with the model's own [T, 32] tables on two sequences (M = 2T): rows >= T take the second
    sequence's positions from 0, and the angles of table column 0 reach T - 1 radians.  64-wide heads through
    esmb200_gemm_qkv_f16 (K = E); the 8M width's 16-wide heads in 64-wide slots (K = E < 64 H) through
    esmb200_gemm_f16, as test_qkv_rope_narrow_head_tables runs them"""
    L = gemm._lib(); lib = L.load()
    Ea = 64 * H
    cos, sin = model_tables(E, H, T)
    M = 2 * T
    a, w, bias = gemm.operands(M, 3 * Ea, E, seed=T + E)
    out = torch.full((M, 3 * Ea), float("nan"), dtype=torch.float16, device="cuda")
    if E == Ea:
        L.check(lib.esmb200_gemm_qkv_f16(a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), M, Ea, 0.125,
                                         cos.data_ptr(), sin.data_ptr(), T, gemm.S()))
    else:
        gemm.run_gemm(kr.EPI_QKV_ROPE, a, w, bias, out, M, 3 * Ea, E, cos, sin, T, Ea)
    y, absdot = gemm.qkv_ref(a, w, bias, 0.125, Ea, T, cos, sin)
    gemm.report(f"gemm qkv rope long E={E} H={H} T={T} M={M}", err_over_bound=gemm.check_qkv(out, y, absdot, E))


@pytest.mark.parametrize("T", [4097, 16384])
def test_qkv_rope_split_long(T):
    """esmb200_gemm_split(EPI_QKV_ROPE) with the model's own table, head_dim 64, two sequences"""
    E, H = 128, 2
    cos, sin = gemm_split.rope_operands(E, H, T, E // H)
    gemm_split.check_qkv_split(2 * T, 64 * H, E, E + T, 0.125, T, cos, sin, label=f"long d=64 T={T}")


def test_qkv_rope_two_slots_per_head_long():
    """the two-slot rotation (table columns 32 .. 63) of 128-wide heads through one layer at T = 2049"""
    gemm.check_two_slot_rope(2049, 2, label="(via one layer) T=2049")


# ---- end to end -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,precision", [(64, 0), (128, 0), (64, 1)])
def test_layer_long(d, precision):
    """one layer at T = 4096, the second sequence padded at about half its length, with the tolerances of the
    shorter layer tests (fp32x3 at d = 64: those of test_gpu_layer_split's 650M-width layer)"""
    gates = (LAYER_DELTA_RELFRO, LAYER_PROBS_MAX_ABS) if precision == 1 else None
    widths.check_layer(d, precision, 4096, [4096, half_length(4096)], gates)


@pytest.mark.parametrize("E,H", [(128, 2), (256, 2)], ids=["d64", "d128"])
def test_predict_contacts_long_against_float64_head(E, H):
    """predict_contacts (the store-free pass) of a 2-layer model at T = 4097 against the contact head evaluated in
    float64 on the library's own attention maps (forward with need_head_weights)"""
    from oracle.weights import make_tokens
    L, T = 2, 4097
    model = conly.esm2(L, E, H, seed=T + E).to(conly.DEV)
    tokens = make_tokens([T - 2, half_length(T)], T, seed=T, n_mask=2).to(conly.DEV)
    head = model.contact_head
    with torch.no_grad():
        got = model.predict_contacts(tokens)
        attn = model(tokens, need_head_weights=True)["attentions"]
        want = head._forward_torch(tokens, attn.double(), head.regression.weight.double().view(L, H), 1, T - 1)
    err = float((got.double() - want).abs().max())
    print(f"PARITY predict_contacts long E={E} H={H} T={T} contacts_max_abs={err:.3e}", flush=True)
    assert got.shape == want.shape and err <= 1e-5
