"""GPU (-m gpu): the fp32x3 GEMM (gemm2_f16_kernel<EPI, true>: operands [M, 2K] / [N, 2K] as fp16 hi | lo, three passes
hi*hi + lo*hi + hi*lo per 64-wide K slab, fp16 outputs written as hi | lo [M, 2N]) through esmb200_gemm_split and
esmb200_gemm_qkv_split, at every (epilogue, N, K) of the models that run fp32x3 and at the tile edges.

  * Pass isolation, bit-exact and independent of K: operands whose halves make only one of the three products
    nonzero.  The other two passes then add exact zeros and the real products arrive in the fp16 kernel's slab order, so
    the output equals esmb200_gemm_f16 / esmb200_gemm_qkv_f16 on the corresponding fp16 operands under torch.equal (the
    hi half of an fp16 output; its lo half is rn16(y - rn16(y)) of the fp16 kernel's fp32 value y).  A lo half read from
    the wrong columns, or a box stored at the wrong place, cannot pass this whatever the size of K.
  * float64 on hi + lo: element-wise within kr.split_acc_bound plus the epilogue's roundings, and every output box
    (64 rows x 64 fp16 or 32 fp32 columns: one TMA store) within BOX_C * kr.split_box_scale(K) in rel-Frobenius.
  * the QKV epilogue with the models' own rope tables and with q_scale only, and the refusals of bad shapes."""
import math

import pytest
import torch

import kernel_refs as kr
from test_gpu_gemm_shapes import qkv_ref

pytestmark = pytest.mark.gpu

# Per-box rel-Frobenius gate in units of (3K/16 + 4) 2^-25: measured at most 1.17 of it (DESIGN.md section 4).  A dropped
# or misplaced lo half costs ~2^-12 = 2.4e-4 relative; the gate is 7.2e-5 at K = 5120 and 1.4e-4 at K = 10240 (3B fc2).
BOX_C = 2.5


def _lib():
    from esm_b200 import _lib
    return _lib


def S():
    return torch.cuda.current_stream().cuda_stream


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def nan(shape, dtype):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def cat(hi, lo):
    return torch.cat((hi, lo), 1).contiguous()


def f16_gemm(epi, a, w, bias, out, M, N, K, cos=None, sin=None, T=0, E=0):
    L = _lib(); lib = L.load()
    L.check(lib.esmb200_gemm_f16(epi, a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K,
                                 cos.data_ptr() if cos is not None else None,
                                 sin.data_ptr() if sin is not None else None, T, E, S()))


def split_gemm(epi, a2, w2, bias, out, M, N, K, cos=None, sin=None, T=0, E=0):
    L = _lib(); lib = L.load()
    L.check(lib.esmb200_gemm_split(epi, a2.data_ptr(), w2.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K,
                                   cos.data_ptr() if cos is not None else None,
                                   sin.data_ptr() if sin is not None else None, T, E, S()))


def qkv_f16(a, w, bias, out, M, E, q_scale):
    L = _lib(); lib = L.load()
    L.check(lib.esmb200_gemm_qkv_f16(a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), M, E, q_scale,
                                     None, None, 0, S()))


def qkv_split(a2, w2, bias, out, M, E, q_scale):
    L = _lib(); lib = L.load()
    L.check(lib.esmb200_gemm_qkv_split(a2.data_ptr(), w2.data_ptr(), bias.data_ptr(), out.data_ptr(), M, E, q_scale,
                                       S()))


def data(M, N, K, seed):
    """fp32 activations ~N(0, 1), weights ~K^-1/2, bias ~0.1 (realistic scale), on the device"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) * K ** -0.5
    bias = 0.1 * torch.randn(N, device="cuda", generator=g)
    return a, w, bias


def lo_of(y32):
    """rn16(y - rn16(y)) of fp32 y: the lo half the split epilogue stores"""
    return (y32 - y32.half().float()).half()


def half_ulp(h):
    """half an fp16 ulp of fp16 h: 2^(e - 11) for |h| in [2^e, 2^(e+1)), 2^-25 below the normal range"""
    e = torch.floor(torch.log2(h.double().abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - 11)


def box_rel_fro(err, ref, bw):
    """max over the output boxes (64 rows x bw columns) of ||err|| / ||ref||, float64 [M, N]"""
    M, N = err.shape
    mp = (M + 63) // 64 * 64
    e = torch.nn.functional.pad(err, (0, 0, 0, mp - M)).view(mp // 64, 64, N // bw, bw)
    r = torch.nn.functional.pad(ref, (0, 0, 0, mp - M)).view(mp // 64, 64, N // bw, bw)
    return float((e.norm(dim=(1, 3)) / r.norm(dim=(1, 3)).clamp_min(1e-300)).max())


# ---- pass isolation -------------------------------------------------------------------------------------------------
PASSES = ("hi*hi", "lo*hi", "hi*lo")


def isolate(which, a16, w16):
    """[a_hi | a_lo], [w_hi | w_lo] with only the `which` product nonzero, equal to a16 . w16^T"""
    za, zw = torch.zeros_like(a16), torch.zeros_like(w16)
    if which == "hi*hi":
        return cat(a16, za), cat(w16, zw)
    if which == "lo*hi":
        return cat(za, a16), cat(w16, zw)
    return cat(a16, za), cat(zw, w16)


def isolation_plain(epi, M, N, K, seed):
    """EPI_BIAS_F32 / EPI_BIAS_GELU_F32 / EPI_BIAS_RESIDUAL / EPI_BIAS_GELU: each pass alone equals the fp16 kernel"""
    a, w, bias = data(M, N, K, seed)
    a16, w16 = a.half(), w.half()
    f16_out = epi == kr.EPI_BIAS_GELU
    x0 = torch.randn(M, N, device="cuda")
    if f16_out:
        want = nan((M, N), torch.float16)
        f16_gemm(epi, a16, w16, bias, want, M, N, K)
        y32 = nan((M, N), torch.float32)
        f16_gemm(kr.EPI_BIAS_GELU_F32, a16, w16, bias, y32, M, N, K)
        assert torch.equal(y32.half(), want)
        want_lo = lo_of(y32)
    elif epi == kr.EPI_BIAS_RESIDUAL:
        want = x0.clone()
        f16_gemm(epi, a16, w16, bias, want, M, N, K)
    else:
        want = nan((M, N), torch.float32)
        f16_gemm(epi, a16, w16, bias, want, M, N, K)
    for which in PASSES:
        a2, w2 = isolate(which, a16, w16)
        if f16_out:
            out = nan((M, 2 * N), torch.float16)
        elif epi == kr.EPI_BIAS_RESIDUAL:
            out = x0.clone()
        else:
            out = nan((M, N), torch.float32)
        split_gemm(epi, a2, w2, bias, out, M, N, K)
        if f16_out:
            assert torch.equal(out[:, :N], want), (which, "hi half")
            assert torch.equal(out[:, N:], want_lo), (which, "lo half")
        else:
            assert torch.equal(out, want), (which, float((out.double() - want.double()).abs().max()))


# ---- float64 on hi + lo ---------------------------------------------------------------------------------------------
def full_plain(epi, M, N, K, seed):
    """The split GEMM on split16 operands against float64 on hi + lo: (max error / element bound, max box rel-Fro /
    kr.split_box_scale(K))."""
    a, w, bias = data(M, N, K, seed + 1)
    ah, al = kr.split16(a)
    wh, wl = kr.split16(w)
    y = kr.join64(ah, al) @ kr.join64(wh, wl).t() + bias.double()
    b = kr.split_acc_bound(ah, al, wh, wl, K, y)
    f16_out = epi == kr.EPI_BIAS_GELU
    if epi == kr.EPI_BIAS_RESIDUAL:
        x0 = torch.randn(M, N, device="cuda")
        out = x0.clone()
    else:
        out = nan((M, 2 * N) if f16_out else (M, N), torch.float16 if f16_out else torch.float32)
    split_gemm(epi, cat(ah, al), cat(wh, wl), bias, out, M, N, K)
    if epi == kr.EPI_BIAS_RESIDUAL:  # x + y: one more fp32 rounding (the L2's reduce-add)
        want = x0.double() + y
        b = b + kr.U32 * want.abs()
    elif epi == kr.EPI_BIAS_F32:
        want = y
    else:  # |gelu'| <= 1.13 carries the accumulation error through; then the erf approximation's own bound
        want = kr.gelu64(y)
        b = 1.13 * b + kr.gelu_bound(y)
    if f16_out:
        got = kr.join64(out[:, :N], out[:, N:])
        b = b + kr.split_rep_bound(want)
    else:
        got = out.double()
    err = (got - want).abs()
    assert not bool(err.isnan().any()), "output not written"
    ratio = float((err / b).max())
    box = box_rel_fro(got - want, want, 64 if f16_out else 32) / kr.split_box_scale(K)
    assert ratio <= 1.0, (epi, M, N, K, ratio)
    assert box <= BOX_C, (epi, M, N, K, box)
    return ratio, box


def check_plain(epi, M, N, K, seed):
    isolation_plain(epi, M, N, K, seed)
    return full_plain(epi, M, N, K, seed)


# ---- QKV ------------------------------------------------------------------------------------------------------------
def rope_operands(E, H, T, d):
    from esm_b200.model import rope_tables
    inv_freq = (1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))).cuda()
    cos, sin = rope_tables(inv_freq, T)
    assert cos.shape == (T, 32)
    assert bool((cos[:, d // 2:] == 1).all()) and bool((sin[:, d // 2:] == 0).all())
    return cos, sin


def split_qkv_bound(ah, al, wh, wl, K, y_pre, E, q_scale, cos=None):
    """Element bound of the split QKV epilogue: kr.split_acc_bound of (a w^T + bias), times q_scale on the q columns
    (one more rounding: u), then for the rotation of pair (c, c + 32) by (cos, sin) the sum of both members' bounds
    (|cos|, |sin| <= 1) plus the rotation's two products and one add (4 u (|x1| + |x2|)).  y_pre: the unrotated
    (a w^T + bias) * scale in float64."""
    b = kr.split_acc_bound(ah, al, wh, wl, K, y_pre)
    b[:, :E] *= q_scale
    b = b + kr.U32 * y_pre.abs()
    if cos is not None:
        b = b.clone()
        for g0 in range(0, 2 * E, 64):
            b1, b2 = b[:, g0:g0 + 32].clone(), b[:, g0 + 32:g0 + 64].clone()
            x = y_pre[:, g0:g0 + 32].abs() + y_pre[:, g0 + 32:g0 + 64].abs()
            b[:, g0:g0 + 32] = b[:, g0 + 32:g0 + 64] = b1 + b2 + 4 * kr.U32 * x
    return b


def check_qkv_split(M, E, K, seed, q_scale, T=None, cos=None, sin=None, bias_gain=1.0, label=""):
    """Pass isolation and float64 for the QKV epilogue: with tables through esmb200_gemm_split (q_scale 0.125), without
    through esmb200_gemm_qkv_split."""
    N = 3 * E
    a, w, bias = data(M, N, K, seed)
    bias = bias * bias_gain
    a16, w16 = a.half(), w.half()
    rope = cos is not None
    want = nan((M, N), torch.float16)
    if rope:
        f16_gemm(kr.EPI_QKV_ROPE, a16, w16, bias, want, M, N, K, cos, sin, T, E)
    else:
        qkv_f16(a16, w16, bias, want, M, E, q_scale)
        y32 = nan((M, N), torch.float32)
        f16_gemm(kr.EPI_BIAS_F32, a16, w16, bias, y32, M, N, K)
        y32[:, :E] *= q_scale
        assert torch.equal(y32.half(), want)
    for which in PASSES:
        a2, w2 = isolate(which, a16, w16)
        out = nan((M, 2 * N), torch.float16)
        if rope:
            split_gemm(kr.EPI_QKV_ROPE, a2, w2, bias, out, M, N, K, cos, sin, T, E)
        else:
            qkv_split(a2, w2, bias, out, M, E, q_scale)
        assert torch.equal(out[:, :N], want), (which, "hi half")
        if rope:  # the rotated value is not reproducible on the host bit for bit: its lo half is a rounding residue
            assert bool((out[:, N:].double().abs() <= half_ulp(out[:, :N])).all()), (which, "lo half")
        else:
            assert torch.equal(out[:, N:], lo_of(y32)), (which, "lo half")
    # float64 on hi + lo
    a, w, _ = data(M, N, K, seed + 1)
    ah, al = kr.split16(a)
    wh, wl = kr.split16(w)
    aj, wj = kr.join64(ah, al), kr.join64(wh, wl)
    y_pre = aj @ wj.t() + bias.double()
    y_pre[:, :E] *= q_scale
    y, _ = qkv_ref(aj, wj, bias, q_scale, E, T, cos, sin)
    b = split_qkv_bound(ah, al, wh, wl, K, y_pre, E, q_scale, cos) + kr.split_rep_bound(y)
    out = nan((M, 2 * N), torch.float16)
    if rope:
        split_gemm(kr.EPI_QKV_ROPE, cat(ah, al), cat(wh, wl), bias, out, M, N, K, cos, sin, T, E)
    else:
        qkv_split(cat(ah, al), cat(wh, wl), bias, out, M, E, q_scale)
    got = kr.join64(out[:, :N], out[:, N:])
    err = (got - y).abs()
    assert not bool(err.isnan().any()), "output not written"
    ratio = float((err / b).max())
    box = box_rel_fro(got - y, y, 64) / kr.split_box_scale(K)
    report(f"gemm_split qkv {label} M={M} E={E} K={K} q_scale={q_scale:.4f} rope={rope}", err_over_bound=ratio,
           box_over_scale=box)
    assert ratio <= 1.0 and box <= BOX_C, (ratio, box)


# ---- every launch of every fp32x3 model -----------------------------------------------------------------------------
TABLE = [(name, role, epi, n, k) for name in kr.FP32X3_MODELS for role, epi, n, k in kr.gemm_launches(name)]


@pytest.mark.parametrize("name,role,epi,N,K", TABLE, ids=[f"{t[0]}-{t[1]}" for t in TABLE])
def test_every_fp32x3_model_launch(name, role, epi, N, K):
    M = 200  # a partial last 128-row tile (72 rows of it: the second warpgroup's half partly past M)
    if epi == kr.EPI_QKV_ROPE:
        _, E, H, _, rotary, _ = kr.MODELS[name]
        Ea, d = N // 3, E // H
        assert kr.head_slots(E, H) == 1
        if rotary:  # ESM-2: the model's own [T, 32] table, two sequences of T = 100
            cos, sin = rope_operands(E, H, M // 2, d)
            check_qkv_split(M, Ea, K, N + K, 0.125, M // 2, cos, sin, label=f"{name} {role}")
        else:       # ESM-1b and the MSA layers: q scale only
            check_qkv_split(M, Ea, K, N + K, d ** -0.5, label=f"{name} {role}")
        return
    ratio, box = check_plain(epi, M, N, K, seed=N + 7 * K)
    report(f"gemm_split {name} {role} M={M} N={N} K={K}", err_over_bound=ratio, box_over_scale=box,
           box_rel_fro=box * kr.split_box_scale(K))


# ---- tile edges -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 129, 191, 193])
def test_rows_around_the_warpgroup_halves(M):
    """N = 320 (a partial 256-column tile), K = 128"""
    r = check_plain(kr.EPI_BIAS_F32, M, 320, 128, seed=M)
    r2 = check_plain(kr.EPI_BIAS_GELU, M, 320, 128, seed=M + 1)
    report(f"gemm_split edge M={M} N=320 K=128", f32=r[0], f32_box=r[1], gelu16=r2[0], gelu16_box=r2[1])


@pytest.mark.parametrize("K", [64, 128, 640])
@pytest.mark.parametrize("N", [320, 640, 1920])
def test_k_slabs_and_partial_column_tiles(K, N):
    """K = 64 is 3 split slabs, fewer than the 4 ring stages"""
    r = check_plain(kr.EPI_BIAS_RESIDUAL, 129, N, K, seed=K + N)
    r2 = check_plain(kr.EPI_BIAS_GELU, 129, N, K, seed=K + N + 1)
    report(f"gemm_split edge M=129 N={N} K={K}", residual=r[0], residual_box=r[1], gelu16=r2[0], gelu16_box=r2[1])


@pytest.mark.parametrize("extra", ["n_sms+1", "2n_sms-1", "3n_sms+5"])
def test_persistent_tile_walk(extra):
    """Tile counts just above the SM count, and >= 3 tiles per CTA: the producer then runs ahead across tile
    boundaries, and each warpgroup's staging-buffer parity flips twice per fp16 box over many boxes."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    if extra == "3n_sms+5":
        tiles_m = (3 * n_sms + 5 + 1) // 2 + 1
        r = check_plain(kr.EPI_BIAS_GELU, 128 * tiles_m - 70, 512, 128, seed=7)    # two column tiles per row tile
        r2 = check_plain(kr.EPI_BIAS_F32, 128 * tiles_m - 3, 320, 64, seed=8)     # one whole, one partial
        tiles = 2 * tiles_m
        assert tiles >= 3 * n_sms + 5
    else:
        tiles = n_sms + 1 if extra == "n_sms+1" else 2 * n_sms - 1
        r = check_plain(kr.EPI_BIAS_GELU, 128 * tiles - 5, 256, 64, seed=tiles)
        r2 = check_plain(kr.EPI_BIAS_RESIDUAL, 128 * tiles - 70, 192, 128, seed=tiles + 1)
    report(f"gemm_split tiles={tiles} (n_sms={n_sms})", gelu16=r[0], gelu16_box=r[1], other=r2[0], other_box=r2[1])


# ---- QKV epilogue ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,H", [(320, 20), (640, 20), (1280, 20)])
@pytest.mark.parametrize("T", [37, 129])
def test_qkv_rope_tables_split(E, H, T):
    """esmb200_gemm_split(EPI_QKV_ROPE) with the model's own table for head_dim 16, 32 and 64, two sequences"""
    d = E // H
    cos, sin = rope_operands(E, H, T, d)
    check_qkv_split(2 * T, 64 * H, E, E + T, 0.125, T, cos, sin, label=f"d={d} T={T}")


def test_qkv_split_without_tables_scales_q_only():
    """esmb200_gemm_qkv_split with the tied row attention's scale d^-1/2 R^-1/2 and a bias x10, so that scaling before
    or after the bias add differ"""
    check_qkv_split(300, 768, 768, 9, 1.0 / math.sqrt(64) / math.sqrt(37), bias_gain=10.0, label="no tables")


# ---- refusals -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("epi,N,K", [(kr.EPI_BIAS_F32, 64, 96), (kr.EPI_BIAS_GELU, 64, 80),
                                     (kr.EPI_BIAS_GELU, 96, 64), (kr.EPI_QKV_ROPE, 96, 64)])
def test_bad_shapes_are_refused(epi, N, K):
    """K % 64 != 0, or an fp16 output with N % 64 != 0: ESMB200_EINVAL with its message, nothing written"""
    L = _lib(); lib = L.load()
    M = 70
    a2 = torch.zeros(M, 2 * K, dtype=torch.float16, device="cuda")
    w2 = torch.zeros(N, 2 * K, dtype=torch.float16, device="cuda")
    bias = torch.zeros(N, device="cuda")
    f16_out = epi in (kr.EPI_BIAS_GELU, kr.EPI_QKV_ROPE)
    out = nan((M, 2 * N) if f16_out else (M, N), torch.float16 if f16_out else torch.float32)
    cos = sin = torch.ones(M, 32, device="cuda")
    rc = lib.esmb200_gemm_split(epi, a2.data_ptr(), w2.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K,
                                cos.data_ptr(), sin.data_ptr(), M, N // 3, S())
    torch.cuda.synchronize()
    assert rc == -1
    assert b"split gemm needs K % 64 == 0" in lib.esmb200_last_error()
    assert bool(out.isnan().all())
    if epi == kr.EPI_QKV_ROPE:
        rc = lib.esmb200_gemm_qkv_split(a2.data_ptr(), w2.data_ptr(), bias.data_ptr(), out.data_ptr(), M, 32, 1.0, S())
        torch.cuda.synchronize()
        assert rc == -1 and b"E % 64 == 0" in lib.esmb200_last_error()
        assert bool(out.isnan().all())
