"""GPU (-m gpu): the wgmma GEMM (csrc/gemm2.cuh) at every (epilogue, N, K) the models launch and at its tile edges,
against float64 on the kernel's own fp16 operands:

  * every launch of ESM-2 8M .. 15B, ESM-1b and the MSA Transformer (kernel_refs.gemm_launches), at an M that leaves a
    partial last 128-row tile;
  * M around the 64-row halves of a tile (the second MMA warpgroup's rows all past M), K not a multiple of 64 (the last
    K slab zero-filled by TMA), partial 256-column tiles, and tile counts just above a multiple of the SM count;
  * the QKV epilogue: q scale, narrow-head rope tables, and the two-slot (rope_ld = 64) rotation of 128-wide heads;
  * the erf-GELU of the fp32 and fp16 epilogues against float64 erf over [-12, 12], bounded by kernel_refs.gelu_bound.

Accumulation bound used throughout: the tensor core sums each k16 step's exact products into the fp32 accumulator with
truncation, so |err| <= (K/16 + 4) 2^-22 sum_k |a_k w_k| (one ulp per step, doubled for slack), plus the rounding of the
bias add and of the output."""
import math

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


def operands(M, N, K, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    w = (torch.randn(N, K, device="cuda", generator=g) * (scale * K ** -0.5)).half()
    bias = 0.1 * torch.randn(N, device="cuda", generator=g)
    return a, w, bias


exact, acc_bound, f16_bound, qkv_ref = kr.gemm_exact, kr.gemm_acc_bound, kr.f16_bound, kr.qkv_ref


def run_gemm(epi, a, w, bias, out, M, N, K, cos=None, sin=None, T=0, E=0):
    L = _lib(); lib = L.load()
    L.check(lib.esmb200_gemm_f16(epi, a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), M, N, K,
                                 cos.data_ptr() if cos is not None else None,
                                 sin.data_ptr() if sin is not None else None, T, E, S()))


def check_plain(epi, M, N, K, seed):
    """EPI_BIAS_F32 / EPI_BIAS_RESIDUAL / EPI_BIAS_GELU_F32 / EPI_BIAS_GELU at (M, N, K) against float64; returns the
    largest error over its bound."""
    a, w, bias = operands(M, N, K, seed)
    y, absdot = exact(a, w, bias)
    b = acc_bound(absdot, K, y)
    if epi in (kr.EPI_BIAS_F32, kr.EPI_BIAS_GELU_F32, kr.EPI_BIAS_GELU):
        f16 = epi == kr.EPI_BIAS_GELU
        out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.float16 if f16 else torch.float32)
        run_gemm(epi, a, w, bias, out, M, N, K)
        if epi == kr.EPI_BIAS_F32:
            want = y
        else:  # |gelu'| <= 1.13: the accumulation error passes through it
            want = kr.gelu64(y)
            b = 1.13 * b + kr.gelu_bound(y)
            if f16:
                b = b + f16_bound(want)
    else:
        x0 = torch.randn(M, N, device="cuda")
        out = x0.clone()
        run_gemm(epi, a, w, bias, out, M, N, K)
        want = x0.double() + y
        b = b + kr.U32 * want.abs()
    err = (out.double() - want).abs()
    assert not bool(err.isnan().any()), "output not written"
    ratio = float((err / b).max())
    assert ratio <= 1.0, (epi, M, N, K, ratio)
    return ratio


def check_qkv(out, y, absdot, K):
    b = kr.qkv_bound(y, absdot, K)
    err = (out.double() - y).abs()
    assert not bool(err.isnan().any())
    ratio = float((err / b).max())
    assert ratio <= 1.0, ratio
    return ratio


# ---- every launch of every model ------------------------------------------------------------------------------------
TABLE = [(name, role, epi, n, k) for name in kr.MODELS for role, epi, n, k in kr.gemm_launches(name)]


@pytest.mark.parametrize("name,role,epi,N,K", TABLE, ids=[f"{t[0]}-{t[1]}" for t in TABLE])
def test_every_model_launch(name, role, epi, N, K):
    M = 130 if "15B" in name else 200  # a partial last row tile (two rows / 72 rows of it)
    if epi == kr.EPI_QKV_ROPE:
        _, E, H, _, rotary, _ = kr.MODELS[name]
        Ea, d = N // 3, E // H
        a, w, bias = operands(M, N, K, seed=N + K)
        out = torch.full((M, N), float("nan"), dtype=torch.float16, device="cuda")
        if rotary and kr.head_slots(E, H) == 1:  # ESM-2 up to 3B: the model's own [T, 32] table, M = 2 sequences
            from esm_b200.model import rope_tables
            T = M // 2
            cos, sin = rope_tables((1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))).cuda(), T)
            run_gemm(epi, a, w, bias, out, M, N, K, cos, sin, T, Ea)
            y, absdot = qkv_ref(a, w, bias, 0.125, Ea, T, cos, sin)
        else:  # ESM-1b, the MSA layers and (table aside, see test_qkv_rope_two_slots_per_head) 15B: q scale only
            L = _lib(); lib = L.load()
            assert K == Ea
            L.check(lib.esmb200_gemm_qkv_f16(a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), M, Ea,
                                             d ** -0.5, None, None, 0, S()))
            y, absdot = qkv_ref(a, w, bias, d ** -0.5, Ea)
        ratio = check_qkv(out, y, absdot, K)
    else:
        ratio = check_plain(epi, M, N, K, seed=N + 7 * K)
    report(f"gemm {name} {role} M={M} N={N} K={K}", err_over_bound=ratio)


# ---- tile edges -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 129, 191, 193])
def test_rows_around_the_warpgroup_halves(M):
    """N = 480, K = 480 (35M): a partial 256-column tile and a partial last K slab as well."""
    r = check_plain(kr.EPI_BIAS_F32, M, 480, 480, seed=M)
    r2 = check_plain(kr.EPI_BIAS_RESIDUAL, M, 480, 480, seed=M + 1)
    report(f"gemm edge M={M} N=480 K=480", f32=r, residual=r2)


@pytest.mark.parametrize("K", [8, 24, 72, 480])
@pytest.mark.parametrize("N", [320, 1920])
def test_k_tails_and_partial_column_tiles(K, N):
    r = check_plain(kr.EPI_BIAS_F32, 129, N, K, seed=K + N)
    r2 = check_plain(kr.EPI_BIAS_GELU, 129, N, K, seed=K + N + 1)
    report(f"gemm edge M=129 N={N} K={K}", f32=r, gelu16=r2)


@pytest.mark.parametrize("extra", ["n_sms+1", "2n_sms-1"])
def test_tile_counts_just_above_the_sm_count(extra):
    """The persistent loop then gives CTAs unequal tile counts (one CTA two tiles, the others one)."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = n_sms + 1 if extra == "n_sms+1" else 2 * n_sms - 1
    r = check_plain(kr.EPI_BIAS_F32, 128 * tiles - 5, 256, 64, seed=tiles)           # one 256-column tile per row tile
    r2 = check_plain(kr.EPI_BIAS_RESIDUAL, 128 * tiles - 70, 192, 72, seed=tiles + 1)  # partial column tile, K tail
    report(f"gemm tiles={tiles} (n_sms={n_sms})", f32=r, residual=r2)


# ---- QKV epilogue ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E,H,T", [(320, 20, 37), (480, 20, 100), (128, 2, 129)])
def test_qkv_rope_narrow_head_tables(E, H, T):
    """The QKV epilogue with a model's own [T, 32] table (rope_tables: columns >= head_dim/2 are cos 1, sin 0) on the
    64-wide slots of 16-, 24- and 64-wide heads."""
    from esm_b200.model import rope_tables
    d = E // H
    Ea = 64 * H
    inv_freq = (1.0 / (10000 ** (torch.arange(0, d, 2).float() / d))).cuda()
    cos, sin = rope_tables(inv_freq, T)
    assert cos.shape == (T, 32)
    B = 3
    M = B * T
    a, w, bias = operands(M, 3 * Ea, E, seed=E + T)
    out = torch.full((M, 3 * Ea), float("nan"), dtype=torch.float16, device="cuda")
    run_gemm(kr.EPI_QKV_ROPE, a, w, bias, out, M, 3 * Ea, E, cos, sin, T, Ea)
    y, absdot = qkv_ref(a, w, bias, 0.125, Ea, T, cos, sin)
    report(f"gemm qkv rope E={E} H={H} T={T}", err_over_bound=check_qkv(out, y, absdot, E))


@pytest.mark.parametrize("q_scale", [0.125, 1.0 / math.sqrt(96) / math.sqrt(37)])
def test_qkv_without_tables_scales_q_only(q_scale):
    """esmb200_gemm_qkv_f16 without rope tables (ESM-1b, the MSA layers: q_scale = d^-1/2, divided by sqrt(R) for the
    tied row attention): q columns scaled after the bias, k and v untouched."""
    L = _lib(); lib = L.load()
    M, E = 300, 768
    a, w, bias = operands(M, 3 * E, E, seed=9)
    bias = bias * 10  # so that scaling the bias before or after the add differ
    out = torch.full((M, 3 * E), float("nan"), dtype=torch.float16, device="cuda")
    L.check(lib.esmb200_gemm_qkv_f16(a.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), M, E, q_scale,
                                     None, None, 0, S()))
    y, absdot = qkv_ref(a, w, bias, q_scale, E)
    report(f"gemm qkv no tables q_scale={q_scale:.4f}", err_over_bound=check_qkv(out, y, absdot, E))


def test_qkv_rope_two_slots_per_head():
    """head_dim 128 (15B): the QKV epilogue runs with rope_ld = 64 and rotates the odd 64-column group of every head
    with table columns [32, 64).  The standalone entry point has no rope_ld, so this runs one layer and compares its
    attention probabilities with float64 attention on q, k rebuilt from the layer's own fp16 LayerNorm output and
    weights; a wrong slot would rotate half of every head's dimensions by the wrong angles."""
    check_two_slot_rope(160, 2)


def check_two_slot_rope(T, B, label="(via one layer)"):
    """test_qkv_rope_two_slots_per_head at T positions and B sequences; returns the probabilities' max-abs error"""
    from esm_b200.model import TransformerLayer, rope_tables
    from oracle.weights import make_state_dict
    E, H = 256, 2
    d = E // H
    sd = make_state_dict(1, E, H, seed=4)
    layer = TransformerLayer(E, 4 * E, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items() if k.startswith("layers.0.")}, strict=True)
    layer = layer.cuda()
    x = torch.randn(T, B, E, generator=torch.Generator().manual_seed(4)).cuda()
    with torch.no_grad():
        _, attn = layer(x, need_head_weights=True)  # [H, B, T, T]
    a = layer.self_attn
    ln = layer.self_attn_layer_norm
    xn = torch.nn.functional.layer_norm(x.transpose(0, 1).double(), (E,), ln.weight.double(), ln.bias.double(), ln.eps)
    xn = xn.float().half().double()
    cos, sin = rope_tables(a.rot_emb.inv_freq, T)
    assert cos.shape == (T, 64)

    def proj(lin):
        return xn @ lin.weight.detach().half().double().t() + lin.bias.detach().double()  # [B,T,E]

    def rope(t):  # rotary_embedding.py:16-20 on [B,T,H,d] with the first d/2 table columns
        t = t.view(B, T, H, d)
        c, s = cos.double()[None, :, None, :d // 2], sin.double()[None, :, None, :d // 2]
        t1, t2 = t[..., :d // 2], t[..., d // 2:]
        return torch.cat((t1 * c - t2 * s, t2 * c + t1 * s), -1)

    q = rope(proj(a.q_proj) * d ** -0.5).half().double()
    k = rope(proj(a.k_proj)).half().double()
    p = torch.softmax(torch.einsum("bihd,bjhd->hbij", q, k), -1)
    # q, k are stored as fp16 (the reference rounds them too); what remains is the fp32 accumulation and a rounding
    # of q or k landing on the other side of an fp16 tie (|ds| <~ 2^-11 |q||k|, ~1e-3 here): max-abs 5e-3
    e = float((attn.double() - p).abs().max())
    report(f"gemm qkv rope two slots per head {label}", probs_max_abs=e)
    assert e <= 5e-3
    return e


# ---- GELU -----------------------------------------------------------------------------------------------------------
def test_gelu_epilogues_against_float64_erf():
    """Pre-activations over [-12, 12] and dense near 0.  The fp32 epilogue's GELU of the kernel's own pre-activation
    (the same GEMM with EPI_BIAS_F32: identical mainloop and bias add) is within kr.gelu_bound of float64 erf; the fp16
    epilogue stores exactly that fp32 value rounded to nearest."""
    L = _lib(); lib = L.load()
    M, N, K = 256, 2048, 64
    g = torch.Generator(device="cuda").manual_seed(1)
    a = (torch.randn(M, K, device="cuda", generator=g) *
         torch.logspace(-5, 0, M, device="cuda")[:, None]).half()   # rows from ~1e-5 to ~1 in size
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).half()
    bias = torch.cat([torch.linspace(-12, 12, N // 2, device="cuda"), torch.linspace(-0.02, 0.02, N // 2, device="cuda")])
    pre = torch.empty(M, N, device="cuda")
    run_gemm(kr.EPI_BIAS_F32, a, w, bias, pre, M, N, K)
    out = torch.full((M, N), float("nan"), device="cuda")
    run_gemm(kr.EPI_BIAS_GELU_F32, a, w, bias, out, M, N, K)
    out16 = torch.full((M, N), float("nan"), dtype=torch.float16, device="cuda")
    run_gemm(kr.EPI_BIAS_GELU, a, w, bias, out16, M, N, K)
    assert float(pre.min()) < -11.5 and float(pre.max()) > 11.5 and int((pre.abs() < 1e-3).sum()) > 1000
    err = (out.double() - kr.gelu64(pre)).abs()
    bound = kr.gelu_bound(pre)
    ratio = float((err / bound).max())
    report("gemm gelu_erf fp32 epilogue over [-12, 12]", max_abs=float(err.max()), err_over_bound=ratio)
    assert ratio <= 1.0
    assert torch.equal(out16, out.half())
