"""Torch statements of the fp8 precision's quantisation (esmb200.h, esmb200_quantize_fp8), shared by the CPU and GPU tests.

A block's scale is the smallest power of two s with amax / s <= 448 (e4m3's largest finite value), at least 2^-126, and 1
for an all-zero block.  Dividing by a power of two is exact, so q = (x / s).to(torch.float8_e4m3fn) and q * s are the
kernel's bits exactly.
"""
import ctypes
import math

import torch

E4M3_MAX = 448.0


def block_scale(amax: float) -> float:
    if amax == 0.0:
        return 1.0
    m, e = math.frexp(amax)  # amax = m 2^e, m in [0.5, 1): the IEEE significand is 2m, exponent e - 1
    s = 2.0 ** (e - 1 - 8) if 2 * m <= 1.75 else 2.0 ** (e - 1 - 7)
    return max(s, 2.0 ** -126)


def scales_of(amax: torch.Tensor) -> torch.Tensor:
    """block_scale over a float32 tensor of block maxima (vectorised with the same exponent rule)."""
    a = amax.double()
    m, e = torch.frexp(a)
    s = torch.where(2 * m <= 1.75, torch.ldexp(torch.ones_like(a), e - 9), torch.ldexp(torch.ones_like(a), e - 8))
    s = torch.clamp(s, min=2.0 ** -126)
    return torch.where(a == 0, torch.ones_like(a), s).float()


def quantize(x: torch.Tensor, block_rows: int):
    """fp32 [rows, K] -> (e4m3 [rows, K], scales) with one scale per block_rows x 128 block: block_rows 1 gives scales
    [ceil(K/128), rows], block_rows 128 gives [ceil(rows/128), ceil(K/128)] (esmb200_quantize_fp8's layouts)."""
    x = x.float()
    R, K = x.shape
    kb, rb = -(-K // 128), -(-R // block_rows)
    pad = torch.zeros(rb * block_rows, kb * 128, dtype=torch.float32, device=x.device)
    pad[:R, :K] = x.abs()
    amax = pad.view(rb, block_rows, kb, 128).amax(dim=(1, 3))  # [rb, kb]
    s = scales_of(amax)
    s_full = s.repeat_interleave(block_rows, 0).repeat_interleave(128, 1)[:R, :K]
    q = (x / s_full).to(torch.float8_e4m3fn)
    return q, (s.t().contiguous() if block_rows == 1 else s.contiguous())


def dequantize(q: torch.Tensor, s: torch.Tensor, block_rows: int) -> torch.Tensor:
    R, K = q.shape
    sf = s.t() if block_rows == 1 else s
    return q.double() * sf.double().repeat_interleave(block_rows, 0).repeat_interleave(128, 1)[:R, :K]


# ---- float64 emulation of one fp8 layer ------------------------------------------------------------------------------
# The emulation performs the same quantisation steps as the library (LayerNorm -> 1 x 128 e4m3, [Wq;Wk;Wv] in head
# slots -> 128 x 128 e4m3, fc1 and fc2 -> 128 x 128 e4m3, GELU -> 1 x 128 e4m3; q, k, v, ctx and out_proj's weights as
# fp16) with exact arithmetic in between.  The library differs from it by its accumulation and rounding errors, and by
# the e4m3 codes those errors flip at rounding boundaries.  Propagated as worst-case element-wise bounds these grow
# without use through softmax and the flips; instead `inject` places an error of the full bound's size, with random
# signs, at every point where the library rounds or accumulates, and the quantisation steps that follow flip codes
# exactly as the library's own errors would.  The spread of such perturbed emulations around the exact one is the
# tolerance for the library's layer (tests/test_gpu_fp8.py).

def requantize(v):
    """1 x 128 e4m3 quantisation of float64 [R, K] v (rounded to fp32 first, as the library's values are): the
    dequantised float64 result."""
    q, s = quantize(v.float().cpu(), 1)
    return dequantize(q, s, 1).to(v.device)


def head_slot(n, d):
    """elementwise.cuh head_slot: projection output index n = h d + j -> column of the attention-side tensors."""
    h, j, half = n // d, n % d, d // 2
    pr = torch.where(j < half, j, j - half)
    slots = 2 if d > 64 else 1
    return (h * slots + pr // 32) * 64 + pr % 32 + torch.where(j < half, 0, 32)


def quantized_qkv(Wq, Wk, Wv, d):
    """[Wq;Wk;Wv] placed in their head slots as fp32, quantised in 128 x 128 blocks and read back in the reference's
    row order: three dequantised float64 [E, E]."""
    E = Wq.shape[0]
    Ea = 64 * (2 if d > 64 else 1) * (E // d)
    rows = head_slot(torch.arange(E), d)
    packed = torch.zeros(3 * Ea, E, dtype=torch.float32)
    for i, W in enumerate((Wq, Wk, Wv)):
        packed[i * Ea + rows] = W.float().cpu()
    q, s = quantize(packed, 128)
    deq = dequantize(q, s, 128).to(Wq.device)
    return [deq[i * Ea + rows.to(Wq.device)] for i in range(3)]


def weight8(W):
    q, s = quantize(W.float().cpu(), 128)
    return dequantize(q, s, 128).to(W.device)


def acc_bound(A, W, per_block=2.0 ** -11):
    """|kernel accumulator - A.W^T| per element.  Each 128-wide K block is 4 chained wgmma k32 steps on the fp8 tensor
    cores, whose internal sum keeps only about 14 significand bits (DeepSeek-V3 section 3.3.2): the block's error is
    taken as at most per_block = 2^-11 of its sum of |products|.  Measured on an H100 it reaches 1.36 2^-12 where one K
    block dominates an output (row and weight-block scales 2^6 .. 2^16 apart, fp8_refs.spread_operands), so that the
    blocks' errors cannot average out; over Gaussian operands, whose blocks contribute comparably, the errors stay
    within 0.61 of per_block = 2^-12, which check_gemm keeps for them.  The promotion
    acc += tmp * (sa sb) into the fp32 accumulator adds 2^-24 of the running sum per block.  Together:
    (per_block + 2^-24 K/128) |A|.|W|^T.  The scales are powers of two and multiply exactly, so the bound holds per
    element whatever the blocks' scales are, as long as every sa sb and every promoted product stays a normal float.
    emulate_layer injects the typical error, per_block = 2^-12."""
    K = A.shape[-1]
    return (A.abs() @ W.abs().t()) * (per_block + 2.0 ** -24 * math.ceil(K / 128))


# ---- checkers of e4m3 outputs against a float64 reference ------------------------------------------------------------
def check_codes(q8, s, y, ybnd, device="cpu"):
    """An e4m3 output q8 [R, N] with its scales s [ceil(N/128), R] (one per row and 128 columns) against the float64
    values y [R, N] it quantises, where the kernel computed each value within ybnd [R, N] of y.  Returns a dict:
      bad_scale  scales that differ from the reference's by other than one power of two, or whose block's float64 amax
                 lies farther than the bound (plus the fp32 rounding of the amax) from the edge 448 min(s, s') between
                 the two scales;
      bad_code   codes whose dequantised value lies farther from y than half an e4m3 ulp (2^-4 relative, 2^-10 s for
                 subnormals) plus the bound: a code under the same scale may only differ from the reference's where y / s
                 lies within the bound of a rounding midpoint, and every code, also under a flipped scale, must still
                 round a value within the bound of y;
      flips      code mismatches under an equal scale (all of them boundary flips when bad_code is 0);
      scale_flips, n.
    On the CPU, or on `device`."""
    q8, s, y, ybnd = q8.to(device), s.to(device).float(), y.to(device).double(), ybnd.to(device).double()
    R, N = y.shape
    kb = -(-N // 128)
    qr, sr = quantize(y.float(), 1)
    sflip = s != sr
    full = lambda t: t.t().repeat_interleave(128, 1)[:, :N]  # noqa: E731  [kb, R] -> [R, N]
    deq = dequantize(q8, s, 1)
    sfull = full(s).double()
    sflip_full = full(sflip.to(torch.uint8)).bool()
    half_ulp = torch.maximum(deq.abs() * 2.0 ** -4, sfull * 2.0 ** -10)
    bad_code = (y - deq).abs() > half_ulp * (1 + 1e-6) + ybnd
    mism = q8.view(torch.uint8) != qr.view(torch.uint8)
    flips = mism & ~sflip_full
    pad = torch.zeros(R, kb * 128, dtype=torch.float64, device=y.device)
    pad[:, :N] = y.abs()
    am = pad.view(R, kb, 128).amax(-1).t()
    pad[:, :N] = ybnd
    bmax = pad.view(R, kb, 128).amax(-1).t()
    ratio = (sr.double() / s.double()).log2().abs()
    edge = 448 * torch.minimum(sr, s).double()
    near = (am - edge).abs() <= bmax + 2.0 ** -23 * am
    bad_scale = sflip & ~((ratio == 1) & near)
    return {"bad_scale": int(bad_scale.sum()), "bad_code": int(bad_code.sum()), "flips": int(flips.sum()),
            "scale_flips": int(sflip.sum()), "n": R * N}


# ---- scale-spread GEMM operands --------------------------------------------------------------------------------------
def spread_operands(M, N, K, seed, out_limit=None):
    """fp32 A [M, K] and W [N, K] whose block scales cover many octaves, so that a scale read from the wrong row, K block
    or weight block moves the result by powers of two:
      * every row of A times 2^U{-12..12}, every (row, 128-wide K block) of A a further 2^U{-6..6}, every 128 x 128 block
        of W 2^U{-16..16} (on top of randn and randn K^-1/2);
      * one all-zero row of A, one all-zero (row, K block) of A and, where W has enough blocks to keep every output
        column live (see below), one all-zero weight block (scale 1 each);
      * one A block whose amax is exactly 448 2^k (a scale edge: 448 / s = 448 exactly).
    out_limit: rows of A are then further scaled by powers of two (which leaves every code and the spread inside a row
    unchanged) until max_n sum_k |A W| <= out_limit (the fp16 QKV output: |y| < 2^15).  Even so every sa sb stays
    >= 2^-100 (tests/test_fp8_host.py), so a product of e4m3 codes (>= 2^-18) times sa sb is a normal float; the
    largest outputs without out_limit are about 2^40, far inside fp32 and e4m3-with-scale range."""
    g = torch.Generator().manual_seed(seed)
    kb, nb = -(-K // 128), -(-N // 128)
    a = torch.randn(M, K, generator=g, dtype=torch.float64)
    a *= torch.ldexp(torch.ones(M, 1, dtype=torch.float64), torch.randint(-12, 13, (M, 1), generator=g))
    blk = torch.ldexp(torch.ones(M, kb, dtype=torch.float64), torch.randint(-6, 7, (M, kb), generator=g))
    a *= blk.repeat_interleave(128, 1)[:, :K]
    w = torch.randn(N, K, generator=g, dtype=torch.float64) * K ** -0.5
    wb = torch.ldexp(torch.ones(nb, kb, dtype=torch.float64), torch.randint(-16, 17, (nb, kb), generator=g))
    w *= wb.repeat_interleave(128, 0).repeat_interleave(128, 1)[:N, :K]
    a[M // 3] = 0.0
    if M > 1:
        a[M // 2, (kb - 1) * 128:] = 0.0
    # the all-zero weight block (last row block, first K block) only where every output column keeps a live K block
    # with at least 128 columns of W: several K blocks, and a full one besides the first, or another row block
    if kb > 1 and (kb > 2 or nb > 1):
        w[(nb - 1) * 128:, :128] = 0.0
    r, c0 = (2 * M) // 3, 0
    am = float(a[r, c0:c0 + 128].abs().max())
    e = math.frexp(am / 448.0)[1] + 1 if am > 0 else 0
    a[r, c0 + 5] = -448.0 * 2.0 ** e  # exactly 448 2^e, above the block's other values
    if out_limit is not None:
        top = (a.abs() @ w.abs().t()).amax(1)
        shift = torch.clamp(torch.ceil(torch.log2(top / out_limit)), min=0).nan_to_num(0.0)
        a = torch.ldexp(a, -shift.long()[:, None])
    return a.float(), w.float()


# ---- guard bands ----------------------------------------------------------------------------------------------------
GUARD = 4096
SENTINEL = 0xA5


def guarded(shape, dtype, device, guard=GUARD, fill=0xFF):
    """A tensor of `shape` / `dtype` inside one byte buffer with `guard` sentinel bytes before and after it.  The tensor's
    bytes are `fill` (0xFF: NaN in fp32, fp16 and float8_e4m3fn).  Returns (tensor, buffer); guard_changes(buffer)
    counts the sentinel bytes that changed."""
    n = math.prod(shape) * torch.tensor([], dtype=dtype).element_size()
    buf = torch.full((2 * guard + n,), SENTINEL, dtype=torch.uint8, device=device)
    buf[guard:guard + n] = fill
    return buf[guard:guard + n].view(dtype).view(shape), buf


def guard_changes(buf, guard=GUARD):
    """Number of changed sentinel bytes in the two guard bands of a `guarded` buffer."""
    return int((buf[:guard] != SENTINEL).sum()) + int((buf[buf.numel() - guard:] != SENTINEL).sum())


# ---- esmb200_gemm_fp8's argument refusals: (case, (epilogue, N, K[, {keyword: value}]), message), M = 128 -------------
GEMM_REFUSALS = [
    ("K%16", (1, 128, 24), "K % 16 == 0"),
    ("K=8", (5, 128, 8), "K % 16 == 0"),
    ("residual N%32", (1, 48, 128), "N % 32 == 0"),
    ("gelu N%128", (5, 192, 128), "N % 128 == 0"),
    ("qkv N!=3E", (0, 384, 128, {"E": 64}), "N == 3E"),
    ("qkv E%64", (0, 288, 128, {"E": 96}), "E % 64 == 0"),
    ("epilogue 2", (2, 128, 128), "must be 0 (qkv), 1 (residual) or 5"),
    ("epilogue 3", (3, 128, 128), "must be 0 (qkv), 1 (residual) or 5"),
    ("epilogue 4", (4, 128, 128), "must be 0 (qkv), 1 (residual) or 5"),
]


# ---- the fp8 kernels through the C ABI (GPU) -------------------------------------------------------------------------
def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def quantize_dev(x, block_rows):
    """esmb200_quantize_fp8 on the device (bit-exact against `quantize`, tests/test_gpu_fp8.py)."""
    from esm_b200 import _lib
    R, K = x.shape
    q = torch.empty(R, K, dtype=torch.uint8, device="cuda")
    s = torch.empty(*((-(-K // 128), R) if block_rows == 1 else (-(-R // 128), -(-K // 128))), device="cuda")
    _lib.check(_lib.load().esmb200_quantize_fp8(_p(x), _p(q), _p(s), R, K, block_rows, _s()))
    return q, s


def gemm_operands(kind, M, N, K, seed, out_limit=None):
    """kind "gauss": randn activations, randn K^-1/2 weights, bias 0.1 randn (nearly uniform scales); "spread":
    spread_operands, bias 0 (a bias would hide the small rows' products under its own rounding).  Quantised on the
    device; returns (qa, sa, qw, sw, bias, A, W) with A, W the dequantised float64 operands on the device."""
    if kind == "gauss":
        g = torch.Generator().manual_seed(seed)
        a = torch.randn(M, K, generator=g)
        w = torch.randn(N, K, generator=g) * K ** -0.5
        bias = 0.1 * torch.randn(N, generator=g)
    else:
        a, w = spread_operands(M, N, K, seed, out_limit)
        bias = torch.zeros(N)
    qa, sa = quantize_dev(a.cuda(), 1)
    qw, sw = quantize_dev(w.cuda(), 128)
    A = dequantize(qa.cpu().view(torch.float8_e4m3fn), sa.cpu(), 1).cuda()
    W = dequantize(qw.cpu().view(torch.float8_e4m3fn), sw.cpu(), 128).cuda()
    return qa, sa, qw, sw, bias.cuda(), A, W


def gelu64(x):
    return x * 0.5 * (1 + torch.erf(x / math.sqrt(2)))


def check_gemm(epi, M, N, K, kind, seed, T=64):
    """esmb200_gemm_fp8 with epilogue `epi` on (kind, M, N, K) operands against float64, every output (and fc1's output
    scales) inside guard bands and prefilled with 0xFF (NaN).  Asserts and returns {"ratio": max error / bound (QKV,
    residual), "flips", "scale_flips" (GELU)}.  QKV: E = N / 3, rope tables of 64-wide heads over T positions."""
    from esm_b200 import _lib as L
    lb = L.load()
    qkv = epi == L.EPI_QKV_ROPE
    # the fp16 QKV output: sum_k |A W| <= 2^14, so that q * 1/8 and k rotated (|c|, |s| <= 1, two terms) stay < 2^15
    qa, sa, qw, sw, bias, A, W = gemm_operands(kind, M, N, K, seed, out_limit=2.0 ** 14 if qkv else None)
    ref = A @ W.t() + bias.double()
    # a degenerate operand set (W all zero, say) would pass every check below by giving zeros
    assert float((ref != 0).double().mean()) >= 0.5, "at least half of the reference must be nonzero"
    # Gaussian operands: the blocks contribute comparably and their errors partly cancel, measured within 0.61 of the
    # 2^-12 per block bound; spread operands, where one K block can dominate an output: 2^-11 (acc_bound)
    bnd = acc_bound(A, W, 2.0 ** -12 if kind == "gauss" else 2.0 ** -11)
    res = {"ratio": 0.0, "flips": 0, "scale_flips": 0}
    tiny = 1e-300  # an exactly zero bound (the all-zero rows) then demands an exactly zero error
    if epi == L.EPI_BIAS_RESIDUAL:  # out += y
        out, buf = guarded((M, N), torch.float32, "cuda")
        g = torch.Generator().manual_seed(seed + 1)
        x0 = (torch.randn(M, N, generator=g) if kind == "gauss" else torch.zeros(M, N)).cuda()
        out.copy_(x0)
        L.check(lb.esmb200_gemm_fp8(epi, _p(qa), _p(sa), _p(qw), _p(sw), _p(bias), _p(out), None, M, N, K,
                                    None, None, 0, 0, _s()))
        torch.cuda.synchronize()
        y = out.double() - x0.double()
        # two fp32 roundings (y, then x + y) on top of the accumulation bound
        tol = bnd + 2.0 ** -23 * (ref.abs() + x0.double().abs()) * 2
        assert not bool(out.isnan().any()), "residual output not written"
        res["ratio"] = float(((y - ref).abs() / (tol + tiny)).max())
        bufs = [buf]
    elif qkv:  # rope tables over T positions (rows r -> position r % T), q columns * 1/8
        E = N // 3
        inv = 1.0 / (10000 ** (torch.arange(0, 64, 2).double() / 64))
        ang = torch.arange(T).double()[:, None] * inv[None]
        cos, sin = ang.cos().float().cuda(), ang.sin().float().cuda()
        out, buf = guarded((M, N), torch.float16, "cuda")
        L.check(lb.esmb200_gemm_fp8(epi, _p(qa), _p(sa), _p(qw), _p(sw), _p(bias), _p(out), None, M, N, K,
                                    _p(cos), _p(sin), T, E, _s()))
        torch.cuda.synchronize()
        y = ref.clone()
        y[:, :E] *= 0.125
        t = torch.arange(M, device="cuda") % T
        c, s = cos.double()[t], sin.double()[t]
        for sect in (0, 1):  # rotate-half inside every 64-wide slot: column j pairs with j + 32
            v = y[:, sect * E:(sect + 1) * E].view(M, -1, 2, 32)
            a0, b0 = v[:, :, 0].clone(), v[:, :, 1].clone()
            v[:, :, 0] = a0 * c[:, None] - b0 * s[:, None]
            v[:, :, 1] = b0 * c[:, None] + a0 * s[:, None]
        b2 = bnd.clone()
        b2[:, :E] *= 0.125
        b2[:, :2 * E] *= 2  # a rotated value mixes two accumulators
        # fp32 epilogue arithmetic and the fp16 rounding (half an ulp, 2^-11 relative; 2^-25 absolute for subnormals)
        tol = b2 + 2.0 ** -11 * y.abs() + 2.0 ** -24
        assert not bool(out.isnan().any()), "qkv output not written"
        assert float(y.abs().max()) < 2.0 ** 15
        res["ratio"] = float(((out.double() - y).abs() / tol).max())
        bufs = [buf]
    else:  # EPI_GELU_FP8 -> e4m3 + one scale per row and 128 columns
        out, buf = guarded((M, N), torch.uint8, "cuda")
        so, sbuf = guarded((N // 128, M), torch.float32, "cuda")
        L.check(lb.esmb200_gemm_fp8(epi, _p(qa), _p(sa), _p(qw), _p(sw), _p(bias), _p(out), _p(so), M, N, K,
                                    None, None, 0, 0, _s()))
        torch.cuda.synchronize()
        assert not bool(((out & 0x7F) == 0x7F).any()), "e4m3 output not written (NaN code)"
        assert not bool(so.isnan().any()), "output scale not written"
        y = gelu64(ref)
        # |GELU'| <= 1.13 carries the accumulation error; the kernel's erf (Abramowitz & Stegun 7.1.26) is within
        # 1.5e-7 absolute, x/2 1.5e-7 on GELU(x); its ex2 / rcp approximations and the fp32 bias add 2^-20 relative
        ybnd = bnd * 1.13 + 1e-7 * ref.abs() + 2.0 ** -20 * y.abs()
        r = check_codes(out.cpu().view(torch.float8_e4m3fn), so, y, ybnd)
        assert r["bad_scale"] == 0 and r["bad_code"] == 0, r
        # measured on an H100 (Gaussian operands): 0.5-0.7 % of the elements flip at a rounding boundary
        assert r["flips"] <= max(64, r["n"] // 50), r
        res.update(flips=r["flips"], scale_flips=r["scale_flips"])
        bufs = [buf, sbuf]
    assert all(guard_changes(b) == 0 for b in bufs), "write outside the output"
    assert res["ratio"] <= 1.0, res
    return res


def _ln(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    xc = x - mu
    rstd = (xc.pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    return xc * rstd * w + b, xc * rstd, rstd


def ln_error(x, w, xhat, rstd, y):
    """The fp32 LayerNorm's own error bound (DESIGN.md section 4): 4 2^-24 (8 + 2 sqrt(E) (1 + |mean| / std)) |w xhat|
    + 2^-24 |y|, with 1 / std = rstd (eps included: an all-zero padded row has xhat = 0)."""
    E = x.shape[-1]
    mean = x.mean(-1, keepdim=True).abs()
    return 4 * 2.0 ** -24 * (8 + 2 * math.sqrt(E) * (1 + mean * rstd)) * (w * xhat).abs() + 2.0 ** -24 * y.abs()


def emulate_layer(layer, x, pad, rope_inv_freq=None, gen=None):
    """One fp8 TransformerLayer (esm_b200.model.TransformerLayer, precision 2) in float64 on x fp32 [B, T, E] (the
    library's input), keys masked where pad [B, T] is true.  gen None: the exact emulation; a torch.Generator: the
    same with an error of the library's bound, random sign, injected wherever the library accumulates or rounds."""
    sa = layer.self_attn
    B, T, E = x.shape
    H = sa.num_heads
    dh = E // H
    M = B * T
    f = lambda t: t.detach().double()  # noqa: E731

    def inject(t, bound):
        if gen is None:
            return t
        sign = torch.randint(0, 2, t.shape, generator=gen).to(t.device, torch.float64) * 2 - 1
        return t + sign * bound

    x = f(x)
    w1, b1 = f(layer.self_attn_layer_norm.weight), f(layer.self_attn_layer_norm.bias)
    ln1, xhat, rstd = _ln(x, w1, b1, layer.self_attn_layer_norm.eps)
    A = requantize(inject(ln1, ln_error(x, w1, xhat, rstd, ln1)).reshape(M, E))
    Wq, Wk, Wv = quantized_qkv(sa.q_proj.weight.detach(), sa.k_proj.weight.detach(), sa.v_proj.weight.detach(), dh)
    qkv = []
    for W, bias in ((Wq, sa.q_proj.bias), (Wk, sa.k_proj.bias), (Wv, sa.v_proj.bias)):
        y = inject(A @ W.t() + f(bias), acc_bound(A, W, 2.0 ** -12))
        qkv.append(y.view(B, T, H, dh).transpose(1, 2))
    q, k, v = qkv
    q = q * dh ** -0.5
    if rope_inv_freq is not None:  # rotary_embedding.py:11-20 on the reference's head order, the library's fp32 angles
        ang = torch.arange(T, device=x.device).float()[:, None] * rope_inv_freq.detach().float()[None]
        c, s = ang.double().cos(), ang.double().sin()
        h2 = dh // 2
        q, k = (torch.cat((t[..., :h2] * c - t[..., h2:] * s, t[..., h2:] * c + t[..., :h2] * s), -1) for t in (q, k))
    q16, k16, v16 = (t.half().double() for t in (q, k, v))  # stored as fp16
    S = inject(q16 @ k16.transpose(-1, -2), dh * 2.0 ** -24 * (q16.abs() @ k16.abs().transpose(-1, -2)))
    P = torch.softmax(S.masked_fill(pad[:, None, None, :], float("-inf")), -1)
    P = inject(P, P * (2.0 ** -11 + 2.0 ** -20))  # P as fp16 for P.V; ex2.approx
    ctx = inject(P @ v16, T * 2.0 ** -24 * (P.abs() @ v16.abs()))
    c16 = ctx.transpose(1, 2).reshape(M, E).half().double()  # stored as fp16
    # out_proj: fp16 weights, fp16 GEMM (accumulation (K/16 + 4) 2^-22 sum|a w|, DESIGN.md section 4), residual add
    Wo = sa.out_proj.weight.detach().half().double()
    o = inject(c16 @ Wo.t() + f(sa.out_proj.bias), (E / 16 + 4) * 2.0 ** -22 * (c16.abs() @ Wo.abs().t()))
    x1 = x.reshape(M, E) + o
    w2, b2 = f(layer.final_layer_norm.weight), f(layer.final_layer_norm.bias)
    ln2, xhat2, rstd2 = _ln(x1, w2, b2, layer.final_layer_norm.eps)
    A2 = requantize(inject(ln2, ln_error(x1, w2, xhat2, rstd2, ln2)))
    W1 = weight8(layer.fc1.weight.detach())
    h = inject(A2 @ W1.t() + f(layer.fc1.bias), acc_bound(A2, W1, 2.0 ** -12))
    g = h * 0.5 * (1 + torch.erf(h / math.sqrt(2)))
    # the library's erf (A&S 7.1.26) is within 1.5e-7, its ex2 / rcp approximations 2^-20 relative
    G = requantize(inject(g, 0.75e-7 * h.abs() + 2.0 ** -20 * g.abs()))
    W2 = weight8(layer.fc2.weight.detach())
    yv = inject(G @ W2.t() + f(layer.fc2.bias), acc_bound(G, W2, 2.0 ** -12))
    return (x1 + yv).view(B, T, E)
