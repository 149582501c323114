"""Torch statements of the fp8 precision's quantisation (esmb200.h, esmb200_quantize_fp8), shared by the CPU and GPU tests.

A block's scale is the smallest power of two s with amax / s <= 448 (e4m3's largest finite value), at least 2^-126, and 1
for an all-zero block.  Dividing by a power of two is exact, so q = (x / s).to(torch.float8_e4m3fn) and q * s are the
kernel's bits exactly.
"""
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


# ---- float64 emulation of one fp8 layer -------------------------------------------------------------------------------
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


def acc_bound(A, W):
    """Accumulation bound of the fp8 GEMM: per 128-wide K block the tensor cores' internal sum keeps at least 13
    significand bits (DeepSeek-V3 section 3.3.2 measured about 14), 2^-12 of the block's sum of |products|; the fp32
    promotion adds 2^-24 of the running sum per block: 2^-12 (1 + 2^-12 K/128) |A|.|W|^T."""
    K = A.shape[-1]
    return (A.abs() @ W.abs().t()) * (2.0 ** -12 * (1 + 2.0 ** -12 * math.ceil(K / 128)))


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
        y = inject(A @ W.t() + f(bias), acc_bound(A, W))
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
    h = inject(A2 @ W1.t() + f(layer.fc1.bias), acc_bound(A2, W1))
    g = h * 0.5 * (1 + torch.erf(h / math.sqrt(2)))
    # the library's erf (A&S 7.1.26) is within 1.5e-7, its ex2 / rcp approximations 2^-20 relative
    G = requantize(inject(g, 0.75e-7 * h.abs() + 2.0 ** -20 * g.abs()))
    W2 = weight8(layer.fc2.weight.detach())
    yv = inject(G @ W2.t() + f(layer.fc2.bias), acc_bound(G, W2))
    return (x1 + yv).view(B, T, E)
