"""GPU (-m gpu): each sm_90a kernel, called through the C ABI, against a plain PyTorch fp32 evaluation of the same
op on the same device.  Inputs to the tensor-core kernels are rounded to fp16 first, so the comparison isolates the
kernel (fp32 accumulation order) from the operand-precision choice; tolerances are stated per test.  The attention
cases run through test_gpu_attention_f16.check16, against float64 within the derived bounds of kernel_refs."""
import ctypes
import math

import pytest
import torch

import test_gpu_attention_f16 as f16

pytestmark = pytest.mark.gpu


def _lib():
    from esm_b200 import _lib
    return _lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def rope_ref(x, cos, sin):
    # x [..., T, 64]; cos/sin [T, 32]
    x1, x2 = x[..., :32], x[..., 32:]
    return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), -1)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.mark.parametrize("M,E", [(8, 128), (1000, 1280), (77, 2560), (33, 320), (5, 5120)])
def test_layernorm_f32_and_f16(dev, M, E):
    L = _lib(); lib = L.load()
    g = torch.Generator(device="cpu").manual_seed(M * 7 + E)
    x = (torch.randn(M, E, generator=g) * 3 + 0.5).to(dev)
    w = (1 + 0.2 * torch.randn(E, generator=g)).to(dev)
    b = (0.1 * torch.randn(E, generator=g)).to(dev)
    ref = torch.nn.functional.layer_norm(x, (E,), w, b, 1e-5)
    out = torch.empty_like(x)
    L.check(lib.esmb200_layernorm(P(x), P(w), P(b), P(out), M, E, 1e-5, S()))
    torch.testing.assert_close(out, ref, atol=2e-5, rtol=2e-5)
    out16 = torch.empty(M, E, dtype=torch.float16, device=dev)
    L.check(lib.esmb200_layernorm_f16(P(x), P(w), P(b), P(out16), M, E, 1e-5, S()))
    torch.testing.assert_close(out16.float(), ref.half().float(), atol=2e-3, rtol=2e-3)  # 1 fp16 ulp of slack


def _gemm_inputs(dev, M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn(M, K, generator=g).half().to(dev)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half().to(dev)
    bias = (0.1 * torch.randn(N, generator=g)).to(dev)
    return a, w, bias


# fp32 accumulation of fp16 products in a different order than cuBLAS: |err| <~ 1e-5 * sqrt(K); fp16 outputs add
# half an ulp (2^-11 relative).
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 256, 128), (256, 512, 1280), (300, 384, 128),
                                   (1000, 1280, 5120), (129, 64, 64), (4096, 3840, 1280)])
def test_gemm_bias_f32(dev, M, N, K):
    L = _lib(); lib = L.load()
    a, w, bias = _gemm_inputs(dev, M, N, K, 1)
    out = torch.full((M, N), float("nan"), device=dev)
    L.check(lib.esmb200_gemm_f16(L.EPI_BIAS_F32, P(a), P(w), P(bias), P(out), M, N, K, None, None, 0, 0, S()))
    ref = a.float() @ w.float().t() + bias
    torch.testing.assert_close(out, ref, atol=2e-4, rtol=1e-4)


@pytest.mark.parametrize("M,N,K", [(300, 1280, 1280), (128, 128, 5120), (1111, 2560, 640)])
def test_gemm_bias_residual_inplace(dev, M, N, K):
    L = _lib(); lib = L.load()
    a, w, bias = _gemm_inputs(dev, M, N, K, 2)
    x0 = torch.randn(M, N, device=dev) * 2
    x = x0.clone()
    L.check(lib.esmb200_gemm_f16(L.EPI_BIAS_RESIDUAL, P(a), P(w), P(bias), P(x), M, N, K, None, None, 0, 0, S()))
    ref = x0 + (a.float() @ w.float().t() + bias)
    torch.testing.assert_close(x, ref, atol=3e-4, rtol=1e-4)


@pytest.mark.parametrize("M,N,K", [(256, 5120, 1280), (130, 512, 128)])
def test_gemm_bias_gelu_f16(dev, M, N, K):
    L = _lib(); lib = L.load()
    a, w, bias = _gemm_inputs(dev, M, N, K, 3)
    out = torch.empty(M, N, dtype=torch.float16, device=dev)
    L.check(lib.esmb200_gemm_f16(L.EPI_BIAS_GELU, P(a), P(w), P(bias), P(out), M, N, K, None, None, 0, 0, S()))
    h = a.float() @ w.float().t() + bias
    ref = h * 0.5 * (1.0 + torch.erf(h / math.sqrt(2.0)))
    torch.testing.assert_close(out.float(), ref, atol=2e-3, rtol=2e-3)


@pytest.mark.parametrize("B,T,H", [(2, 40, 2), (3, 200, 4), (2, 1024, 20)])
def test_gemm_qkv_rope(dev, B, T, H):
    """q/k/v projection + bias + q*d^-1/2 + rotate-half RoPE, against multihead_attention.py:258-261,354-355 semantics."""
    from esm_b200.model import rope_tables
    L = _lib(); lib = L.load()
    E = 64 * H
    M = B * T
    a, w, bias = _gemm_inputs(dev, M, 3 * E, E, 4)
    inv_freq = (1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))).to(dev)
    cos, sin = rope_tables(inv_freq, T)
    out = torch.empty(M, 3 * E, dtype=torch.float16, device=dev)
    L.check(lib.esmb200_gemm_f16(L.EPI_QKV_ROPE, P(a), P(w), P(bias), P(out), M, 3 * E, E, P(cos), P(sin), T, E, S()))
    y = (a.float() @ w.float().t() + bias).view(B, T, 3, H, 64)
    q = rope_ref(y[:, :, 0].transpose(1, 2) * 0.125, cos, sin)  # [B,H,T,64]
    k = rope_ref(y[:, :, 1].transpose(1, 2), cos, sin)
    v = y[:, :, 2].transpose(1, 2)
    ref = torch.stack((q, k, v), 0).permute(1, 3, 0, 2, 4).reshape(M, 3 * E)
    torch.testing.assert_close(out.float(), ref, atol=3e-3, rtol=2e-3)


@pytest.mark.parametrize("B,T,H,lengths", [
    (1, 128, 1, None), (2, 40, 2, [40, 23]), (3, 200, 4, [200, 150, 7]), (2, 300, 2, None),
    (2, 1024, 20, [1024, 517]), (1, 129, 1, [129]), (2, 256, 1, [256, 128]),
])
def test_attention_forward_and_probs(dev, B, T, H, lengths):
    """softmax(QK^T + key-padding mask) V (multihead_attention.py:357-394) incl. ragged lengths, T not a multiple of
    128, fully padded key blocks; and the need_head_weights probabilities (:397-400).  Against float64 on the same fp16
    q, k, v within the bounds of kernel_refs (test_gpu_attention_f16.check16)."""
    g = torch.Generator(device="cpu").manual_seed(B * 1000 + T)
    qkv = torch.randn(B * T, 3 * 64 * H, generator=g)
    qkv[:, :64 * H] *= 0.5  # q is pre-scaled in the real pipeline; keep logits O(1..10)
    f16.check16("forward and probs", qkv.half().to(dev), f16.pad_of(B, T, lengths), B, T, H, 64)


@pytest.mark.parametrize("B,T,H,lengths", [(1, 128, 1, None), (2, 200, 3, [200, 61]), (2, 1024, 4, [1024, 517]),
                                            (1, 129, 2, [129])])
def test_attention_head_dim_128(dev, B, T, H, lengths):
    """esm2_t48_15B's head width (pretrained.py:390-397): the same contract as above on 128-wide heads (two 64-wide
    column slots per head: QK^T sums both, P.V runs once per slot), context and probabilities."""
    g = torch.Generator(device="cpu").manual_seed(B * 977 + T)
    qkv = torch.randn(B * T, 3 * 128 * H, generator=g)
    qkv[:, :128 * H] *= 0.35
    f16.check16("head dim 128", qkv.half().to(dev), f16.pad_of(B, T, lengths), B, T, H, 128)


@pytest.mark.parametrize("D,B,H", [(64, 1, 2), (128, 1, 2), (128, 3, 40)])
def test_attention_reference_max_raise(dev, D, B, H):
    """Scores that keep growing along the key axis (each 128-key block beats the previous maximum by far more than
    the lazy-rescale threshold) force the O-rescale / block-redo path; result must still be the exact softmax.
    (D = 128: the double-buffered two-slot kernel, whose rescale waits for the previous P.V; the 3 x 40-head case keeps
    every CTA of the GPU busy with several tiles.)"""
    T = 640
    E = D * H
    g = torch.Generator(device="cpu").manual_seed(5)
    qkv = torch.randn(B * T, 3 * E, generator=g)
    u = torch.randn(D, generator=g)
    u = u / u.norm() * (8.0 ** 0.5)                              # |u|^2 = 8
    blk = (torch.arange(B * T).float() % T / 128).floor()
    for h in range(H):
        qkv[:, h * D:(h + 1) * D] = u + 0.1 * torch.randn(B * T, D, generator=g)
        # logits ~ 8 * 0.8 * block index: every block tops the previous maximum by ~6.4 > tau (5.5)
        qkv[:, E + h * D:E + (h + 1) * D] = u * (0.8 * blk[:, None]) + 0.3 * torch.randn(B * T, D, generator=g)
    f16.check16("max raise", qkv.half().to(dev), None, B, T, H, D)


@pytest.mark.parametrize("D", [64, 128])
def test_attention_left_and_interior_padding_with_very_negative_scores(dev, D):
    """ADVICE r1: when the first key block is fully padded the reference maximum must be seeded from the first block that
    has an attendable key — with scores around -40 a reference of 0 would round every probability to 0 in fp16.  Left
    padding (first 130 keys) and an interior gap, all valid logits ~ -40."""
    B, T, H = 2, 400, 2
    E = D * H
    g = torch.Generator(device="cpu").manual_seed(17)
    u = torch.randn(D, generator=g)
    u = u / u.norm() * (40.0 ** 0.5)
    qkv = 0.05 * torch.randn(B * T, 3 * E, generator=g)
    for h in range(H):
        qkv[:, h * D:(h + 1) * D] += u
        qkv[:, E + h * D:E + (h + 1) * D] -= u
    qkv[:, 2 * E:] = torch.randn(B * T, E, generator=g)
    pad = torch.zeros(B, T, dtype=torch.uint8)
    pad[0, :130] = 1            # left padding: blocks 0 and 1 (64-key blocks) fully masked, block 2 partially
    pad[1, 64:200] = 1          # interior gap
    pad[1, 390:] = 1
    out = f16.check16("left padding, gap, logits ~-40", qkv.half().to(dev), pad.to(dev), B, T, H, D)
    assert out["ctx_absmax"] > 0.05


def test_embed_tokens(dev):
    from oracle import esm2_oracle
    from oracle.weights import make_state_dict, make_tokens
    L = _lib(); lib = L.load()
    sd = make_state_dict(1, 128, 2)
    tokens = make_tokens([38, 21, 30], 40, n_mask=3)
    ref = esm2_oracle.embed(tokens, sd)
    x = torch.empty(3, 40, 128, device=dev)
    tab = sd["embed_tokens.weight"].to(dev)
    tk = tokens.to(dev)
    L.check(lib.esmb200_embed_tokens(P(tk), P(tab), P(x), 3, 40, 128, 1, 32, 1, S()))
    torch.testing.assert_close(x.cpu(), ref, atol=1e-6, rtol=1e-6)


def test_embed_tokens_row_chunks(dev):
    """The row-chunked grid (several blocks per sequence) against the oracle on a longer ragged batch, with and without
    token dropout; T is not a multiple of the chunk size."""
    from oracle import esm2_oracle
    from oracle.weights import make_state_dict, make_tokens
    L = _lib(); lib = L.load()
    sd = make_state_dict(1, 320, 20)
    tokens = make_tokens([1001, 333, 20], 1003, n_mask=5)
    tab = sd["embed_tokens.weight"].to(dev)
    for dropout in (1, 0):
        ref = esm2_oracle.embed(tokens, sd, bool(dropout))
        x = torch.full((3, 1003, 320), float("nan"), device=dev)
        L.check(lib.esmb200_embed_tokens(P(tokens.to(dev)), P(tab), P(x), 3, 1003, 320, 1, 32, dropout, S()))
        torch.testing.assert_close(x.cpu(), ref, atol=1e-6, rtol=1e-6)


@pytest.mark.parametrize("B,T,E", [(3, 40, 128), (2, 1024, 1280), (5, 77, 320), (1, 2, 64)])
def test_mean_pool(dev, B, T, E):
    """scripts/extract.py:116-119: mean over the residues 1 .. len (the <cls> row excluded), lengths 1 .. T-1."""
    L = _lib(); lib = L.load()
    g = torch.Generator().manual_seed(B * 31 + T)
    x = torch.randn(B, T, E, generator=g).to(dev)
    lens = [T - 1] + [max(1, (T - 1) // (b + 2)) for b in range(B - 1)]
    lengths = torch.tensor(lens, dtype=torch.int32, device=dev)
    out = torch.full((B, E), float("nan"), device=dev)
    L.check(lib.esmb200_mean_pool(P(x), P(lengths), P(out), B, T, E, S()))
    ref = torch.stack([x[b, 1: 1 + n].double().mean(0) for b, n in enumerate(lens)]).float()
    torch.testing.assert_close(out, ref, atol=2e-6, rtol=1e-5)
    out2 = torch.empty_like(out)
    L.check(lib.esmb200_mean_pool(P(x), P(lengths), P(out2), B, T, E, S()))
    assert torch.equal(out, out2)


def test_error_reporting(dev):
    L = _lib(); lib = L.load()
    a = torch.zeros(128, 100, dtype=torch.float16, device=dev)
    rc = lib.esmb200_gemm_f16(L.EPI_BIAS_F32, P(a), P(a), P(a), P(a), 128, 128, 100, None, None, 0, 0, S())
    assert rc == -1 and b"K % 8" in lib.esmb200_last_error()
    with pytest.raises(L.Esmb200Error):
        L.check(rc)
