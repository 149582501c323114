"""GPU (-m gpu): the warpgroup-MMA attention forward (csrc/attention_wg.cuh), which runs every fp16 attention with
64-wide heads: esmb200_attention and esmb200_column_attention against an fp32 PyTorch softmax attention of the same
fp16 inputs.  Tolerances as in test_gpu_kernels.py: P is rounded to fp16 before P.V (ctx 4e-3), the statistics are
fp32 (compared through the probabilities the probability kernel forms from them, and directly)."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

pytestmark = pytest.mark.gpu


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def L():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    from esm_b200 import _lib
    return _lib


def _pad(B, T, lengths, dev):
    if lengths is None:
        return None
    pad = torch.zeros(B, T, dtype=torch.uint8)
    for b, n in enumerate(lengths):
        pad[b, n:] = 1
    return pad.to(dev)


def _ref(qkv, pad, B, T, H):
    """ctx [B*T, 64H], probabilities [B,H,T,T], row max of the scaled scores and sum of exp(s - max) [B,H,T]."""
    E = 64 * H
    y = qkv.float().view(B, T, 3, H, 64)
    q, k, v = (y[:, :, i].transpose(1, 2) for i in range(3))
    s = q @ k.transpose(-1, -2)
    if pad is not None:
        s = s.masked_fill(pad[:, None, None, :].bool(), float("-inf"))
    m = s.amax(-1)
    m0 = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m0[..., None])
    l = e.sum(-1)
    p = e / torch.where(l > 0, l, torch.ones_like(l))[..., None]
    o = (p @ v).transpose(1, 2).reshape(B * T, E)
    return o, p, m0, l


def _run(L, qkv, pad, B, T, H, probs=True):
    lib = L.load()
    dev = qkv.device
    ctx = torch.full((B * T, 64 * H), float("nan"), dtype=torch.float16, device=dev)
    pr = torch.full((B, H, T, T), float("nan"), device=dev) if probs else None
    scratch = torch.empty(lib.esmb200_attention_scratch_bytes(B, T), dtype=torch.uint8, device=dev)
    L.check(lib.esmb200_attention(P(qkv), P(pad), P(ctx), P(pr), B, T, H, P(scratch), S()))
    torch.cuda.synchronize()
    return ctx, pr, scratch


def _stats(scratch, B, T, H):
    """row_max / row_sum from the scratch layout (api.cu attn_scratch_layout)"""
    def up(v):
        return (v + 255) // 256 * 256
    words = (T + 31) // 32
    words = (words + 3) // 4 * 4
    off = up(B * words * 4) + up(B * 4)
    n = B * H * T
    raw = scratch[off:off + up(n * 4) + n * 4]
    mx = raw[:n * 4].view(torch.float32).view(B, H, T)
    sm = raw[up(n * 4):up(n * 4) + n * 4].view(torch.float32).view(B, H, T)
    return mx, sm


def _qkv(B, T, H, seed, q_scale=0.5):
    g = torch.Generator(device="cpu").manual_seed(seed)
    qkv = torch.randn(B * T, 3 * 64 * H, generator=g)
    qkv[:, :64 * H] *= q_scale
    return qkv.half().cuda()


@pytest.mark.parametrize("T", [1, 63, 64, 65, 127, 128, 129, 200, 1023, 1024])
def test_lengths_context_probs_and_stats(L, T):
    B, H = 3, 2
    lengths = [T, max(1, T // 2), max(1, (2 * T) // 3 - 1)]
    qkv = _qkv(B, T, H, 100 + T)
    pad = _pad(B, T, lengths, qkv.device)
    ctx, pr, scratch = _run(L, qkv, pad, B, T, H)
    ref_o, ref_p, ref_m, ref_l = _ref(qkv, pad, B, T, H)
    torch.testing.assert_close(ctx.float(), ref_o, atol=4e-3, rtol=4e-3)
    torch.testing.assert_close(pr, ref_p, atol=2e-5, rtol=2e-4)
    mx, sm = _stats(scratch, B, T, H)
    torch.testing.assert_close(mx, ref_m, atol=2e-5, rtol=2e-5)
    torch.testing.assert_close(sm, ref_l, atol=1e-4, rtol=2e-5)
    ctx2, _, _ = _run(L, qkv, pad, B, T, H, probs=False)
    assert torch.equal(ctx, ctx2)  # with and without probabilities
    ctx3, _, _ = _run(L, qkv, pad, B, T, H, probs=False)
    assert torch.equal(ctx2, ctx3)  # two identical calls


def test_all_padding_sequence_gives_zero(L):
    B, T, H = 3, 300, 2
    qkv = _qkv(B, T, H, 7)
    pad = _pad(B, T, [300, 0, 131], qkv.device)
    ctx, pr, scratch = _run(L, qkv, pad, B, T, H)
    ref_o, _, ref_m, ref_l = _ref(qkv, pad, B, T, H)
    assert torch.equal(ctx[T:2 * T], torch.zeros_like(ctx[T:2 * T]))
    mx, sm = _stats(scratch, B, T, H)
    assert torch.equal(mx[1], torch.zeros_like(mx[1])) and torch.equal(sm[1], torch.zeros_like(sm[1]))
    torch.testing.assert_close(ctx.float(), ref_o, atol=4e-3, rtol=4e-3)
    torch.testing.assert_close(mx, ref_m, atol=2e-5, rtol=2e-5)
    torch.testing.assert_close(sm, ref_l, atol=1e-4, rtol=2e-5)


def test_left_padding_and_interior_gap_at_minus_40(L):
    """The first 128-key block fully padded and an interior gap; every valid score is about -40, so a reference
    maximum that is not seeded from the first attendable key would flush P to zero."""
    B, T, H = 2, 500, 2
    E = 64 * H
    g = torch.Generator(device="cpu").manual_seed(17)
    u = torch.randn(64, generator=g)
    u = u / u.norm() * (40.0 ** 0.5)
    qkv = 0.05 * torch.randn(B * T, 3 * E, generator=g)
    for h in range(H):
        qkv[:, h * 64:(h + 1) * 64] += u
        qkv[:, E + h * 64:E + (h + 1) * 64] -= u
    qkv[:, 2 * E:] = torch.randn(B * T, E, generator=g)
    qkv = qkv.half().cuda()
    pad = torch.zeros(B, T, dtype=torch.uint8)
    pad[0, :260] = 1          # blocks 0 and 1 fully masked, block 2 partially
    pad[1, 64:300] = 1        # interior gap across a block boundary
    pad[1, 490:] = 1
    pad = pad.cuda()
    ctx, pr, scratch = _run(L, qkv, pad, B, T, H)
    ref_o, ref_p, ref_m, ref_l = _ref(qkv, pad, B, T, H)
    assert float(ref_o.abs().max()) > 0.05
    torch.testing.assert_close(ctx.float(), ref_o, atol=4e-3, rtol=4e-3)
    torch.testing.assert_close(pr, ref_p, atol=2e-5, rtol=1e-3)
    mx, sm = _stats(scratch, B, T, H)
    torch.testing.assert_close(mx, ref_m, atol=1e-4, rtol=2e-5)
    torch.testing.assert_close(sm, ref_l, atol=1e-4, rtol=1e-4)


def test_running_maximum_rises_every_block(L):
    """Scores grow block after block (each 128-key block beats the previous maximum by ~6.4): every block rescales
    O and l."""
    B, H, T = 2, 3, 1000
    E = 64 * H
    g = torch.Generator(device="cpu").manual_seed(5)
    qkv = torch.randn(B * T, 3 * E, generator=g)
    u = torch.randn(64, generator=g)
    u = u / u.norm() * (8.0 ** 0.5)
    blk = (torch.arange(B * T).float() % T / 128).floor()
    for h in range(H):
        qkv[:, h * 64:(h + 1) * 64] = u + 0.1 * torch.randn(B * T, 64, generator=g)
        qkv[:, E + h * 64:E + (h + 1) * 64] = u * (0.8 * blk[:, None]) + 0.3 * torch.randn(B * T, 64, generator=g)
    qkv = qkv.half().cuda()
    ctx, pr, scratch = _run(L, qkv, None, B, T, H)
    ref_o, ref_p, ref_m, ref_l = _ref(qkv, None, B, T, H)
    torch.testing.assert_close(ctx.float(), ref_o, atol=4e-3, rtol=4e-3)
    torch.testing.assert_close(pr, ref_p, atol=1e-4, rtol=1e-3)
    mx, sm = _stats(scratch, B, T, H)
    torch.testing.assert_close(mx, ref_m, atol=1e-4, rtol=2e-5)
    torch.testing.assert_close(sm, ref_l, atol=1e-4, rtol=1e-4)


def test_one_hot_rows_read_every_value_exactly(L):
    """Query i scores 60 on key perm[i] and at most ~30 on every other key, so its fp16 P row is exactly one-hot and
    ctx row i is v[perm[i]] bit for bit: pins the element mapping of the MN-major V descriptor and of the P register
    operand over all 128 keys and 64 columns of a block, in every block of the sequence."""
    B, T, H = 1, 384, 1
    g = torch.Generator(device="cpu").manual_seed(3)
    perm = torch.randperm(T, generator=g)
    k = torch.randn(T, 64, generator=g)
    k = k / k.norm(dim=1, keepdim=True) * 8.0  # |k|^2 = 64; k_i . k_j ~ 64 * N(0, 1/64) for i != j
    qkv = torch.empty(T, 3 * 64)
    qkv[:, :64] = k[perm] * (60.0 / 64.0)
    qkv[:, 64:128] = k
    qkv[:, 128:] = torch.randn(T, 64, generator=g)
    qkv = qkv.half().cuda()
    s = qkv[:, :64].float() @ qkv[:, 64:128].float().t()
    top2 = s.topk(2, dim=1).values
    assert float((top2[:, 0] - top2[:, 1]).min()) > 25.0  # exp(-25) is below the smallest fp16 subnormal
    ctx, _, _ = _run(L, qkv, None, B, T, H, probs=False)
    assert torch.equal(ctx, qkv[perm.cuda(), 128:])


@pytest.mark.parametrize("B,R,C,H,ragged", [(1, 128, 8, 2, False), (2, 77, 5, 3, True), (1, 200, 3, 12, True)])
def test_column_attention(L, B, R, C, H, ragged):
    """MSA column attention (cols > 1: the R tokens of a column are C rows of qkv apart) against torch on the
    regrouped tensor [B*C, R, 3E]; R not a multiple of 128 and padded rows."""
    lib = L.load()
    E = 64 * H
    g = torch.Generator(device="cpu").manual_seed(B * 31 + R + C)
    qkv = torch.randn(B, R, C, 3 * E, generator=g)
    qkv[..., :E] *= 0.5
    qkv = qkv.half().cuda()
    pad = torch.zeros(B, C, R, dtype=torch.uint8)
    if ragged:
        for b in range(B):
            for c in range(C):
                pad[b, c, (R * (c + 1)) // (C + 1) + 1:] = 1
        pad[0, 0, :] = 1  # a column that is all padding
    pad = pad.cuda()
    ctx = torch.full((B * R * C, E), float("nan"), dtype=torch.float16, device="cuda")
    scratch = torch.empty(lib.esmb200_attention_scratch_bytes(B * C, R), dtype=torch.uint8, device="cuda")
    L.check(lib.esmb200_column_attention(P(qkv), P(pad), P(ctx), B, R, C, H, P(scratch), S()))
    torch.cuda.synchronize()
    reg = qkv.permute(0, 2, 1, 3).reshape(B * C * R, 3 * E).contiguous()
    ref_o, _, _, _ = _ref(reg, pad.view(B * C, R), B * C, R, H)
    ref_o = ref_o.view(B, C, R, E).permute(0, 2, 1, 3).reshape(B * R * C, E)
    torch.testing.assert_close(ctx.float(), ref_o, atol=4e-3, rtol=4e-3)


def test_many_more_items_than_sms_at_full_size(L):
    """The configs[1] shape (256 x 1024 tokens, 20 heads): ~40k work items, so every persistent CTA walks hundreds;
    ragged lengths; checked against torch in chunks of sequences."""
    B, T, H = 256, 1024, 20
    E = 64 * H
    g = torch.Generator(device="cpu").manual_seed(11)
    lengths = [T - (37 * b) % 700 for b in range(B)]
    qkv = torch.randn(B * T, 3 * E, generator=g)
    qkv[:, :E] *= 0.5
    qkv = qkv.half().cuda()
    pad = _pad(B, T, lengths, qkv.device)
    ctx, _, _ = _run(L, qkv, pad, B, T, H, probs=False)
    ctx2, _, _ = _run(L, qkv, pad, B, T, H, probs=False)
    assert torch.equal(ctx, ctx2)
    for b0 in range(0, B, 32):
        rows = slice(b0 * T, (b0 + 32) * T)
        ref_o, _, _, _ = _ref(qkv[rows], pad[b0:b0 + 32], 32, T, H)
        torch.testing.assert_close(ctx[rows].float(), ref_o, atol=4e-3, rtol=4e-3)


def test_kernel_runs_on_warpgroup_mma(L):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump) or not os.path.exists(L.LIB_PATH):
        pytest.skip("cuobjdump or the built library is not available")
    sass = subprocess.run([cuobjdump, "-sass", L.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    counts, cur = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            counts[cur] = 0
        elif cur and "HGMMA" in line:
            counts[cur] += 1
    wg = [n for n in counts if "attention_wg_kernel" in n]
    assert len(wg) == 1 and counts[wg[0]] > 0, counts
