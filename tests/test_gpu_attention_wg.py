"""GPU (-m gpu): the warpgroup-MMA attention forward (csrc/attention_wg.cuh), which runs every fp16 attention with
64-wide heads: esmb200_attention and esmb200_column_attention against float64 softmax attention of the same fp16
inputs, through test_gpu_attention_f16.check16 (ctx element-wise and per (sequence, head), the probabilities and the
saved statistics, each within its derived bound in kernel_refs)."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

import test_gpu_attention_f16 as f16

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
    f16.check16(f"lengths={lengths}", qkv, _pad(B, T, lengths, qkv.device), B, T, H, 64)


def test_all_padding_sequence_gives_zero(L):
    B, T, H = 3, 300, 2
    qkv = _qkv(B, T, H, 7)
    pad = _pad(B, T, [300, 0, 131], qkv.device)
    ctx, pr, scratch = _run(L, qkv, pad, B, T, H)
    mx, sm = _stats(scratch, B, T, H)
    name = f"attention_f16 D=64 all-padding sequence B={B} T={T} H={H}"
    assert f16.exact(name + " ctx", ctx[T:2 * T], torch.zeros_like(ctx[T:2 * T]))
    assert f16.exact(name + " row max", mx[1], torch.zeros_like(mx[1]))
    assert f16.exact(name + " row sum", sm[1], torch.zeros_like(sm[1]))
    f16.check16("all padding", qkv, pad, B, T, H, 64)


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
    out = f16.check16("left padding, gap, logits ~-40", qkv, pad.cuda(), B, T, H, 64)
    assert out["ctx_absmax"] > 0.05


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
    f16.check16("rising maximum", qkv.half().cuda(), None, B, T, H, 64)


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
    assert f16.exact(f"attention_f16 D=64 one-hot rows B={B} T={T} H={H}", ctx, qkv[perm.cuda(), 128:])


@pytest.mark.parametrize("B,R,C,H,ragged", [(1, 128, 8, 2, False), (2, 77, 5, 3, True), (1, 200, 3, 12, True)])
def test_column_attention(L, B, R, C, H, ragged):
    """MSA column attention (cols > 1: the R tokens of a column are C rows of qkv apart) against float64 on the
    regrouped tensor [B*C, R, 3E]; R not a multiple of 128 and padded rows."""
    E = 64 * H
    g = torch.Generator(device="cpu").manual_seed(B * 31 + R + C)
    qkv = torch.randn(B, R, C, 3 * E, generator=g)
    qkv[..., :E] *= 0.5
    qkv = qkv.half().cuda().view(B * R * C, 3 * E)
    pad = torch.zeros(B, C, R, dtype=torch.uint8)
    if ragged:
        for b in range(B):
            for c in range(C):
                pad[b, c, (R * (c + 1)) // (C + 1) + 1:] = 1
        pad[0, 0, :] = 1  # a column that is all padding
    f16.check_column("ragged" if ragged else "full", qkv, pad.cuda(), B, R, C, H)


def test_many_more_items_than_sms_at_full_size(L):
    """The configs[1] shape (256 x 1024 tokens, 20 heads): ~40k work items, so every persistent CTA walks hundreds;
    ragged lengths; ctx element-wise and per (sequence, head) against float64, checked in chunks of sequences."""
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
    out = f16.measure(qkv, pad, B, T, H, 64, ctx)
    f16.assert_within(f"attention_f16 D=64 many items B={B} T={T} H={H}", out)


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
