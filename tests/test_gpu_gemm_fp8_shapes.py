"""GPU (-m gpu): the block-scaled e4m3 GEMM (csrc/gemm_fp8.cuh) at its tile, K-block and scale edges, every epilogue
against float64 on the kernel's own dequantised operands (fp8_refs.check_gemm):

  * M around the 64-row halves of a 128-row tile (rows >= M take scale 0 in the second MMA warpgroup);
  * K < 128 (one K block, zero-filled by TMA), K just past a 128 boundary, and num_kb = 5, 6, 7 against the 6-stage
    ring with at least 3 tiles per CTA, so that the ring's phase crosses tile boundaries;
  * residual N with a partial 32-column box, QKV with E = 64 and 192 (the q / k / v section changes inside a 128-column
    tile), GELU N = 128 and 384;
  * tile counts n_sms - 1, n_sms, n_sms + 1 and 2 n_sms + 1.

Every case runs on scale-spread operands (row, K-block and weight-block scales over many octaves, all-zero blocks, a
block at a scale edge), inside guard bands, with the outputs prefilled with NaN.  The bound is fp8_refs.acc_bound, per
element and relative to |A| |W|^T, plus the epilogue's roundings.  Last, the entry point's argument refusals on a
device, with real buffers."""
import ctypes

import pytest
import torch

import fp8_refs as fr

pytestmark = pytest.mark.gpu

QKV, RESIDUAL, GELU = 0, 1, 5
NAMES = {QKV: "qkv", RESIDUAL: "residual", GELU: "gelu"}


def run(epi, M, N, K, seed, kind="spread"):
    r = fr.check_gemm(epi, M, N, K, kind, seed)
    print(f"PARITY fp8 gemm edge {NAMES[epi]} {kind} M={M} N={N} K={K}: err/bound={r['ratio']:.3f} "
          f"flips={r['flips']}/{M * N} scale_flips={r['scale_flips']}", flush=True)
    return r


@pytest.mark.parametrize("M", [63, 64, 65, 191, 192, 193])
def test_rows_around_the_warpgroup_halves(M):
    run(QKV, M, 3 * 128, 320, seed=M)          # E = 128; K = 320: a partial last K block
    run(RESIDUAL, M, 160, 320, seed=M + 1)     # a partial 128-column tile, one 32-column box in it
    run(GELU, M, 256, 320, seed=M + 2)


@pytest.mark.parametrize("K", [16, 112, 128, 144, 272])
def test_k_blocks(K):
    """K < 128: one K block, zero-filled past K by TMA on both operands; K = 144, 272: one column tail block."""
    run(QKV, 129, 3 * 64, K, seed=K)
    run(RESIDUAL, 129, 96, K, seed=K + 1)
    run(GELU, 129, 128, K, seed=K + 2)


@pytest.mark.parametrize("K", [640, 768, 784])
def test_k_blocks_against_the_stage_ring(K):
    """num_kb = 5, 6, 7 against the 6 stages, with at least 3 tiles per CTA (the ring index runs on across tiles)."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = 128 * n_sms + 1  # n_sms + 1 row tiles, 3 column tiles: >= 3 tiles per CTA
    run(RESIDUAL, M, 384, K, seed=K)
    run(GELU, M, 384, K, seed=K + 1)
    run(QKV, M, 384, K, seed=K + 2)


@pytest.mark.parametrize("N", [32, 96, 160])
def test_residual_partial_column_boxes(N):
    """N % 128 != 0: the last tile's 32-column boxes past N are skipped (the col0 >= N break)."""
    run(RESIDUAL, 200, N, 256, seed=N)


@pytest.mark.parametrize("E", [64, 192])
def test_qkv_sections_inside_a_tile(E):
    """E = 64 / 192: the q, k and v sections (q scaled, q and k rotated, v neither) change inside a 128-column tile."""
    run(QKV, 150, 3 * E, E, seed=E)
    run(QKV, 150, 3 * E, E, seed=E + 1, kind="gauss")


@pytest.mark.parametrize("N", [128, 384])
def test_gelu_widths(N):
    run(GELU, 130, N, 256, seed=N)
    run(GELU, 130, N, 256, seed=N + 1, kind="gauss")


@pytest.mark.parametrize("extra", ["n_sms-1", "n_sms", "n_sms+1", "2n_sms+1"])
def test_tile_counts_around_the_sm_count(extra):
    """The persistent loop with one tile per CTA and idle CTAs, exactly one each, and one or two CTAs with a second or
    third tile."""
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = {"n_sms-1": n_sms - 1, "n_sms": n_sms, "n_sms+1": n_sms + 1, "2n_sms+1": 2 * n_sms + 1}[extra]
    run(RESIDUAL, 128 * tiles - 5, 128, 144, seed=tiles)  # one column tile
    run(GELU, 128 * tiles - 70, 128, 144, seed=tiles + 1)
    if tiles % 3 == 0:  # QKV: N = 3E >= 192 has 3 column tiles at E = 128
        run(QKV, 128 * (tiles // 3) - 3, 3 * 128, 144, seed=tiles + 2)


@pytest.mark.parametrize("case,args,msg", fr.GEMM_REFUSALS + [
    ("gelu null out_scales", (5, 256, 128, {"out_scales": None}), "out_scales"),
    ("qkv no tables", (0, 384, 128, {"cos": None, "sin": None}), "rope tables"),
], ids=lambda v: v if isinstance(v, str) else "")
def test_refusals_with_real_buffers(case, args, msg):
    """The argument refusals of esmb200_gemm_fp8 (also checked on the CPU) on a device, with real buffers large enough
    for every shape here (M = 128, N <= 384, K <= 128): the call returns ESMB200_EINVAL and launches nothing."""
    from esm_b200 import _lib as L
    lib = L.load()
    epi, N, K = args[:3]
    kw = {"out_scales": True, "cos": True, "sin": True, **(args[3] if len(args) > 3 else {})}
    bufs = [torch.zeros(1 << 20, dtype=torch.uint8, device="cuda") for _ in range(9)]
    p = [ctypes.c_void_p(b.data_ptr()) for b in bufs]
    opt = lambda key, i: p[i] if kw[key] is not None else None  # noqa: E731
    E = kw.get("E", N // 3)
    torch.cuda.synchronize()
    before = lib.esmb200_launch_count()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.esmb200_gemm_fp8(epi, p[0], p[1], p[2], p[3], p[4], p[5], opt("out_scales", 6), 128, N, K,
                              opt("cos", 7), opt("sin", 8), 64, E, stream)
    assert rc == -1 and msg in lib.esmb200_last_error().decode()
    assert lib.esmb200_launch_count() == before
