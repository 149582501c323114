"""CPU: the fp8 precision, everything that needs no device — the scale rule and e4m3 rounding of the torch reference the
GPU tests compare the kernels with, set_precision("fp8") on every model shape, the pinned workspace size, the offload
refusals, extract_cli --precision fp8, and the fp8 GEMM in the SASS of the shipped library."""
import ctypes
import os
import shutil
import subprocess
from argparse import Namespace

import pytest
import torch

import fp8_refs as fr


def test_scale_is_the_smallest_power_of_two():
    assert fr.block_scale(0.0) == 1.0                       # all-zero block
    assert fr.block_scale(448.0) == 1.0                     # the exact amax: 448 / 1 <= 448
    assert fr.block_scale(448.0 * (1 + 2 ** -20)) == 2.0    # just above it
    assert fr.block_scale(1.0) == 2.0 ** -8                 # 256 <= 448 < 512
    assert fr.block_scale(1.75) == 2.0 ** -8 and fr.block_scale(1.76) == 2.0 ** -7
    assert fr.block_scale(1e-40) == 2.0 ** -126             # never below the smallest normal float
    for a in torch.rand(200, dtype=torch.float64) * 1e4:
        s = fr.block_scale(float(a))
        assert a / s <= 448 < a / (s / 2)
    amax = torch.tensor([0.0, 448.0, 449.0, 1.0, 1e-40, 3.5e7])
    assert [fr.block_scale(float(a)) for a in amax] == fr.scales_of(amax).tolist()


def test_quantize_rounds_to_nearest_even_and_keeps_signs():
    x = torch.zeros(2, 256)
    x[0, 0] = 448.0                      # scale 1
    x[0, 1] = -17.0                      # between 16 and 18: a tie, rounds to the even code 16
    x[0, 2] = -19.0                      # tie between 18 and 20: 20
    x[0, 3] = 2.0 ** -9                  # the smallest e4m3 subnormal at scale 1
    x[0, 4] = 2.0 ** -11                 # half of it: rounds to zero (even)
    x[0, 5] = 3 * 2.0 ** -10             # tie between 2^-9 and 2^-8: the even code 2^-8
    q, s = fr.quantize(x, 1)
    assert s.shape == (2, 2) and s[0, 0] == 1.0 and s[1, 0] == 1.0  # block 1 of row 0 and row 1: all zero
    d = q.float()[0, :6].tolist()
    assert d == [448.0, -16.0, -20.0, 2.0 ** -9, 0.0, 2.0 ** -8]


def test_partial_blocks_take_their_scale_over_valid_columns():
    x = torch.zeros(130, 320)
    x[:, 256:] = 3.0                     # the partial third K block (64 valid columns)
    x[129, 5] = 900.0                    # a weight block of 2 valid rows
    q, s = fr.quantize(x, 1)
    assert s.shape == (3, 130) and bool((s[2] == 2.0 ** -7).all()) and bool((s[:2, :129] == 1).all())
    qw, sw = fr.quantize(x, 128)
    assert sw.shape == (2, 3) and sw[1, 0] == 4.0 and sw[0, 2] == 2.0 ** -7
    back = fr.dequantize(q, s, 1)
    assert torch.equal(back[:, 256:].float(), x[:, 256:])


def _layer_shapes():
    # (num_layers, embed_dim, heads): every esm2_* size's layer shape, ESM-1b / 1v's
    return [(1, 320, 20), (1, 480, 20), (1, 640, 20), (1, 1280, 20), (1, 2560, 40), (1, 5120, 40)]


@pytest.mark.parametrize("L,E,H", _layer_shapes())
def test_set_precision_fp8_on_every_esm2_shape(L, E, H):
    from esm_b200 import ESM2
    with torch.device("meta"):
        model = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    model.set_precision("fp8")
    assert model.precision == "fp8" and all(layer.precision == 2 for layer in model.layers)
    assert model._lm_head_precision() == 0  # the fp8 mode's LM head runs fp16
    model.set_precision("fp16")
    assert all(layer.precision == 0 for layer in model.layers)


def test_set_precision_fp8_on_esm1b():
    from esm_b200 import ProteinBertModel
    args = Namespace(arch="roberta_large", layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2,
                     max_positions=1024, token_dropout=True, emb_layer_norm_before=True)
    model = ProteinBertModel(args, "roberta_large")
    model.set_precision("fp8")
    assert model.layers[0].precision == 2


def test_msa_transformer_refuses_fp8():
    from esm_b200.msa import MSATransformer
    m = MSATransformer(Namespace(layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2, max_positions=1024,
                                 embed_positions_msa=True))
    with pytest.raises(ValueError):
        m.set_precision("fp8")


@pytest.mark.parametrize("args,nbytes", [
    ((1280, 20, 5120, 256, 1024), 3072362496),   # 650M, the bulk-embedding batch
    ((320, 20, 1280, 2, 100), 2149376),          # 8M: partial K blocks (E = 320)
    ((480, 20, 1920, 3, 77), 2521088),           # 35M
    ((5120, 40, 20480, 1, 1024), 47678976),      # 15B: two-slot heads
])
def test_fp8_workspace_bytes_are_pinned(args, nbytes):
    from esm_b200 import _lib
    lib = _lib.load()
    assert lib.esmb200_workspace_bytes(*args, 2) == nbytes
    assert lib.esmb200_layer_packed_bytes(args[0], args[1], args[2], 2) == 0  # fp8 layers are not streamed


def test_cpu_offload_refuses_fp8():
    from esm_b200 import ESM2, _lib
    model = ESM2(num_layers=1, embed_dim=64, attention_heads=2).set_precision("fp8")
    with pytest.raises(_lib.Esmb200Error, match="fp8"):
        model.cpu_offload()
    model.set_precision("fp16")
    model._offload = ("cuda:0", None)  # an offloaded model (cpu_offload() needs a device)
    with pytest.raises(_lib.Esmb200Error, match="fp8"):
        model.set_precision("fp8")
    assert model.precision == "fp16" and model.layers[0].precision == 0
    model._offload = None


def test_extract_cli_parses_fp8():
    from esm_b200.extract_cli import create_parser
    a = create_parser().parse_args(["esm2_t6_8M_UR50D", "x.fasta", "out", "--include", "mean", "--precision", "fp8"])
    assert a.precision == "fp8"


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump not available")
def test_fp8_gemm_runs_e4m3_wgmma_without_spills():
    from esm_b200 import _lib
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for epi in (0, 1, 5):
        name = f"gemm_fp8_e4m3_kernelILi{epi}E"
        i = sass.index(name)
        j = sass.find("Function :", i)
        body = sass[i:j if j > 0 else None]
        assert body.count("QGMMA.64x128x32.F32.E4M3.E4M3") == 4
        assert "LDL" not in body and "STL" not in body
    assert sass.count("gemm2_f16_kernel") >= 10


# ---- argument refusals of the fp8 entry points: every check below returns before the device is touched ---------------
# The calls pass a placeholder pointer, which a refused call never dereferences.  They run only where no CUDA device is
# present, so that a refusal lost from the library can never turn into a kernel launch on a bad address; on a machine
# with a device, tests/test_gpu_gemm_fp8_shapes.py checks the GEMM refusals with real buffers.
_FAKE = ctypes.c_void_p(4096)
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="placeholder pointers: only where nothing can launch")


def _gemm(epi, N, K, M=128, out_scales=_FAKE, cos=_FAKE, sin=_FAKE, T=64, E=None):
    from esm_b200 import _lib
    lib = _lib.load()
    E = N // 3 if E is None else E
    rc = lib.esmb200_gemm_fp8(epi, _FAKE, _FAKE, _FAKE, _FAKE, _FAKE, _FAKE, out_scales, M, N, K, cos, sin, T, E, None)
    return rc, lib.esmb200_last_error().decode()




@no_device
@pytest.mark.parametrize("case,args,msg", fr.GEMM_REFUSALS, ids=lambda v: v if isinstance(v, str) else "")
def test_gemm_fp8_refuses_bad_shapes(case, args, msg):
    from esm_b200 import _lib
    kw = args[3] if len(args) > 3 else {}
    before = _lib.load().esmb200_launch_count()
    rc, err = _gemm(*args[:3], **kw)
    assert rc == -1 and msg in err, err
    assert _lib.load().esmb200_launch_count() == before


@no_device
@pytest.mark.parametrize("kw", [{"out_scales": None}], ids=["gelu-null-out_scales"])
def test_gemm_fp8_gelu_refuses_null_out_scales(kw):
    rc, err = _gemm(5, 256, 128, **kw)
    assert rc == -1 and "out_scales" in err


@no_device
@pytest.mark.parametrize("kw", [{"cos": None}, {"sin": None}, {"cos": None, "sin": None}, {"T": 0}],
                         ids=["no-cos", "no-sin", "no-tables", "T=0"])
def test_gemm_fp8_qkv_refuses_missing_tables(kw):
    rc, err = _gemm(0, 384, 128, **kw)
    assert rc == -1 and "rope tables" in err


@no_device
@pytest.mark.parametrize("M,E", [(8, 130), (8, 5122), (8, 5124), (8, 6144), (0, 128), (8, 0)])
def test_layernorm_fp8_refuses_bad_shapes(M, E):
    from esm_b200 import _lib
    lib = _lib.load()
    rc = lib.esmb200_layernorm_fp8(_FAKE, _FAKE, _FAKE, _FAKE, _FAKE, M, E, 1e-5, None)
    assert rc == -1 and b"bad shape" in lib.esmb200_last_error()


@no_device
@pytest.mark.parametrize("block_rows", [0, 2, 64, 127, 129, 256, -1])
def test_quantize_fp8_refuses_block_rows(block_rows):
    from esm_b200 import _lib
    lib = _lib.load()
    rc = lib.esmb200_quantize_fp8(_FAKE, _FAKE, _FAKE, 256, 256, block_rows, None)
    assert rc == -1 and b"block_rows 1 or 128" in lib.esmb200_last_error()


# ---- the helpers the fp8 GPU tests compare with (fp8_refs): a checker that cannot fail tests nothing -----------------
# the (M, N, K) of the scale-spread runs in tests/test_gpu_gemm_fp8_shapes.py with N or K of at most a few blocks
SMALL_SHAPES = ([(129, n, k) for k in (16, 112, 128, 144, 272) for n in (192, 96, 128)]
                + [(200, 32, 256), (200, 96, 256), (200, 160, 256), (150, 192, 64), (150, 576, 192), (130, 128, 256),
                   (130, 384, 256), (63, 384, 320), (63, 160, 320), (63, 256, 320), (123, 128, 144)])


@pytest.mark.parametrize("M,N,K", SMALL_SHAPES)
def test_spread_operands_keep_every_output_live(M, N, K):
    """Every output column and every K block of W (the partial last one included) carries nonzero weights, and the
    reference A W^T is nonzero almost everywhere: no edge case can pass by multiplying by zero."""
    a, w = fr.spread_operands(M, N, K, seed=M + N + K)
    kb = -(-K // 128)
    assert bool((w != 0).any(1).all())
    for k in range(kb):
        assert bool((w[:, 128 * k:128 * (k + 1)] != 0).any(1).all()) or (k == 0 and kb > 1), k
    ref = a.double() @ w.double().t()
    assert float((ref != 0).double().mean()) >= 0.9


def test_spread_operands_spread_the_scales():
    M, N, K = 300, 384, 640
    a, w = fr.spread_operands(M, N, K, seed=1)
    qa, sa = fr.quantize(a, 1)      # [5, 300]
    qw, sw = fr.quantize(w, 128)    # [3, 5]
    ea, ew = torch.log2(sa).round().long(), torch.log2(sw).round().long()
    assert len(ea.unique()) >= 30 and len(ew.unique()) >= 8
    assert float((ea[:, 1:] != ea[:, :-1]).float().mean()) >= 0.8      # neighbouring rows
    assert float((ea[1:, :] != ea[:-1, :]).float().mean()) >= 0.8      # neighbouring K blocks of a row
    assert float((ew[:, 1:] != ew[:, :-1]).float().mean()) >= 0.75     # neighbouring weight blocks
    assert bool((sa[:, M // 3] == 1).all()) and bool((a[M // 3] == 0).all())      # the all-zero row
    assert sa[-1, M // 2] == 1 and bool((a[M // 2, 512:] == 0).all())             # the all-zero A block
    assert sw[-1, 0] == 1 and bool((w[256:, :128] == 0).all())                    # the all-zero weight block
    r = (2 * M) // 3                                                                # the block at a scale edge
    assert float(a[r, :128].abs().max()) == 448.0 * float(sa[0, r])
    assert float(qa[r, 5]) == -448.0
    # every sa sb stays a normal float far above 2^-126, also after out_limit's row shifts
    a2, w2 = fr.spread_operands(M, N, K, seed=1, out_limit=2.0 ** 14)
    qa2, sa2 = fr.quantize(a2, 1)
    assert float(sa2.min()) * float(sw.min()) >= 2.0 ** -100
    assert float((a2.double().abs() @ w2.double().abs().t()).max()) <= 2.0 ** 14
    d = torch.log2(sa2) - torch.log2(sa)  # one power of two per row: the spread inside a row is kept
    live = a.view(M, 5, 128).abs().amax(-1).t() > 0
    assert all(len(d[:, m][live[:, m]].unique()) <= 1 for m in range(M))
    assert torch.equal(qa2.view(torch.uint8), qa.view(torch.uint8))


def _ln_like(R, N, seed):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(R, N, generator=g, dtype=torch.float64) * torch.exp(2 * torch.randn(R, 1, generator=g,
                                                                                          dtype=torch.float64))
    return y, 1e-7 * y.abs()


def test_code_checker_accepts_the_reference():
    y, ybnd = _ln_like(40, 260, seed=2)
    q, s = fr.quantize(y.float(), 1)
    r = fr.check_codes(q, s, y, ybnd)
    assert r["bad_scale"] == 0 and r["bad_code"] == 0 and r["flips"] == 0 and r["scale_flips"] == 0


def test_code_checker_rejects_a_doubled_scale_away_from_an_edge():
    y, ybnd = _ln_like(40, 260, seed=3)
    y[7, 128:256] *= 300.0 / float(y[7, 128:256].abs().max())  # block (row 7, K block 1): amax 300, far from 256 and 512
    q, s = fr.quantize(y.float(), 1)
    s2 = s.clone()
    s2[1, 7] *= 2                                               # the LayerNorm with its scale doubled
    q2 = q.clone()
    q2[7, 128:256] = (y[7, 128:256].float() / float(s2[1, 7])).to(torch.float8_e4m3fn)
    r = fr.check_codes(q2, s2, y, ybnd)
    assert r["bad_scale"] == 1
    # at an edge the same doubling is a legal flip: amax within the bound of 448 s
    y[7, 128:256] *= 448.0 * float(s[1, 7]) * (1 - 1e-9) / float(y[7, 128:256].abs().max())
    q, s = fr.quantize(y.float(), 1)
    s2 = s.clone()
    s2[1, 7] *= 2
    q2 = q.clone()
    q2[7, 128:256] = (y[7, 128:256].float() / float(s2[1, 7])).to(torch.float8_e4m3fn)
    r = fr.check_codes(q2, s2, y, ybnd)
    assert r["bad_scale"] == 0 and r["bad_code"] == 0 and r["scale_flips"] == 1


def test_code_checker_rejects_a_code_one_step_off():
    y, ybnd = _ln_like(40, 260, seed=4)
    q, s = fr.quantize(y.float(), 1)
    y = fr.dequantize(q, s, 1)              # y exactly on its codes: as far from a midpoint as it gets
    b = q.view(torch.uint8).clone()
    i, j = 11, 140
    assert 0 < (int(b[i, j]) & 0x7F) < 0x7E
    b[i, j] += 1                            # one e4m3 step up in magnitude
    r = fr.check_codes(b.view(torch.float8_e4m3fn), s, y, ybnd)
    assert r["bad_code"] == 1 and r["bad_scale"] == 0
    # a value within the bound of a midpoint may flip
    y2 = y.clone()
    lo, hi = fr.dequantize(q, s, 1)[i, j], fr.dequantize(b.view(torch.float8_e4m3fn), s, 1)[i, j]
    y2[i, j] = (lo + hi) / 2 + (lo - hi) * 1e-6  # just on the reference's side of the midpoint
    r = fr.check_codes(b.view(torch.float8_e4m3fn), s, y2, ybnd)
    assert r["bad_code"] == 0 and r["flips"] == 1


def test_guard_band_helper_reports_one_changed_byte():
    for where in (0, fr.GUARD - 1, -fr.GUARD, -1):
        t, buf = fr.guarded((3, 5), torch.float32, "cpu")
        assert bool(t.isnan().all()) and fr.guard_changes(buf) == 0
        t.fill_(1.0)                          # the tensor itself is not guarded
        assert fr.guard_changes(buf) == 0
        buf[where] ^= 1
        assert fr.guard_changes(buf) == 1
