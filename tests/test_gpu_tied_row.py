"""GPU (-m gpu): the fp16 tied row attention of the MSA Transformer (esmb200_tied_row_attention: tied_scores_kernel,
tied_softmax_kernel, tied_pv_kernel <false>) at the shapes where the kernels have edges: C not a multiple of 64 / 128
(boxes that read into the next alignment row, zero P columns in [C, Cp)), R not a multiple of the four alignment rows
a P.V CTA handles, C = 1, C = 1024 (the softmax's register limit), R = 1024 (the longest K chain of the logits), key
padding, and an alignment whose key columns are all padded.  Each case runs through
test_gpu_tied_attention.check_tied: every stage and ctx end to end against float64 within the bounds of kernel_refs,
with and without probabilities."""
import pytest
import torch

import test_gpu_tied_attention as tied

pytestmark = pytest.mark.gpu


def inputs(B, R, C, H, seed, pad_cols=0, pad_all=None):
    """fp16 qkv [B*R*C, 3E] with q scaled so that the summed logits have std ~3, and key_pad [B,C] (uint8) or None.
    q is zeroed at padded columns, as the MSA layer does (axial_attention.py:82-85)."""
    pad = None
    if pad_cols or pad_all is not None:
        pad = torch.zeros(B, C, dtype=torch.uint8, device="cuda")
        if pad_cols:
            pad[:, C - pad_cols:] = 1
            pad[0, C // 3] = 1
        if pad_all is not None:
            pad[pad_all] = 1
    return tied.make_qkv(B, R, C, H, seed, key_pad=pad), pad


SHAPES = [(1, 1, 1, 1), (2, 3, 64, 2), (1, 5, 65, 1), (1, 7, 127, 2), (2, 6, 128, 4), (1, 2, 129, 12),
          (1, 2, 1024, 1), (1, 1024, 64, 2)]


@pytest.mark.parametrize("B,R,C,H", SHAPES)
def test_tied_row_attention_against_float64(B, R, C, H):
    qkv, _ = inputs(B, R, C, H, seed=B * 7919 + R * 31 + C)
    tied.check_tied("shape", qkv, None, B, R, C, H, False)


@pytest.mark.parametrize("pad_cols", [0, 40])
def test_tied_row_attention_with_key_padding(pad_cols):
    B, R, C, H = 3, 6, 300, 2
    qkv, pad = inputs(B, R, C, H, seed=11 + pad_cols, pad_cols=pad_cols)
    if pad is None:
        pad = torch.zeros(B, C, dtype=torch.uint8, device="cuda")  # a key_pad with nothing padded
    tied.check_tied(f"key_pad pad_cols={pad_cols}", qkv, pad, B, R, C, H, False)


def test_tied_row_attention_all_keys_padded():
    """Every key column of alignment 1 is padded: all its logits are -10000 and the softmax is uniform, 1 / C."""
    B, R, C, H = 2, 3, 130, 2
    qkv, pad = inputs(B, R, C, H, seed=5, pad_all=1)
    _, pr = tied.check_tied("all keys padded", qkv, pad, B, R, C, H, False)
    assert bool((pr[:, 1] == torch.ones((), device="cuda") / C).all())


def test_tied_row_attention_rejects_more_than_1024_columns():
    from esm_b200 import _lib
    lib = _lib.load()
    B, R, C, H = 1, 1, 1025, 1
    qkv = torch.zeros(B * R * C, 3 * 64 * H, dtype=torch.float16, device="cuda")
    ctx = torch.empty(B * R * C, 64 * H, dtype=torch.float16, device="cuda")
    nbytes = lib.esmb200_tied_row_attention_scratch_bytes(B, C, H)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    rc = lib.esmb200_tied_row_attention(qkv.data_ptr(), None, ctx.data_ptr(), None, B, R, C, H, scratch.data_ptr(),
                                        nbytes, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"1024" in lib.esmb200_last_error()
