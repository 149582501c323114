"""GPU (-m gpu): one whole TransformerLayer (esmb200_layer_forward) at every kind of head width esmb200_layer_create
accepts, against kernel_refs.layer64 in float64 on the same fp32 parameters.

Heads run in zero-padded 64-wide column slots (csrc/elementwise.cuh head_slot): one slot for d <= 64, two above, the
rotation pair p = (j, j + d/2) at columns (p % 32, 32 + p % 32) of slot p / 32.  d = 40 and 48 leave d/2 short of the
32 pairs of a slot without dividing it; d = 66 .. 126 fill the second slot only partly (d = 66: one pair, d = 72: four,
d = 96: sixteen, d = 126: thirty-one).  A dimension packed into the wrong slot, or rotated by the wrong table column,
changes the attention logits by O(1).

T = 130 (one row past a 128-row tile), B = 2 with the second sequence padded, probabilities requested."""
import ctypes

import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

# rel-Frobenius of the layer's residual update (out - x) at the valid positions, and max-abs of the probabilities of the
# valid query rows; about twice what an H100 (80 GB HBM3, 700 W) gave:
#   precision 0 (the error of the fp16 q, k, v and P): update 6.7e-4 .. 7.1e-4, probabilities 8.7e-4 .. 1.6e-3 over the
#                twelve widths, no trend with d
#   precision 1: update 2.1e-6 .. 4.1e-6, probabilities 1.8e-6 .. 3.3e-6 at d = 8, 32, 48
# head_slot sending every pair to slot 0 moves the update by 0.32 .. 0.72 and the probabilities by 0.68 .. 0.99 at d > 64.
GATES = {0: (1.4e-3, 3.2e-3), 1: (1e-5, 1e-5)}

# d: (E, H); E % 16 == 0, and E % 64 == 0 where precision 1 runs
SHAPES = {8: (64, 8), 16: (320, 20), 24: (480, 20), 32: (128, 4), 40: (160, 4), 48: (192, 4), 64: (256, 4),
          66: (528, 8), 72: (288, 4), 96: (384, 4), 126: (1008, 8), 128: (256, 2)}
CASES = [(d, 0) for d in SHAPES] + [(8, 1), (32, 1), (48, 1)]


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


@pytest.mark.parametrize("d,precision", CASES)
def test_layer_at_head_width_against_float64(d, precision):
    check_layer(d, precision, 130, [130, 97])


def check_layer(d, precision, T, lengths, gates=None):
    """One layer of head width d (SHAPES) on B = len(lengths) sequences of T positions, sequence b padded from
    lengths[b] on, against layer64; held to `gates` (default GATES[precision]).  Returns (update rel-Fro, probs
    max-abs)."""
    from esm_b200.model import TransformerLayer
    from oracle.weights import make_state_dict
    E, H = SHAPES[d]
    assert E // H == d
    B = len(lengths)
    sd = make_state_dict(1, E, H, seed=d)
    layer = TransformerLayer(E, 4 * E, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items() if k.startswith("layers.0.")}, strict=True)
    layer = layer.cuda()
    layer.precision = precision
    x = torch.randn(T, B, E, generator=torch.Generator().manual_seed(d + 1))
    pad = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lengths):
        pad[b, n:] = True
    with torch.no_grad():
        out, attn = layer(x.cuda(), self_attn_padding_mask=pad.cuda(), need_head_weights=True)  # (T,B,E), (H,B,T,T)
    torch.cuda.synchronize()
    xb = x.transpose(0, 1).double()
    ref, p = kr.layer64(xb, {k: v.double() for k, v in sd.items()}, "layers.0.", H, pad)  # [B,T,E], [B,H,T,T]
    keep = ~pad
    got = out.transpose(0, 1).double().cpu()
    d_got, d_ref = (got - xb)[keep], (ref - xb)[keep]
    r = float((d_got - d_ref).norm() / d_ref.norm())
    pa = float((attn.transpose(0, 1).double().cpu() - p).abs()[keep[:, None, :, None].expand_as(p)].max())
    report(f"layer head width d={d} E={E} H={H} precision={precision} T={T}", delta_rel_fro=r, probs_max_abs=pa)
    gate_r, gate_p = gates or GATES[precision]
    assert r <= gate_r and pa <= gate_p
    layer.release()
    return r, pa


REFUSED_WIDTHS = [
    (240, 16, 0, b"even head_dim <= 128"),                 # d = 15
    (1040, 8, 0, b"even head_dim <= 128"),                 # d = 130
    (40, 5, 0, b"multiple of 16"),                         # d = 8, E % 16 = 8
    (576, 8, 1, b"not available for head_dim > 64"),       # d = 72 in fp32x3
    (480, 20, 1, b"embed_dim % 64 == 0"),                  # d = 24, E % 64 = 32 in fp32x3
]


@pytest.mark.parametrize("E,H,precision,message", REFUSED_WIDTHS)
def test_layer_create_refuses_unsupported_widths(E, H, precision, message):
    from esm_b200 import _lib
    lib = _lib.load()
    torch.cuda.init()
    w = _lib.LayerWeights()
    w.embed_dim, w.num_heads, w.ffn_dim, w.precision = E, H, 4 * E, precision
    w.fc1_weight = 1  # a feed-forward layer; no pointer is read before the shape is refused
    before = lib.esmb200_launch_count()
    out = ctypes.c_void_p()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.esmb200_layer_create(ctypes.byref(w), stream, ctypes.byref(out)) == -1
    assert message in lib.esmb200_last_error(), lib.esmb200_last_error()
    assert not out.value and lib.esmb200_launch_count() == before


@pytest.mark.parametrize("E,H,precision,message", REFUSED_WIDTHS + [
    (320, 20, 3, b"precision must be 0"),
    (320, 20, 2, b"needs a_scales and w_scales"),          # scales not given
    (320, 20, 0, b"rope tables must be given together"),   # cos without sin
])
def test_gemm_qkv_heads_refuses_what_layer_create_refuses(E, H, precision, message):
    """esmb200_gemm_qkv_heads refuses the widths and precisions esmb200_layer_create refuses, with its messages, before
    any launch and without reading an operand (the pointers below are not device memory)"""
    from esm_b200 import _lib
    lib = _lib.load()
    torch.cuda.init()
    fake = ctypes.c_void_p(256)
    scales = None if message == b"needs a_scales and w_scales" else fake
    sin = None if message == b"rope tables must be given together" else fake
    before = lib.esmb200_launch_count()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.esmb200_gemm_qkv_heads(precision, fake, scales, fake, scales, fake, fake, 128, E, H, 0.125, fake, sin, 16,
                                    stream)
    assert rc == -1
    assert message in lib.esmb200_last_error(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before
