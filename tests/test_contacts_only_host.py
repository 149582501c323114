"""CPU: esmb200_stack_contacts_bytes (the partial buffers and probability scratch of the contacts-only stack) is pure
host arithmetic; its values are pinned here, and ContactPredictionHead.begin_contacts allocates exactly that much."""
import ctypes

import pytest
import torch


def contact_bytes(*args):
    from esm_b200 import _lib
    out = [ctypes.c_size_t(7) for _ in range(3)]
    rc = _lib.load().esmb200_stack_contacts_bytes(*args, *[ctypes.byref(o) for o in out])
    return rc, tuple(o.value for o in out)


@pytest.mark.parametrize("args,sizes", [
    # (n_layers, heads, B, T, S, precision): (row_part, col_part, scratch) bytes
    ((33, 20, 64, 1024, 1022, 0), (5525667840, 5525667840, 0)),      # 650M, extract_cli's default 64 x 1024 batch
    ((36, 40, 16, 512, 510, 0), (752025600, 752025600, 0)),          # 3B, 16 x 512
    ((48, 40, 1, 4096, 4094, 0), (4024565760, 4024565760, 0)),       # 15B, one 4096-token protein
    ((6, 20, 3, 77, 75, 2), (432000, 432000, 0)),                     # fp8: the fused layout
    ((3, 4, 2, 300, 298, 1), (28608, 543552, 2880000)),              # fp32x3: row sums, 16-row stripes, one layer
    ((33, 20, 64, 1024, 1022, 1), (172677120, 11051335680, 5368709120)),
    ((1, 1, 1, 1, 1, 0), (16, 16, 0)),
])
def test_sizes_are_pinned(args, sizes):
    assert contact_bytes(*args) == (0, sizes)


def test_partials_are_a_sixteenth_of_the_stack():
    L, H, B, T = 33, 20, 64, 1024
    _, (row, col, _) = contact_bytes(L, H, B, T, T - 2, 0)
    stack = 4 * B * L * H * T * T
    assert 16 < stack / (row + col) < 16.1  # T^2 / (2 * 32 * (T - 2))


@pytest.mark.parametrize("args", [(0, 20, 1, 10, 8, 0), (1, 0, 1, 10, 8, 0), (1, 20, 0, 10, 8, 0), (1, 20, 1, 0, 1, 0),
                                  (1, 20, 1, 10, 0, 0), (1, 20, 1, 10, 11, 0), (1, 20, 1, 10, 8, 3),
                                  (1, 20, 1, 10, 8, -1)])
def test_bad_arguments_are_refused(args):
    from esm_b200 import _lib
    rc, sizes = contact_bytes(*args)
    assert rc == -1 and sizes == (7, 7, 7)  # ESMB200_EINVAL, nothing written
    assert _lib.load().esmb200_last_error() == b"bad shape"


def test_null_out_pointers_are_allowed():
    from esm_b200 import _lib
    assert _lib.load().esmb200_stack_contacts_bytes(2, 2, 1, 10, 8, 0, None, None, None) == 0


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("append_eos", [True, False])
def test_begin_contacts_allocates_what_the_helper_states(precision, append_eos):
    from esm_b200.model import ContactPredictionHead
    L, H, B, T = 3, 4, 2, 300
    head = ContactPredictionHead(L * H, prepend_bos=True, append_eos=append_eos, eos_idx=2)
    tokens = torch.full((B, T), 5, dtype=torch.int64)
    st = head.begin_contacts(tokens, L, H, precision)
    S = T - 1 - int(append_eos)
    _, (row, col, scratch) = contact_bytes(L, H, B, T, S, precision)
    assert st["row"].nbytes == row and st["col"].nbytes == col
    assert (st["scratch"].nbytes if "scratch" in st else 0) == scratch
    assert st["acc"].shape == (B, S, S) and bool((st["acc"] == 0).all())
    assert (st["job"].lo, st["job"].hi) == (1, 1 + S)
    assert (st["keep"] is not None) == append_eos
