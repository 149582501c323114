"""Greedy row selection of a deep alignment for the MSA Transformer, on the GPU.

The MSA Transformer takes a few hundred rows, while an a3m file often holds thousands. The reference's contact workflow
(examples/contact_prediction.ipynb, "MSA Transformer") passes each alignment through greedy_select(msa, num_seqs=128)
before predict_contacts: starting from the query, it adds one row at a time, the one with the largest ("max") or
smallest ("min") mean Hamming distance to the rows already picked. The selection is discrete, so this module returns
the same rows as the notebook's function for every input, exactly (the rule, including the order in which numpy sums
the distances, is stated in include/esmb200.h at esmb200_msa_greedy_select). Bytes are compared, as the notebook
compares them, not token ids.

    msa = variants.read_msa("family.a3m", None)
    msa = msa_select.greedy_select(msa, num_seqs=128)
    tokens = alphabet.get_batch_converter()([msa])[2].cuda()
    contacts = model.predict_contacts(tokens)

Each step is one kernel launch that reads the alignment once; the picked row's index stays on the device, so nothing
waits for the host until the indices are returned.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from .model import _ptr, _stream

MODES = {"max": _lib.SELECT_MAX, "min": _lib.SELECT_MIN}
MAX_COLUMNS = 65535  # the Hamming counts are stored as uint16


def _check_mode(mode: str) -> int:
    if mode not in MODES:
        raise ValueError(f"mode must be 'max' or 'min', got {mode!r}")
    return MODES[mode]


def _order(rows_u8: torch.Tensor, num_seqs: int, mode: str) -> torch.Tensor:
    """The picked rows' indices int64 [min(num_seqs, N)] on the device, in selection order."""
    code = _check_mode(mode)
    if not isinstance(rows_u8, torch.Tensor) or rows_u8.dtype != torch.uint8 or rows_u8.dim() != 2:
        raise ValueError("rows_u8 must be a uint8 tensor [N, C]")
    if not rows_u8.is_cuda:
        raise ValueError("rows_u8 must be on a CUDA device")
    N, C = rows_u8.shape
    if N >= 2 ** 31:
        raise ValueError(f"at most 2^31 - 1 rows, got {N}")
    dev = rows_u8.device
    if N <= num_seqs:
        return torch.arange(N, dtype=torch.int64, device=dev)
    if num_seqs <= 1:
        return torch.zeros(1, dtype=torch.int64, device=dev)
    if not 1 <= C <= MAX_COLUMNS:
        raise ValueError(f"rows must have 1 to {MAX_COLUMNS} columns, got {C}")
    ld = -(-C // 16) * 16
    if C == ld and rows_u8.stride() == (ld, 1) and rows_u8.data_ptr() % 16 == 0:
        rows = rows_u8
    else:  # pad every row to 16 bytes with the same byte, which then never counts as a difference
        rows = torch.zeros((N, ld), dtype=torch.uint8, device=dev)
        rows[:, :C] = rows_u8
    lib = _lib.load()
    with torch.cuda.device(dev):
        selected = torch.empty(num_seqs, dtype=torch.int64, device=dev)
        nbytes = lib.esmb200_msa_select_scratch_bytes(N, C, num_seqs)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _lib.check(lib.esmb200_msa_greedy_select(_ptr(rows), ld, N, C, num_seqs, code, _ptr(selected), _ptr(scratch),
                                                 nbytes, _stream()))
    return selected


def greedy_select_indices(rows_u8: torch.Tensor, num_seqs: int, mode: str = "max") -> torch.Tensor:
    """The rows greedy_select keeps, as sorted int64 indices on the device, for an alignment already on the GPU as
    bytes: rows_u8 uint8 [N, C] (any strides). All N rows when N <= num_seqs, only the query (row 0) when
    num_seqs <= 1. Nothing synchronises with the host."""
    return torch.sort(_order(rows_u8, num_seqs, mode)).values


def _as_bytes(msa: Sequence[Tuple[str, str]]) -> np.ndarray:
    """The notebook's byte array uint8 [N, C]; rows of unequal length raise ValueError, as np.array raises it."""
    seqs = [seq for _, seq in msa]
    C = len(seqs[0])
    if any(len(s) != C for s in seqs):
        raise ValueError("every alignment row must have the same length")
    return np.frombuffer(bytearray("".join(seqs).encode("ascii")), dtype=np.uint8).reshape(len(seqs), C)


def greedy_select(msa: List[Tuple[str, str]], num_seqs: int, mode: str = "max",
                  device: Optional[torch.device] = None) -> List[Tuple[str, str]]:
    """greedy_select of examples/contact_prediction.ipynb on the GPU, with the same rows for every input: msa is a list
    of (description, sequence) of one length. Returns msa itself when len(msa) <= num_seqs; otherwise num_seqs rows
    (only the query when num_seqs <= 1), in their order in msa. device: the CUDA device to run on (default: the
    current one)."""
    _check_mode(mode)
    if len(msa) <= num_seqs:
        return msa
    rows = _as_bytes(msa)
    if num_seqs <= 1:
        return [msa[0]]
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    idx = greedy_select_indices(torch.from_numpy(rows).to(dev), num_seqs, mode)
    return [msa[i] for i in idx.tolist()]
