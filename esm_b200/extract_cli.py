"""`python -m esm_b200.extract_cli MODEL FASTA OUT_DIR --include mean per_tok ...` — bulk extraction driver with the
command line and the output files of the reference's `esm-extract` (/root/reference/scripts/extract.py:15-131): one
`{label}.pt` per sequence holding {"label", "representations": {layer: [len,E]}, "mean_representations",
"bos_representations", "contacts"} as selected by --include.

What differs from the reference's loop (which runs the model, copies whole padded batches to the host and calls
torch.save in line, so the GPU idles during the copies and the pickling):
  * the model runs through libesmb200.so (GPU required; there is no --nogpu path);
  * --include contacts runs the forward without the [B,L,H,T,T] attention stack (same contacts, bit for bit), so the
    default token budget fits long sequences;
  * the per-sequence mean (extract.py:116-119) is reduced on the device (`esmb200_mean_pool`), `bos` is sliced on the
    device: only what was asked for crosses PCIe;
  * device->host copies go to pinned staging buffers on a side stream and are overlapped with the next batch's forward
    (two staging slots); slicing + `torch.save` run in writer threads;
  * the default token budget is larger (the reference's 4096 tokens leave an H100 idle);
  * --window N writes sequences longer than N residues whole instead of truncating them: each runs as overlapping
    windows of N residues merged with tapered weights (ProteinLanguageModel.forward_windowed); --truncation_seq_length
    is then not applied, and --include contacts is refused;
  * under torchrun the token-budget batches are dealt round-robin to the ranks, each rank writes its own files, and no
    collective is needed because the outputs are files.
"""
from __future__ import annotations

import argparse
import os
import pathlib
import queue
import threading
from typing import Dict, List, Optional

import torch

from . import pretrained
from .data import FastaBatchedDataset
from .extract import mean_pool

INCLUDE_CHOICES = ("mean", "per_tok", "bos", "contacts")


def create_parser():
    p = argparse.ArgumentParser(description="Extract per-token representations and model outputs for sequences in a FASTA file")
    p.add_argument("model_location", type=str,
                   help="ESM-2, ESM-1b or ESM-1v model name (esm2_t33_650M_UR50D, esm1b_t33_650M_UR50S, "
                        "esm1v_t33_650M_UR90S_1, ...) or a local .pt file")
    p.add_argument("fasta_file", type=pathlib.Path)
    p.add_argument("output_dir", type=pathlib.Path)
    p.add_argument("--toks_per_batch", type=int, default=65536, help="maximum batch size in tokens")
    p.add_argument("--repr_layers", type=int, default=[-1], nargs="+")
    p.add_argument("--include", type=str, nargs="+", choices=list(INCLUDE_CHOICES), required=True)
    p.add_argument("--truncation_seq_length", type=int, default=1022)
    p.add_argument("--precision", choices=["fp16", "fp32x3", "fp8"], default="fp16",
                   help="fp16: fp16 MMA operands (default); fp32x3: hi+lo operand pairs, fp32-grade results (~2.6x "
                        "slower); fp8: e4m3 QKV/fc1/fc2 projections with block scales (faster, less accurate)")
    p.add_argument("--cpu-offload", action="store_true",
                   help="keep the transformer layers' weights in pinned host memory and stream them to the GPU layer "
                        "by layer (ESM-2 15B on one GPU); same outputs")
    p.add_argument("--window", type=int, default=None,
                   help="instead of truncating, run sequences longer than this many residues as overlapping windows "
                        "merged with tapered weights (1022 fits ESM-1b / ESM-1v); not with --include contacts")
    return p


WINDOW_CONTACTS = "--include contacts cannot be combined with --window: contacts across windows are not predicted"


class FileWriter:
    """torch.save off the critical path: a bounded queue drained by a few threads (pickling releases the GIL in the
    tensor serialisation). `close()` joins and re-raises the first error."""

    def __init__(self, n_threads: int = 2, depth: int = 256):
        self._q: "queue.Queue" = queue.Queue(maxsize=depth)
        self._err: List[BaseException] = []
        self._threads = [threading.Thread(target=self._drain, daemon=True) for _ in range(n_threads)]
        for t in self._threads:
            t.start()
        self.n_written = 0
        self._lock = threading.Lock()

    def _drain(self):
        while True:
            item = self._q.get()
            if item is None:
                return
            path, obj = item
            try:
                torch.save(obj, path)
                with self._lock:
                    self.n_written += 1
            except BaseException as e:  # surfaced by close()
                self._err.append(e)

    def put(self, path, obj):
        if self._err:
            raise self._err[0]
        self._q.put((path, obj))

    def close(self) -> int:
        for _ in self._threads:
            self._q.put(None)
        for t in self._threads:
            t.join()
        if self._err:
            raise self._err[0]
        return self.n_written


class StagingSlot:
    """One pinned host arena, grown on demand and carved into tensors for a batch's device->host copies."""

    def __init__(self):
        self._buf: Optional[torch.Tensor] = None
        self._used = 0

    def reset(self, nbytes: int):
        if self._buf is None or self._buf.numel() < nbytes:
            self._buf = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=True)
        self._used = 0

    def take(self, shape, dtype=torch.float32) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= int(s)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        start = (self._used + 255) // 256 * 256
        out = self._buf[start: start + nbytes].view(dtype).view(*shape)
        self._used = start + nbytes
        return out


def plan_bytes(shapes) -> int:
    """Upper bound of the arena size for a list of (shape, element size) with 256-byte alignment per tensor."""
    total = 0
    for shape, esize in shapes:
        n = esize
        for s in shape:
            n *= int(s)
        total = (total + 255) // 256 * 256 + n
    return total + 256


class _Pending:
    """A batch whose copies are in flight: host views, the event that ends them, and the device tensors kept alive."""

    def __init__(self, labels, lengths, host: Dict[str, Dict[int, torch.Tensor]], contacts, done, keep):
        self.labels, self.lengths, self.host, self.contacts, self.done, self.keep = labels, lengths, host, contacts, done, keep


def _finalize(p: _Pending, include, out_dir: pathlib.Path, writer: FileWriter):
    p.done.synchronize()
    for i, label in enumerate(p.labels):
        n = p.lengths[i]
        result = {"label": label}
        # clone(): the saved file must hold only the slice (extract.py:104-125), and the staging arena is reused
        if "per_tok" in include:
            result["representations"] = {layer: t[i, 1: n + 1].clone() for layer, t in p.host["per_tok"].items()}
        if "mean" in include:
            result["mean_representations"] = {layer: t[i].clone() for layer, t in p.host["mean"].items()}
        if "bos" in include:
            result["bos_representations"] = {layer: t[i].clone() for layer, t in p.host["bos"].items()}
        if p.contacts is not None:
            result["contacts"] = p.contacts[i, :n, :n].clone()
        path = out_dir / f"{label}.pt"
        path.parent.mkdir(parents=True, exist_ok=True)  # labels may contain '/' (extract.py:99-101)
        writer.put(path, result)
    p.keep.clear()


def run(args) -> int:
    window = getattr(args, "window", None)
    if window is not None:
        if "contacts" in args.include:
            raise ValueError(WINDOW_CONTACTS)
        if window < 2:
            raise ValueError(f"--window must be at least 2 residues, got {window}")
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    model, alphabet = pretrained.load_model_and_alphabet(args.model_location)
    if getattr(model, "random_init", False):
        raise RuntimeError("refusing to write embeddings of a random-init model: give --model_location a checkpoint")
    model = model.eval()
    if getattr(args, "precision", "fp16") != "fp16":
        model.set_precision(args.precision)
    model = model.cpu_offload(dev) if getattr(args, "cpu_offload", False) else model.to(dev)
    n_layers = model.num_layers
    if not all(-(n_layers + 1) <= i <= n_layers for i in args.repr_layers):
        raise ValueError(f"--repr_layers must lie in [-{n_layers + 1}, {n_layers}]")
    layers = [(i + n_layers + 1) % (n_layers + 1) for i in args.repr_layers]
    include = set(args.include)
    want_contacts = "contacts" in include

    dataset = FastaBatchedDataset.from_file(args.fasta_file)
    my_batches = dataset.get_batch_indices(args.toks_per_batch, extra_toks_per_seq=1)[rank::world]
    if window is not None:
        from .windows import check_window
        check_window(model, window)
    truncation = None if window is not None else args.truncation_seq_length
    to_tokens = alphabet.get_batch_converter(truncation)
    args.output_dir.mkdir(parents=True, exist_ok=True)

    writer = FileWriter()
    copy_stream = torch.cuda.Stream(device=dev)
    slots = [StagingSlot(), StagingSlot()]
    pending: Optional[_Pending] = None
    try:
        with torch.no_grad():
            for k, idxs in enumerate(my_batches):
                labels, strs, toks = to_tokens([dataset[i] for i in idxs])
                lengths = [len(s) if truncation is None else min(truncation, len(s)) for s in strs]
                toks_dev = toks.pin_memory().to(dev, non_blocking=True)
                # contacts: the forward without the attention stack (ProteinLanguageModel._contacts_forward), so only
                # the representations and the [B,S,S] contacts stay alive with the batch while its copies run
                if window is not None:
                    out = model.forward_windowed(toks_dev, window, repr_layers=layers)
                elif want_contacts:
                    out = model._contacts_forward(toks_dev, repr_layers=layers)
                else:
                    out = model(toks_dev, repr_layers=layers)
                reps = out["representations"]
                B, T, E = next(iter(reps.values())).shape
                computed = torch.cuda.Event()
                computed.record()

                shapes = []
                for _ in layers:
                    if "per_tok" in include:
                        shapes.append(((B, T, E), 4))
                    if "mean" in include:
                        shapes.append(((B, E), 4))
                    if "bos" in include:
                        shapes.append(((B, E), 4))
                if want_contacts:
                    shapes.append((tuple(out["contacts"].shape), 4))
                slot = slots[k % 2]   # the other slot still belongs to the batch being finalised below
                slot.reset(plan_bytes(shapes))
                host: Dict[str, Dict[int, torch.Tensor]] = {"per_tok": {}, "mean": {}, "bos": {}}
                keep: list = [out, toks_dev]
                with torch.cuda.stream(copy_stream):
                    copy_stream.wait_event(computed)
                    len_dev = torch.tensor(lengths, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
                    keep.append(len_dev)
                    for layer, t in reps.items():
                        if "per_tok" in include:
                            host["per_tok"][layer] = slot.take((B, T, E)).copy_(t, non_blocking=True)
                        if "mean" in include:
                            m = mean_pool(t, len_dev)          # launched on the copy stream, after `computed`
                            keep.append(m)
                            host["mean"][layer] = slot.take((B, E)).copy_(m, non_blocking=True)
                        if "bos" in include:
                            b0 = t[:, 0].contiguous()
                            keep.append(b0)
                            host["bos"][layer] = slot.take((B, E)).copy_(b0, non_blocking=True)
                    contacts = None
                    if want_contacts:
                        contacts = slot.take(tuple(out["contacts"].shape)).copy_(out["contacts"], non_blocking=True)
                    done = torch.cuda.Event()
                    done.record(copy_stream)
                if pending is not None:      # batch k-1: its copies overlapped this batch's forward
                    _finalize(pending, include, args.output_dir, writer)
                pending = _Pending(labels, lengths, host, contacts, done, keep)
            if pending is not None:
                _finalize(pending, include, args.output_dir, writer)
    finally:
        n_written = writer.close()
    return n_written


def main():
    run(create_parser().parse_args())


if __name__ == "__main__":
    main()
