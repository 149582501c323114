"""Host-side mirror of the reference's ESM-2 interface, dispatching the transformer-layer path to libesmb200.so.

Mirrors (same names, argument meaning, state-dict keys and result dict):
    esm.modules.TransformerLayer.forward       /root/reference/esm/modules.py:120-142
    esm.model.esm2.ESM2.__init__ / forward     /root/reference/esm/model/esm2.py:15-144
(ProteinLanguageModel holds ESM2's forward; esm_b200.esm1.ProteinBertModel, ESM-1b / ESM-1v, reuses it with learned
positions and layers built with use_rotary_embeddings=False.)
PyTorch owns parameters, activations and the workspace (torch tensors) and provides the CUDA stream; every layer's
compute goes through the C ABI in include/esmb200.h.  There is no CPU or eager fallback: on a non-CUDA tensor, or
when libesmb200.so is missing, the forward raises.

Documented deviations from the reference:
  * `TransformerLayer.forward` returns `attn=None` unless `need_head_weights=True` (the reference always computes a
    head-averaged (B,T,T) map that ESM2.forward discards, modules.py:130 / esm2.py:112-121).
  * MMA operands are fp16 (fp32 accumulate, fp32 residual stream / LayerNorm / softmax); tolerance in DESIGN.md.
  * head_dim <= 128 (every ESM-2 checkpoint); heads other than 64 wide run in zero-padded 64-wide slots (two per head
    above 64: 15B).
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence, Union

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .alphabet import Alphabet


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class RotaryEmbedding(nn.Module):
    """Holds the `inv_freq` buffer under the reference's key (rotary_embedding.py:37-41); tables are built by
    ESM2._rope_tables with the same torch ops as rotary_embedding.py:47-61."""

    def __init__(self, dim: int):
        super().__init__()
        inv_freq = 1.0 / (10000 ** (torch.arange(0, dim, 2).float() / dim))
        self.register_buffer("inv_freq", inv_freq)


class MultiheadAttention(nn.Module):
    """Parameter container with the reference's names (multihead_attention.py:109-113,130-132)."""

    def __init__(self, embed_dim: int, num_heads: int, use_rotary_embeddings: bool = True):
        super().__init__()
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.head_dim = embed_dim // num_heads
        self.k_proj = nn.Linear(embed_dim, embed_dim)
        self.v_proj = nn.Linear(embed_dim, embed_dim)
        self.q_proj = nn.Linear(embed_dim, embed_dim)
        self.out_proj = nn.Linear(embed_dim, embed_dim)
        # ESM-1b / ESM-1v layers have no rotary embedding (multihead_attention.py:126-128): no inv_freq key
        self.rot_emb = RotaryEmbedding(self.head_dim) if use_rotary_embeddings else None


def rope_tables(inv_freq: torch.Tensor, seq_len: int):
    """cos/sin [T, 32] fp32 (head_dim <= 64) or [T, 64] (head_dim <= 128) — rotary_embedding.py:53-59 (the reference's
    table is the first d/2 columns duplicated on the last dim); columns >= d/2 are padding the kernels never use."""
    inv_freq = inv_freq.float()
    t = torch.arange(seq_len, device=inv_freq.device).type_as(inv_freq)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    cos, sin = freqs.cos(), freqs.sin()
    width = 32 if cos.shape[1] <= 32 else 64
    if cos.shape[1] < width:
        pad = width - cos.shape[1]
        cos, sin = F.pad(cos, (0, pad), value=1.0), F.pad(sin, (0, pad), value=0.0)
    return cos.contiguous(), sin.contiguous()


def _f32(p: torch.Tensor) -> torch.Tensor:
    """fp32 contiguous view of a parameter (the tensor itself when it already is one)."""
    t = p.detach()
    if t.dtype != torch.float32 or not t.is_contiguous():
        t = t.float().contiguous()
    return t


class LayerBinding:
    """The esmb200_layer handle of one transformer block, built from a module that carries the reference's attribute
    names (self_attn.{q,k,v,out}_proj, self_attn_layer_norm, fc1, fc2, final_layer_norm: modules.py:99-118) — this
    repo's TransformerLayer or the reference's own esm.modules.TransformerLayer (esm_b200.integration).  Parameters that
    are not fp32 (model.half(), esmfold.py:59-62) are mirrored to fp32 copies owned by the binding; the handle is
    re-packed when a parameter is replaced or modified in place."""

    def __init__(self, module: nn.Module):
        self.module = module
        a = module.self_attn
        self.embed_dim = a.q_proj.weight.shape[1]
        self.attention_heads = a.num_heads
        self.head_dim = self.embed_dim // self.attention_heads
        self.ffn_embed_dim = module.fc1.weight.shape[0]
        if self.head_dim * self.attention_heads != self.embed_dim or self.head_dim > 128 or self.head_dim % 2:
            raise ValueError("esm_b200 supports even head_dim <= 128 (every ESM-2 model); "
                             f"got embed_dim={self.embed_dim}, heads={self.attention_heads}")
        self.precision = 0  # 0 = fp16 MMA operands, 1 = "fp32x3", 2 = "fp8" (esmb200.h: esmb200_layer_weights.precision)
        self._handle = None
        self._key = None
        self._keep = None
        # cpu_offload(): the pinned uint8 slice that holds the packed matrices (esmb200_layer_offload), and the device
        # the layer is packed and streamed to
        self.host: Optional[torch.Tensor] = None
        self.device: Optional[torch.device] = None

    # _params() positions of the vectors an esmb200_layer borrows: LayerNorms, out/fc1/fc2 biases
    _BORROWED = (0, 1, 9, 10, 11, 13, 15)

    @property
    def offloaded(self) -> bool:
        return self.host is not None

    def offload(self, device: torch.device, host: torch.Tensor) -> None:
        """Pack into `host` (pinned) on the next handle(); the layer then runs in esmb200_stack_forward_streamed."""
        self.release()
        self.device, self.host = device, host

    def end_offload(self) -> None:
        self.release()
        self.device, self.host = None, None

    def _params(self) -> List[torch.Tensor]:
        m, a = self.module, self.module.self_attn
        return [m.self_attn_layer_norm.weight, m.self_attn_layer_norm.bias, a.q_proj.weight, a.q_proj.bias,
                a.k_proj.weight, a.k_proj.bias, a.v_proj.weight, a.v_proj.bias, a.out_proj.weight, a.out_proj.bias,
                m.final_layer_norm.weight, m.final_layer_norm.bias, m.fc1.weight, m.fc1.bias, m.fc2.weight, m.fc2.bias]

    def handle(self):
        ps = self._params()
        key = (self.precision,) + tuple((p.data_ptr(), p._version, p.dtype) for p in ps)
        if self._handle is not None and key == self._key:
            return self._handle
        self.release()
        if self.host is None:
            for p in ps:
                if not p.is_cuda:
                    raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only: move the model with .cuda(); "
                                            "there is no CPU fallback")
            keep = [_f32(p) for p in ps]
        else:  # fp32 device copies of the host parameters for as long as the packing takes
            keep = [p.detach().to(self.device, torch.float32).contiguous() for p in ps]
        lib = _lib.load()
        w = _lib.LayerWeights()
        w.embed_dim, w.num_heads, w.ffn_dim = self.embed_dim, self.attention_heads, self.ffn_embed_dim
        w.head_dim = self.head_dim
        w.precision = self.precision
        w.ln_eps = self.module.self_attn_layer_norm.eps
        names = [f[0] for f in _lib.LayerWeights._fields_[4:20]]
        for n, p in zip(names, keep):
            setattr(w, n, p.data_ptr())
        out = ctypes.c_void_p()
        with torch.cuda.device(keep[0].device):
            _lib.check(lib.esmb200_layer_create(ctypes.byref(w), _stream(), ctypes.byref(out)))
            if self.host is not None:
                rc = lib.esmb200_layer_offload(out, _ptr(self.host), self.host.numel(), _stream())
                if rc:
                    lib.esmb200_layer_destroy(out)
                    _lib.check(rc)
                keep = [keep[i] for i in self._BORROWED]
        self._handle, self._key, self._keep = out, key, keep  # the library borrows LN weights and biases from `keep`
        return out

    def release(self):
        if self._handle is not None:
            _lib.load().esmb200_layer_destroy(self._handle)
            self._handle, self._key, self._keep = None, None, None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class TransformerLayer(nn.Module):
    """Pre-LN transformer block of ESM-2 (modules.py:84-142) executed by libesmb200.so.  With
    `use_rotary_embeddings=False` it is the ESM-1b / ESM-1v block (esm1.py:73-79: no bias_kv, ESM1bLayerNorm)."""

    def __init__(self, embed_dim: int, ffn_embed_dim: int, attention_heads: int, use_rotary_embeddings: bool = True):
        super().__init__()
        self.embed_dim = embed_dim
        self.ffn_embed_dim = ffn_embed_dim
        self.attention_heads = attention_heads
        self.use_rotary_embeddings = use_rotary_embeddings
        self.self_attn = MultiheadAttention(embed_dim, attention_heads, use_rotary_embeddings)
        self.self_attn_layer_norm = nn.LayerNorm(embed_dim)
        self.fc1 = nn.Linear(embed_dim, ffn_embed_dim)
        self.fc2 = nn.Linear(ffn_embed_dim, embed_dim)
        self.final_layer_norm = nn.LayerNorm(embed_dim)
        self._binding = LayerBinding(self)

    def handle(self):
        """esmb200_layer* for the current parameters."""
        return self._binding.handle()

    def release(self):
        self._binding.release()

    @property
    def precision(self) -> int:
        return self._binding.precision

    @precision.setter
    def precision(self, value: int):
        self._binding.precision = int(value)

    @property
    def offloaded(self) -> bool:
        return self._binding.offloaded

    # ---- reference-facing forward ------------------------------------------------------------------------------
    def forward(self, x, self_attn_mask=None, self_attn_padding_mask=None, need_head_weights=False):
        """x: (T, B, E) like the reference (modules.py:120-122). Returns (x (T,B,E), attn (H,B,T,T) or None)."""
        return layer_forward(self._binding, x, self_attn_mask, self_attn_padding_mask, need_head_weights)


def layer_forward(binding: LayerBinding, x, self_attn_mask=None, self_attn_padding_mask=None, need_head_weights=False):
    """TransformerLayer.forward (modules.py:120-142) through the C ABI, for any module a LayerBinding wraps."""
    if self_attn_mask is not None:
        raise NotImplementedError("ESM-2 never passes self_attn_mask (esm2.py:112-116)")
    T, B, E = x.shape
    # (B,T,E) batch-major PRIVATE copy, updated in place.  Layer 0 of the reference receives a transposed view of the
    # tensor it also returns as representations[0] (esm2.py:99-106): contiguous()/float() would hand that storage back.
    xb = torch.empty((B, T, E), dtype=torch.float32, device=x.device)
    xb.copy_(x.transpose(0, 1))
    rot = getattr(binding.module.self_attn, "rot_emb", None)
    cos, sin = rope_tables(rot.inv_freq, T) if rot is not None else (None, None)  # ESM-1b layers: no rotation
    attn = run_stack([binding], xb, self_attn_padding_mask, cos, sin, None, [0] if need_head_weights else [])
    out = xb.transpose(0, 1).to(x.dtype)
    if need_head_weights:
        return out, attn[0].transpose(0, 1).contiguous().to(x.dtype)  # (B,H,T,T) -> (H,B,T,T), multihead_attention.py:398-400
    return out, None


_workspaces: Dict[tuple, torch.Tensor] = {}


def _workspace(nbytes: int, device: torch.device) -> torch.Tensor:
    """Scratch for one stack call, cached per (device, CUDA stream): calls on different streams never share it, calls
    on one stream are ordered by the stream (the library is re-entrant across handles and streams)."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        _workspaces.pop(key, None)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


_rings: Dict[tuple, tuple] = {}


def _ring(nbytes: int, device: torch.device):
    """(ring, copy stream) of esmb200_stack_forward_streamed, cached per (device, CUDA stream) like the workspace: the
    library orders a call's copies after the work already queued on the stream, and the stream after the copies."""
    key = (device, torch.cuda.current_stream(device).cuda_stream)
    hit = _rings.get(key)
    if hit is None or hit[0].numel() < nbytes:
        copy = hit[1] if hit is not None else torch.cuda.Stream(device=device)
        _rings.pop(key, None)
        hit = (torch.empty(nbytes, dtype=torch.uint8, device=device), copy)
        _rings[key] = hit
    return hit


def run_stack(layers: Sequence, x: torch.Tensor, padding_mask: Optional[torch.Tensor],
              rope_cos: Optional[torch.Tensor], rope_sin: Optional[torch.Tensor],
              repr_out: Optional[Dict[int, torch.Tensor]], attn_layers: Sequence[int], zero_pad_rows: bool = False,
              contact_job=None, contacts_only: bool = False, probs_scratch: Optional[torch.Tensor] = None):
    """esmb200_stack_forward on x fp32 (B,T,E) in place. repr_out: {layer index (0-based): (B,T,E) tensor to fill}.
    rope_cos = rope_sin = None: layers without rotary embedding (ESM-1b / ESM-1v).
    Layers offloaded by cpu_offload() run through esmb200_stack_forward_streamed instead, with the same results.
    contacts_only: esmb200_stack_contacts with `contact_job` (ContactPredictionHead.begin_contacts) and no attention
    maps; probs_scratch is its fp32x3 scratch.
    Returns {layer index: (B,H,T,T) fp32} for the indices in attn_layers."""
    if not x.is_cuda:
        raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")
    assert x.dtype == torch.float32 and x.is_contiguous()
    lib = _lib.load()
    B, T, E = x.shape
    n = len(layers)
    Fdim, H = layers[0].ffn_embed_dim, layers[0].attention_heads
    precision = getattr(layers[0], "precision", 0)
    with torch.cuda.device(x.device):
        handles = (ctypes.c_void_p * n)(*[l.handle() for l in layers])
        nbytes = lib.esmb200_workspace_bytes(E, H, Fdim, B, T, precision)
        ws = _workspace(nbytes, x.device)
        mask = None
        if padding_mask is not None:
            mask = padding_mask.to(device=x.device, dtype=torch.uint8).contiguous()
            assert mask.shape == (B, T)
        reprs = (ctypes.c_void_p * n)()
        keep = []
        if repr_out:
            for i, t in repr_out.items():
                assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.shape == x.shape
                reprs[i] = t.data_ptr()
        attns = (ctypes.c_void_p * n)()
        attn_t = {}
        stacked = None
        if attn_layers:
            # one [B, n_attn, H, T, T] allocation, layer i written straight into its slice (esm2.py:134's stack)
            stacked = torch.empty((B, len(attn_layers), H, T, T), dtype=torch.float32, device=x.device)
            for pos, i in enumerate(attn_layers):
                a = stacked[:, pos]
                attn_t[i] = a
                attns[i] = a.data_ptr()
        keep.append(mask)
        offloaded = getattr(layers[0], "offloaded", False)
        if contacts_only:
            assert contact_job is not None and not attn_layers
            args = (handles, n, _ptr(x), _ptr(mask), B, T, _ptr(rope_cos), _ptr(rope_sin),
                    reprs if repr_out else None, ctypes.byref(contact_job), _ptr(probs_scratch),
                    probs_scratch.nbytes if probs_scratch is not None else 0, _ptr(ws), ws.numel())
            if offloaded:
                ring, copy = _ring(2 * lib.esmb200_layer_packed_bytes(E, H, Fdim, precision), x.device)
                _lib.check(lib.esmb200_stack_contacts(*args, _ptr(ring), ring.numel(),
                                                      ctypes.c_void_p(copy.cuda_stream), _stream()))
            else:
                _lib.check(lib.esmb200_stack_contacts(*args, None, 0, None, _stream()))
            return {}
        args = (handles, n, _ptr(x), _ptr(mask), B, T, _ptr(rope_cos), _ptr(rope_sin),
                reprs if repr_out else None, attns if attn_layers else None,
                (len(attn_layers) * H * T * T) if attn_layers else 0, 1 if zero_pad_rows else 0,
                ctypes.byref(contact_job) if contact_job is not None else None, _ptr(ws), ws.numel())
        if offloaded:
            ring, copy = _ring(2 * lib.esmb200_layer_packed_bytes(E, H, Fdim, precision), x.device)
            _lib.check(lib.esmb200_stack_forward_streamed(*args, _ptr(ring), ring.numel(),
                                                          ctypes.c_void_p(copy.cuda_stream), _stream()))
        else:
            _lib.check(lib.esmb200_stack_forward(*args, _stream()))
    if stacked is not None:
        attn_t["stacked"] = stacked
    return attn_t


def gelu(x):
    """modules.py:17-24"""
    return x * 0.5 * (1.0 + torch.erf(x / 1.4142135623730951))


class RobertaLMHead(nn.Module):
    """modules.py:298-314: dense -> gelu -> LayerNorm -> tied-embedding projection + bias.

    `forward(features)` is the plain PyTorch evaluation (used on already layer-normed features, e.g. by callers that
    hold a representation).  `forward_native(x_pre_ln, ln_w, ln_b, eps)` is what ESM2.forward uses on the GPU: it
    starts from the residual stream BEFORE emb_layer_norm_after and runs the whole tail through libesmb200.so
    (LayerNorm->fp16 | wgmma GEMM + bias + erf-GELU | LayerNorm->fp16 | wgmma GEMM onto the 33 tokens, padded to 64
    output columns) instead of fp32 cuBLAS + elementwise passes."""

    def __init__(self, embed_dim, output_dim, weight):
        super().__init__()
        self.dense = nn.Linear(embed_dim, embed_dim)
        self.layer_norm = nn.LayerNorm(embed_dim)
        self.weight = weight
        self.bias = nn.Parameter(torch.zeros(output_dim))
        self._packed = None
        self._packed_key = None
        self._packed_split = None

    def forward(self, features):
        x = self.dense(features)
        x = gelu(x)
        x = self.layer_norm(x)
        return F.linear(x, self.weight) + self.bias

    def _pack(self):
        ps = [self.dense.weight, self.weight, self.bias, self.dense.bias, self.layer_norm.weight, self.layer_norm.bias]
        key = tuple((p.data_ptr(), p._version, p.dtype) for p in ps)
        if self._packed is None or key != self._packed_key:
            E = self.dense.weight.shape[1]
            V = self.weight.shape[0]
            npad = (V + 63) // 64 * 64  # GEMM N must be a multiple of 64
            w_out = torch.zeros((npad, E), dtype=torch.float16, device=self.weight.device)
            w_out[:V] = self.weight.detach().half()
            b_out = torch.zeros((npad,), dtype=torch.float32, device=self.weight.device)
            b_out[:V] = self.bias.detach().float()
            self._packed = (self.dense.weight.detach().half().contiguous(), w_out, b_out, V, npad,
                            _f32(self.dense.bias), _f32(self.layer_norm.weight), _f32(self.layer_norm.bias))
            self._packed_key = key
        return self._packed

    def _pack_split(self):
        """fp32x3 operands of the two GEMMs: fp16 hi | lo halves along K (esmb200_convert_split)."""
        ps = [self.dense.weight, self.weight]
        key = tuple((p.data_ptr(), p._version, p.dtype) for p in ps)
        if self._packed_split is None or key != self._packed_split[0]:
            lib = _lib.load()
            E = self.dense.weight.shape[1]
            V = self.weight.shape[0]
            npad = (V + 63) // 64 * 64
            dev = self.weight.device
            wd32 = _f32(self.dense.weight)
            wo32 = torch.zeros((npad, E), dtype=torch.float32, device=dev)
            wo32[:V] = self.weight.detach().float()
            wd = torch.empty((E, 2 * E), dtype=torch.float16, device=dev)
            wo = torch.empty((npad, 2 * E), dtype=torch.float16, device=dev)
            _lib.check(lib.esmb200_convert_split(_ptr(wd32), _ptr(wd), E, E, _stream()))
            _lib.check(lib.esmb200_convert_split(_ptr(wo32), _ptr(wo), npad, E, _stream()))
            self._packed_split = (key, wd, wo)
        return self._packed_split[1], self._packed_split[2]

    def forward_native(self, x_pre: torch.Tensor, ln_w: torch.Tensor, ln_b: torch.Tensor, eps: float,
                       precision: int = 0) -> torch.Tensor:
        """x_pre: fp32 [B,T,E] residual stream before emb_layer_norm_after (esm2.py:123). Returns logits [B,T,V]."""
        lib = _lib.load()
        B, T, E = x_pre.shape
        M = B * T
        dev = x_pre.device
        w_dense, w_out, b_out, V, npad, b_dense, ln2_w, ln2_b = self._pack()
        if precision:  # fp32x3: the GEMM operands are fp16 hi | lo halves along K
            w_dense, w_out = self._pack_split()
            layernorm, gemm, width = lib.esmb200_layernorm_split, lib.esmb200_gemm_split, 2 * E
        else:
            layernorm, gemm, width = lib.esmb200_layernorm_f16, lib.esmb200_gemm_f16, E
        a16 = torch.empty((M, width), dtype=torch.float16, device=dev)
        _lib.check(layernorm(_ptr(x_pre), _ptr(ln_w), _ptr(ln_b), _ptr(a16), M, E, eps, _stream()))
        h = torch.empty((M, E), dtype=torch.float32, device=dev)
        _lib.check(gemm(_lib.EPI_BIAS_GELU_F32, _ptr(a16), _ptr(w_dense), _ptr(b_dense), _ptr(h), M, E, E,
                        None, None, 0, 0, _stream()))
        _lib.check(layernorm(_ptr(h), _ptr(ln2_w), _ptr(ln2_b), _ptr(a16), M, E, self.layer_norm.eps, _stream()))
        logits = torch.empty((M, npad), dtype=torch.float32, device=dev)
        _lib.check(gemm(_lib.EPI_BIAS_F32, _ptr(a16), _ptr(w_out), _ptr(b_out), _ptr(logits), M, npad, E,
                        None, None, 0, 0, _stream()))
        return logits.view(B, T, npad)[:, :, :V].contiguous()  # [B,T,V] packed like the reference's (esm2.py:129)


class ContactPredictionHead(nn.Module):
    """modules.py:317-357 (symmetrize :27-29, apc :32-41) — PyTorch; SURVEY §8f #1 lists it as a next row."""

    def __init__(self, in_features: int, prepend_bos: bool, append_eos: bool, bias=True, eos_idx: Optional[int] = None):
        super().__init__()
        self.in_features = in_features
        self.prepend_bos = prepend_bos
        self.append_eos = append_eos
        if append_eos and eos_idx is None:
            raise ValueError("Using an alphabet with eos token, but no eos token was passed in.")
        self.eos_idx = eos_idx
        self.regression = nn.Linear(in_features, 1, bias)
        self.activation = nn.Sigmoid()

    def forward(self, tokens, attentions):
        """modules.py:338-357 evaluated without the [B, L*H, S, S] temporaries of symmetrize/apc (which need ~6x the
        24 GB attention stack of configs[3]): with A_c the eos-masked, cropped map of channel c = (layer, head),
            logit_ij = sum_c w_c (A_c + A_c^T)_ij - sum_c (w_c / a12_c) a1_c[i] a1_c[j] + b,
            a1_c = rowsum(A_c) + colsum(A_c),  a12_c = sum(a1_c).
        On the GPU every layer's maps are read once by esmb200_contact_accumulate (sum over heads + row/column sums,
        no atomics: bit-reproducible) and esmb200_contact_finalize fuses the rank-(L*H) correction, the symmetrisation,
        the bias and the sigmoid."""
        B, L, H, T, _ = attentions.shape
        lo = 1 if self.prepend_bos else 0
        hi = T - 1 if self.append_eos else T
        S = hi - lo
        w = self.regression.weight.view(L, H).to(attentions.dtype)
        if not (attentions.is_cuda and attentions.dtype == torch.float32 and attentions.is_contiguous()):
            return self._forward_torch(tokens, attentions, w, lo, hi)
        lib = _lib.load()
        dev = attentions.device
        keep8 = tokens.ne(self.eos_idx).to(torch.uint8).contiguous() if self.append_eos else None
        nt = (S + 15) // 16
        acc = torch.zeros((B, S, S), dtype=torch.float32, device=dev)
        a1 = torch.empty((B, L, H, S), dtype=torch.float32, device=dev)
        row = torch.empty((B, H, S), dtype=torch.float32, device=dev)
        col = torch.empty((B, H, nt, S), dtype=torch.float32, device=dev)
        wl = w.float().contiguous()
        with torch.cuda.device(dev):
            for l in range(L):
                _lib.check(lib.esmb200_contact_accumulate(
                    ctypes.c_void_p(attentions.data_ptr() + l * H * T * T * 4), L * H * T * T,
                    ctypes.c_void_p(wl.data_ptr() + l * H * 4), _ptr(keep8), _ptr(acc), _ptr(row), _ptr(col),
                    B, H, T, lo, hi, _stream()))
                torch.add(row, col.sum(2), out=a1[:, l])               # a1_c = rowsum + colsum, fixed summation order
        return self._finalize(acc, a1.view(B, L * H, S), wl)

    def _finalize(self, acc: torch.Tensor, a1f: torch.Tensor, wl: torch.Tensor) -> torch.Tensor:
        """acc [B,S,S], a1f [B,L*H,S] (rowsum + colsum per channel), wl [L,H] -> contacts [B,S,S]."""
        lib = _lib.load()
        B, C, S = a1f.shape
        with torch.cuda.device(acc.device):
            a1f = a1f.contiguous()
            a12 = a1f.sum(-1, keepdim=True)                               # [B, L*H, 1]
            u = (a1f * (wl.reshape(1, C, 1) / a12)).contiguous()
            bias = _f32(self.regression.bias) if self.regression.bias is not None else None
            out = torch.empty((B, S, S), dtype=torch.float32, device=acc.device)
            _lib.check(lib.esmb200_contact_finalize(_ptr(acc), _ptr(u), _ptr(a1f), _ptr(bias), _ptr(out), B, C, S, _stream()))
        return out

    # ---- fused path: the accumulators are filled by esmb200_stack_forward while the probabilities are written -------
    def begin_job(self, tokens: torch.Tensor, num_layers: int, num_heads: int):
        """Buffers + esmb200_contact_job for a [B,T] batch (attention_contact.cuh); finish_job() turns them into contacts."""
        B, T = tokens.shape
        nt = (T + 127) // 128
        shape = lambda S: (num_layers, B, num_heads, 4 * nt, S)
        return self._job(tokens, num_layers, num_heads, shape, shape)

    def begin_contacts(self, tokens: torch.Tensor, num_layers: int, num_heads: int, precision: int):
        """Buffers + esmb200_contact_job for esmb200_stack_contacts (contacts without the attention stack); precision
        as esmb200_layer_weights.precision. fp16 and fp8: begin_job's. fp32x3: per layer the row sums and 16-row
        column stripes of esmb200_contact_accumulate, plus one layer's [B,H,T,T] probability scratch.
        finish_contacts() turns them into contacts."""
        if precision != 1:
            return self.begin_job(tokens, num_layers, num_heads)
        B, T = tokens.shape
        st = self._job(tokens, num_layers, num_heads, lambda S: (num_layers, B, num_heads, S),
                       lambda S: (num_layers, B, num_heads, (S + 15) // 16, S))
        st["scratch"] = torch.empty((B, num_heads, T, T), dtype=torch.float32, device=tokens.device)
        return st

    def _job(self, tokens, num_layers, num_heads, row_shape, col_shape):
        B, T = tokens.shape
        lo = 1 if self.prepend_bos else 0
        hi = T - 1 if self.append_eos else T
        S = hi - lo
        dev = tokens.device
        st = {
            "keep": tokens.ne(self.eos_idx).to(torch.uint8).contiguous() if self.append_eos else None,
            "acc": torch.zeros((B, S, S), dtype=torch.float32, device=dev),
            "row": torch.empty(row_shape(S), dtype=torch.float32, device=dev),
            "col": torch.empty(col_shape(S), dtype=torch.float32, device=dev),
            "w": _f32(self.regression.weight).view(num_layers, num_heads).contiguous(),
        }
        job = _lib.ContactJob()
        job.weights, job.keep = st["w"].data_ptr(), (st["keep"].data_ptr() if st["keep"] is not None else None)
        job.acc, job.row_part, job.col_part = st["acc"].data_ptr(), st["row"].data_ptr(), st["col"].data_ptr()
        job.lo, job.hi = lo, hi
        st["job"] = job
        return st

    def finish_job(self, st) -> torch.Tensor:
        L, B, H, _, S = st["row"].shape
        a1 = st["row"].sum(3) + st["col"].sum(3)                          # [L,B,H,S], fixed summation order
        return self._finalize(st["acc"], a1.permute(1, 0, 2, 3).reshape(B, L * H, S), st["w"])

    def finish_contacts(self, st) -> torch.Tensor:
        """Contacts from begin_contacts' buffers once esmb200_stack_contacts has filled them."""
        if st["row"].dim() == 5:
            return self.finish_job(st)
        L, B, H, S = st["row"].shape  # fp32x3: a1 exactly as forward() builds it from the per-layer accumulations
        a1 = torch.empty((B, L, H, S), dtype=torch.float32, device=st["acc"].device)
        for l in range(L):
            torch.add(st["row"][l], st["col"][l].sum(2), out=a1[:, l])
        return self._finalize(st["acc"], a1.view(B, L * H, S), st["w"])

    def _forward_torch(self, tokens, attentions, w, lo, hi):
        """The same formula with PyTorch ops (non-CUDA or non-fp32 inputs; cross-check in the tests)."""
        B, L, H, T, _ = attentions.shape
        S = hi - lo
        keep = None
        if self.append_eos:
            keep = tokens.ne(self.eos_idx).to(attentions)[:, lo:hi]  # [B,S]
        acc = torch.zeros((B, S, S), dtype=attentions.dtype, device=attentions.device)
        corr = torch.zeros_like(acc)
        for l in range(L):
            a = attentions[:, l, :, lo:hi, lo:hi]  # [B,H,S,S] view
            if keep is not None:
                a = a * (keep[:, None, :, None] * keep[:, None, None, :])
            acc += torch.einsum("bhij,h->bij", a, w[l])
            a1 = a.sum(-1) + a.sum(-2)  # [B,H,S]
            a12 = a1.sum(-1)            # [B,H]
            corr += torch.einsum("bhi,bhj->bij", a1 * (w[l][None, :] / a12)[:, :, None], a1)
        logits = acc + acc.transpose(-1, -2) - corr
        if self.regression.bias is not None:
            logits = logits + self.regression.bias
        return self.activation(logits)


class ProteinLanguageModel(nn.Module):
    """The forward path ESM2 and ProteinBertModel (ESM-1b / ESM-1v, esm_b200.esm1) share: embedding prologue (`_embed`)
    -> one esmb200_stack_forward (rotary tables from `_rope_tables`, or none) with the contact job fused -> LM head from
    the pre-LN stream -> final LayerNorm.  The two models differ only in those two hooks and their constructors."""

    def _init_encoder(self, num_layers: int, embed_dim: int, attention_heads: int, ffn_embed_dim: int,
                      alphabet: Union[Alphabet, str], token_dropout: bool, use_rotary_embeddings: bool):
        self.num_layers = num_layers
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        if isinstance(alphabet, str):
            alphabet = Alphabet.from_architecture(alphabet)
        self.alphabet = alphabet
        self.alphabet_size = len(alphabet)
        self.padding_idx = alphabet.padding_idx
        self.mask_idx = alphabet.mask_idx
        self.cls_idx = alphabet.cls_idx
        self.eos_idx = alphabet.eos_idx
        self.prepend_bos = alphabet.prepend_bos
        self.append_eos = alphabet.append_eos
        self.token_dropout = token_dropout
        self.embed_scale = 1
        self.embed_tokens = nn.Embedding(self.alphabet_size, embed_dim, padding_idx=self.padding_idx)
        self.layers = nn.ModuleList(
            [TransformerLayer(embed_dim, ffn_embed_dim, attention_heads, use_rotary_embeddings)
             for _ in range(num_layers)])
        self.contact_head = ContactPredictionHead(num_layers * attention_heads, self.prepend_bos, self.append_eos,
                                                  eos_idx=self.eos_idx)

    def _init_head(self, embed_dim: int):
        self.emb_layer_norm_after = nn.LayerNorm(embed_dim)
        self.lm_head = RobertaLMHead(embed_dim, self.alphabet_size, self.embed_tokens.weight)
        self._mirrors: Dict[str, tuple] = {}
        self.precision = "fp16"
        self._offload = None  # cpu_offload(): (device, pinned arena)

    PRECISIONS = {"fp16": 0, "fp32x3": 1}  # the precisions the MSA Transformer shares
    # every precision of the ESM-2 / ESM-1b layer stack (esmb200_layer_weights.precision): PRECISIONS and "fp8"
    LAYER_PRECISIONS = {**PRECISIONS, "fp8": 2}

    def cpu_offload(self, device=None) -> "ProteinLanguageModel":
        """Run on `device` (default: the current CUDA device) with the transformer layers' weights in host memory, the
        way the reference runs ESM-2 15B on one GPU (examples/esm2_infer_fairscale_fsdp_cpu_offloading.py,
        scripts/fold.py --cpu-offload).  The layers' parameters stay on the host, in any dtype; every other module moves
        to `device`.  Each distinct layer is packed once by the library (its parameters staged on the device as fp32
        one layer at a time) and its fp16 matrices moved into one pinned host arena.  From then on every forward
        streams them to the device through a two-slot ring, the copy of layer i + 1 overlapping the kernels of layer i,
        with results bit-identical to the resident model.  At 15B the device then holds two layers' matrices (1.26 GB)
        instead of 30 GB.  set_precision() and in-place changes of a host parameter re-pack as usual; model.cuda(),
        .to() or any other module conversion ends the mode and frees the arena."""
        if self.precision == "fp8":
            raise _lib.Esmb200Error("cpu_offload() streams fp16 or fp32x3 layers; fp8 layers stay resident")
        if not torch.cuda.is_available():
            raise _lib.Esmb200Error("cpu_offload() streams the layers to a CUDA (sm_90a) device; none is available")
        device = torch.device("cuda") if device is None else torch.device(device)
        if device.type != "cuda":
            raise _lib.Esmb200Error(f"cpu_offload() needs a CUDA device, got {device}")
        if device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        lib = _lib.load()
        self._end_offload()
        for name, child in self.named_children():
            if name != "layers":
                child.to(device)
        layers = list({id(l): l for l in self.layers}.values())  # a module repeated in the list is packed once
        for layer in layers:
            layer.cpu()
            if layer.self_attn.rot_emb is not None:  # rope tables are built on the device
                layer.self_attn.rot_emb.to(device)
        nbytes = lib.esmb200_layer_packed_bytes(self.embed_dim, self.attention_heads, layers[0].ffn_embed_dim,
                                                self.LAYER_PRECISIONS[self.precision])
        # one arena: torch's pinned allocator rounds every allocation up to a power of two
        arena = torch.empty(len(layers) * nbytes, dtype=torch.uint8, pin_memory=True)
        self._offload = (device, arena)
        for i, layer in enumerate(layers):
            layer._binding.offload(device, arena[i * nbytes:(i + 1) * nbytes])
            layer.handle()
        torch.cuda.empty_cache()  # return the fp32 staging of the packing to the device
        return self

    def _end_offload(self) -> None:
        if getattr(self, "_offload", None) is None:
            return
        torch.cuda.synchronize(self._offload[0])  # a streamed forward may still be copying from the arena
        for layer in self.layers:
            layer._binding.end_offload()
        self._offload = None

    def _apply(self, fn, *args, **kwargs):
        self._end_offload()  # model.cuda() / .to() / .half() after cpu_offload(): the resident path again
        return super()._apply(fn, *args, **kwargs)

    def set_precision(self, name: str) -> "ProteinLanguageModel":
        """"fp16" (default): fp16 MMA operands, fp32 accumulation — the fast path bench.py measures.
        "fp32x3": every MMA operand (LayerNorm output, weights, q, k, v, softmax probabilities, context, FFN hidden) is
        an fp16 hi + lo pair and every product runs hi*hi + lo*hi + hi*lo into the fp32 accumulator: 22 significand bits
        per operand, fp32-grade parity with the reference at ~3x the tensor work (DESIGN.md section 4).  Needs
        embed_dim % 64 == 0.
        "fp8": the QKV, fc1 and fc2 projections run e4m3 GEMMs with power-of-two block scales (activations one per row
        and 128 columns, weights one per 128 x 128 block) and fp32 accumulation; attention, out_proj, LayerNorm
        statistics, the residual stream and the LM head stay as in "fp16" (DESIGN.md section 4).  Not available on a
        cpu_offload() model."""
        ids = ProteinLanguageModel.LAYER_PRECISIONS
        if name not in ids:
            raise ValueError(f"precision must be one of {sorted(ids)}")
        if name == "fp8" and self._offload is not None:
            raise _lib.Esmb200Error("fp8 layers cannot be streamed from host memory: undo cpu_offload() (model.cuda()) "
                                    "first")
        if name == "fp32x3" and (self.embed_dim % 64 != 0 or self.embed_dim // self.attention_heads > 64):
            raise ValueError("fp32x3 precision needs embed_dim % 64 == 0 and head_dim <= 64")
        changed = name != self.precision
        self.precision = name
        for layer in self.layers:
            layer.precision = ids[name]
        if changed and self._offload is not None:
            self.cpu_offload(self._offload[0])  # the packed size depends on the precision: a new arena
        return self

    def _rope_tables(self, T: int):
        """(cos, sin) tables for esmb200_stack_forward, or (None, None) for layers without rotary embedding."""
        raise NotImplementedError

    def _embed(self, tokens: torch.Tensor, x: torch.Tensor) -> None:
        """Embedding prologue: fill the fp32 residual stream x [B,T,E] from tokens [B,T] (int64, contiguous)."""
        raise NotImplementedError

    def _mirror(self, name: str, p: torch.Tensor) -> torch.Tensor:
        """fp32 mirror of a non-fp32 parameter (model.half()), cached until the parameter changes."""
        if p.dtype == torch.float32 and p.is_contiguous():
            return p.detach()
        key = (p.data_ptr(), p._version, p.dtype)
        hit = self._mirrors.get(name)
        if hit is None or hit[0] != key:
            hit = (key, _f32(p))
            self._mirrors[name] = hit
        return hit[1]

    def _stack(self, tokens, repr_layers=frozenset(), need_head_weights=False, return_contacts=False,
               cast=lambda t: t, contacts_only=False):
        """The stack step of `forward` (esm2.py:82-121): embedding prologue and one esmb200_stack_forward.
        Returns (tokens int64 contiguous, x, hidden, attn_t, cjob): x is the fp32 residual stream [B,T,E] BEFORE
        emb_layer_norm_after, hidden {i: cast(representation)} for the requested layers below num_layers, attn_t
        run_stack's attention maps, cjob the fused contact job or None.  Runs under torch.cuda.device(tokens.device).
        contacts_only: esmb200_stack_contacts instead, no attention maps; cjob is begin_contacts' job."""
        assert tokens.ndim == 2
        if not tokens.is_cuda:
            raise _lib.Esmb200Error("esm_b200 runs on CUDA (sm_90a) only: pass tokens.cuda(); no CPU fallback")
        _lib.load()
        if tokens.dtype != torch.int64:
            if tokens.dtype.is_floating_point or tokens.dtype == torch.bool:
                raise TypeError(f"tokens must be an integer tensor, got {tokens.dtype}")
            tokens = tokens.long()
        tokens = tokens.contiguous()
        # nn.Embedding raises a device-side assert on an out-of-range id (esm2.py:84); same here, without a host sync
        torch._assert_async(((tokens >= 0) & (tokens < self.alphabet_size)).all())
        B, T = tokens.shape
        E, N = self.embed_dim, self.num_layers
        padding_mask = tokens.eq(self.padding_idx)  # esm2.py:82
        hidden: Dict[int, torch.Tensor] = {}

        with torch.cuda.device(tokens.device):
            x = torch.empty((B, T, E), dtype=torch.float32, device=tokens.device)
            self._embed(tokens, x)
            if 0 in repr_layers:
                hidden[0] = cast(x.clone())
            # esm2.py:108-109 drops the mask when the batch has no padding; that test is a device->host sync, which
            # would serialise back-to-back forwards (bulk extraction). The kernels take the all-false mask at no cost
            # (one uniform compare per 32 keys), so the mask is always passed.
            mask = padding_mask
            # esm2.py:111-121 layer loop (intermediate representations are copied out by the library)
            repr_out = {i - 1: torch.empty_like(x) for i in repr_layers if 0 < i < N}
            cos, sin = self._rope_tables(T)
            # contacts: folded into the probability pass (fp16 and fp8 modes, whose attention is the fp16 kernel; fp32x3
            # runs the separate kernels afterwards)
            if contacts_only:
                cjob = self.contact_head.begin_contacts(tokens, N, self.attention_heads,
                                                        self.LAYER_PRECISIONS[self.precision])
                attn_t = run_stack(list(self.layers), x, mask, cos, sin, repr_out, [], zero_pad_rows=True,
                                   contact_job=cjob["job"], contacts_only=True, probs_scratch=cjob.pop("scratch", None))
            else:
                cjob = (self.contact_head.begin_job(tokens, N, self.attention_heads)
                        if return_contacts and self.precision in ("fp16", "fp8") else None)
                attn_t = run_stack(list(self.layers), x, mask, cos, sin, repr_out,
                                   list(range(N)) if need_head_weights else [], zero_pad_rows=True,
                                   contact_job=cjob["job"] if cjob else None)
            for i, t in repr_out.items():
                hidden[i + 1] = cast(t)
        return tokens, x, hidden, attn_t, cjob

    def _lm_head_rows(self, x_rows: torch.Tensor) -> torch.Tensor:
        """The LM head (esm2.py:123,129) on selected rows [n,E] of the pre-LN stream: fp32 logits [n,V], also after
        model.half()."""
        ln = self.emb_layer_norm_after
        ln_w, ln_b = self._mirror("ln_after.w", ln.weight), self._mirror("ln_after.b", ln.bias)
        return self.lm_head.forward_native(x_rows.unsqueeze(0), ln_w, ln_b, ln.eps, self._lm_head_precision())[0]

    def _lm_head_precision(self) -> int:
        """RobertaLMHead.forward_native's precision id: 1 for fp32x3, else 0 (the fp8 mode's head runs fp16)."""
        return int(self.precision == "fp32x3")

    @torch.no_grad()
    def forward(self, tokens, repr_layers=[], need_head_weights=False, return_contacts=False):
        if return_contacts:
            need_head_weights = True
        dtype = self.embed_tokens.weight.dtype  # fp32, or fp16/bf16 after model.half() (esmfold.py:59-62)
        repr_layers = set(repr_layers)
        cast = (lambda t: t) if dtype == torch.float32 else (lambda t: t.to(dtype))
        tokens, x, hidden, attn_t, cjob = self._stack(tokens, repr_layers, need_head_weights, return_contacts, cast)
        lib = _lib.load()
        B, T = tokens.shape
        E, N = self.embed_dim, self.num_layers

        with torch.cuda.device(tokens.device):
            # esm2.py:129 LM head, from the pre-LN stream (its first step is the same emb_layer_norm_after)
            ln = self.emb_layer_norm_after
            ln_w, ln_b = self._mirror("ln_after.w", ln.weight), self._mirror("ln_after.b", ln.bias)
            logits = cast(self.lm_head.forward_native(x, ln_w, ln_b, ln.eps, self._lm_head_precision()))
            # esm2.py:123-128 final LayerNorm; the last representation is post-LN
            _lib.check(lib.esmb200_layernorm(_ptr(x), _ptr(ln_w), _ptr(ln_b), _ptr(x), B * T, E, ln.eps, _stream()))
        if N in repr_layers:
            hidden[N] = cast(x)
        result = {"logits": logits, "representations": hidden}
        if need_head_weights:
            # B x L x H x T x T (esm2.py:134), each layer written in place by the library; rows/columns of padded
            # tokens are already zero (esm2.py:135-139: padded keys have probability 0, padded query rows are zeroed
            # by the probability kernel), so no masking pass over the stack is needed
            attentions = attn_t["stacked"]
            result["attentions"] = cast(attentions)
            if return_contacts:
                contacts = self.contact_head.finish_job(cjob) if cjob else self.contact_head(tokens, attentions)
                result["contacts"] = cast(contacts)
        return result

    @torch.no_grad()
    def forward_windowed(self, tokens, window: int, repr_layers=(), max_tokens: Optional[int] = None):
        """forward(tokens, repr_layers) for proteins of any length: each row of tokens [B, T] (right-padded) runs as
        overlapping windows of `window` residues, merged by the rule of esm_b200.windows. Returns {"logits": [B,T,V],
        "representations": {layer: [B,T,E]}} (the last layer post-LN, as forward returns it; pad rows zero). The
        windows of all rows form one batch, padded only where a protein is shorter than the window, and run through
        the stack in chunks of at most `max_tokens` tokens (at least one window per chunk; the result does not depend
        on it). A protein of at most `window` residues gets forward's rows bit for bit. No attention maps or
        contacts."""
        dtype = self.embed_tokens.weight.dtype
        out = self._windowed(tokens, window, repr_layers, max_tokens)
        if dtype == torch.float32:
            return out
        return {"logits": out["logits"].to(dtype),
                "representations": {i: t.to(dtype) for i, t in out["representations"].items()}}

    def _windowed(self, tokens, window: int, repr_layers=(), max_tokens: Optional[int] = None):
        """forward_windowed in fp32 whatever the parameters' dtype (the variant scorers' logits)."""
        from . import windows
        from .variants import _copies_per_chunk
        W = windows.check_window(self, window)
        dev = self.embed_tokens.weight.device
        tokens = torch.as_tensor(tokens)
        if tokens.dim() != 2:
            raise ValueError("tokens must be [B, T]")
        if tokens.dtype.is_floating_point or tokens.dtype == torch.bool:
            raise TypeError(f"tokens must be an integer tensor, got {tokens.dtype}")
        B, T = tokens.shape
        E, N, V = self.embed_dim, self.num_layers, self.alphabet_size
        layers = sorted(i for i in set(repr_layers) if 0 <= i <= N)
        bos, eos = int(self.prepend_bos), int(self.append_eos)
        host = tokens.cpu().long()
        Tw = min(T, W + bos + eos)
        gather, out_rows, src_rows, weights = [], [], [], []
        nw = 0
        # a protein ends at its last non-pad token (a <pad> inside it stays in its window, as forward keeps it)
        keep = host.ne(self.padding_idx)
        extent = torch.where(keep.any(1), T - keep.flip(1).int().argmax(1), 0)
        for b, n in enumerate((extent - bos - eos).tolist()):
            plan = windows.Plan(max(n, 0), W, bos, eos)
            gather.append(plan.gather(T, Tw) + b * (T + 1))
            pos, win, row, w = plan.terms()
            out_rows.append(b * T + pos)
            src_rows.append((nw + win) * Tw + row)
            weights.append(w)
            nw += plan.K
        ext = torch.cat([host, torch.full((B, 1), self.padding_idx, dtype=torch.int64)], 1).view(-1)
        wtok = ext[torch.cat(gather)].to(dev)  # [nw, Tw]
        logits = torch.empty((nw, Tw, V), dtype=torch.float32, device=dev)
        reps = {i: torch.empty((nw, Tw, E), dtype=torch.float32, device=dev) for i in layers}
        per = _copies_per_chunk(Tw, max_tokens)
        ln = self.emb_layer_norm_after
        for s in range(0, nw, per):
            _, x, hidden, _, _ = self._stack(wtok[s:s + per], set(layers))
            with torch.cuda.device(dev):
                logits[s:s + per] = self._lm_head_rows(x.view(-1, E)).view(-1, Tw, V)
                for i, t in hidden.items():
                    reps[i][s:s + per] = t
                if N in reps:  # esm2.py:123-128 final LayerNorm, as forward applies it
                    ln_w, ln_b = self._mirror("ln_after.w", ln.weight), self._mirror("ln_after.b", ln.bias)
                    _lib.check(_lib.load().esmb200_layernorm(_ptr(x), _ptr(ln_w), _ptr(ln_b), _ptr(x), x.shape[0] * Tw,
                                                             E, ln.eps, _stream()))
                    reps[N][s:s + per] = x
        out_rows = torch.cat(out_rows)
        idx, w, seg = torch.cat(src_rows), torch.cat(weights), windows.segments(out_rows, B * T)
        merge = lambda src, C: windows.merge_rows(src.view(-1, C), idx, w, seg).view(B, T, C)
        return {"logits": merge(logits, V), "representations": {i: merge(t, E) for i, t in reps.items()}}

    def predict_contacts(self, tokens):
        """forward(tokens, return_contacts=True)["contacts"], bit for bit, without the [B,L,H,T,T] attention stack:
        its peak memory is the contact partials (about 1/16 of the stack) instead of the stack."""
        return self._contacts_forward(tokens)["contacts"]

    @torch.no_grad()
    def _contacts_forward(self, tokens, repr_layers=()):
        """forward(tokens, repr_layers, return_contacts=True) without the attention stack and the LM head:
        {"representations", "contacts"}, each bit-identical to forward's (the last layer post-LN, every tensor in
        forward's dtype). Runs esmb200_stack_contacts (esmb200_stack_forward's layer loop, store-free contact pass)."""
        dtype = self.embed_tokens.weight.dtype
        repr_layers = set(repr_layers)
        cast = (lambda t: t) if dtype == torch.float32 else (lambda t: t.to(dtype))
        tokens, x, hidden, _, cjob = self._stack(tokens, repr_layers, cast=cast, contacts_only=True)
        B, T = tokens.shape
        E, N = self.embed_dim, self.num_layers
        with torch.cuda.device(tokens.device):
            contacts = cast(self.contact_head.finish_contacts(cjob))
            if N in repr_layers:  # esm2.py:123-128 final LayerNorm, as forward applies it
                ln = self.emb_layer_norm_after
                ln_w, ln_b = self._mirror("ln_after.w", ln.weight), self._mirror("ln_after.b", ln.bias)
                _lib.check(_lib.load().esmb200_layernorm(_ptr(x), _ptr(ln_w), _ptr(ln_b), _ptr(x), B * T, E, ln.eps,
                                                         _stream()))
                hidden[N] = cast(x)
        return {"representations": hidden, "contacts": contacts}


class ESM2(ProteinLanguageModel):
    """Drop-in for esm.model.esm2.ESM2 (esm2.py:14-147): same constructor, same state-dict keys (so
    `load_state_dict(reference_model.state_dict())` and the esm2_t*.pt checkpoints load), same forward contract."""

    def __init__(self, num_layers: int = 33, embed_dim: int = 1280, attention_heads: int = 20,
                 alphabet: Union[Alphabet, str] = "ESM-1b", token_dropout: bool = True):
        super().__init__()
        self._init_encoder(num_layers, embed_dim, attention_heads, 4 * embed_dim, alphabet, token_dropout, True)
        self._init_head(embed_dim)
        self._rope_cache = None

    def _rope_tables(self, T: int):
        inv = self.layers[0].self_attn.rot_emb.inv_freq
        key = (T, inv.device, inv.data_ptr())
        if self._rope_cache is None or self._rope_cache[0] != key:
            self._rope_cache = (key,) + rope_tables(inv, T)
        return self._rope_cache[1], self._rope_cache[2]

    def _embed(self, tokens: torch.Tensor, x: torch.Tensor) -> None:
        """esm2.py:84-95"""
        B, T, E = x.shape
        table = self._mirror("embed_tokens", self.embed_tokens.weight)
        _lib.check(_lib.load().esmb200_embed_tokens(_ptr(tokens), _ptr(table), _ptr(x), B, T, E, self.padding_idx,
                                                    self.mask_idx, int(self.token_dropout), _stream()))
