"""GPU (-m gpu): esmb200_stack_forward against its workspace and output contract, and the independence of a sequence's
result from everything but its own valid positions, in each precision (0 fp16, 1 fp32x3, 2 fp8).

  * Exact workspace: a call given exactly esmb200_workspace_bytes(...) bytes, at byte offsets 0, 16 and 1008 past a
    1024-aligned address and filled with 0xFF, writes no byte outside it, leaves no NaN in x, the representations, the
    attention maps or the contact partials (which the models hand to the user from torch.empty), and gives the same bits
    as a call with a generously sized, zero-filled workspace.  Every output sits inside its own guard bands.
  * Batch isolation: a sequence's x, representations, attention maps and contact accumulators are the same bits alone,
    at index 0 or 3 of a batch of four different sequences, and trailing-padded to T + 64.  Every fp8 scale is per row
    (activations) or per weight block, the attention walks keys up to the sequence's own last valid key (kvlen), so
    nothing of a batch-mate or of a padded position may enter.  Some sequences carry rows with a single large outlier
    column, so that their fp8 block scales differ from their neighbours'.
  * Padded-value invariance: changing x only at padded positions leaves the valid rows and the attention between valid
    positions bit-identical (the ESM-2 counterpart of tests/test_gpu_layer_split.py's axial check).

Shapes: head_dim 16 (E = 320, H = 20), 64 (E = 256, H = 4), 128 (E = 256, H = 2; fp32x3 takes head_dim <= 64 only)
and an ESM-1b layer (no rotary tables); T = 77 and 130."""
import ctypes

import pytest
import torch

import fp8_refs as fr

pytestmark = pytest.mark.gpu

NL = 2  # layers
SHAPES = {"d16": (320, 20, True), "d64": (256, 4, True), "d128": (256, 2, True), "esm1b": (256, 4, False)}
PRECISIONS = ["fp16", "fp32x3", "fp8"]
CASES = [(s, p, T) for s in SHAPES for p in range(3) for T in (77, 130) if not (s == "d128" and p == 1)]


def _lib():
    from esm_b200 import _lib
    return _lib


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def model_for(shape, precision):
    E, H, rotary = SHAPES[shape]
    if rotary:
        from esm_b200 import ESM2
        from oracle.weights import make_state_dict
        m = ESM2(num_layers=NL, embed_dim=E, attention_heads=H)
        m.load_state_dict(make_state_dict(NL, E, H, seed=E + H), strict=True)
    else:
        from argparse import Namespace
        from esm_b200 import ProteinBertModel
        torch.manual_seed(E + H)
        m = ProteinBertModel(Namespace(arch="roberta_large", layers=NL, embed_dim=E, ffn_embed_dim=4 * E,
                                       attention_heads=H, max_positions=1024, token_dropout=True,
                                       emb_layer_norm_before=True), "roberta_large")
    return m.eval().cuda().set_precision(PRECISIONS[precision])


def inputs(E, T, lengths, seed):
    """x [B, T, E] (rows with one outlier column in sequences 1 and 3), the padding mask and the contact keep mask (1
    at positions 0 .. n - 2: the last valid token plays <eos>)."""
    g = torch.Generator().manual_seed(seed)
    B = len(lengths)
    x = torch.randn(B, T, E, generator=g)
    for b in (1, 3):
        if b < B:
            rows = torch.randint(0, lengths[b], (5,), generator=g)
            cols = torch.randint(0, E, (5,), generator=g)
            x[b, rows, cols] = 200.0 * (1 + b)
    pad = torch.ones(B, T, dtype=torch.uint8)
    keep = torch.zeros(B, T, dtype=torch.uint8)
    for b, n in enumerate(lengths):
        pad[b, :n] = 0
        keep[b, :n - 1] = 1
    return x.cuda(), pad.cuda(), keep.cuda()


def run(m, x0, pad, keep, flags=1, ws_off=None):
    """One esmb200_stack_forward with every output requested.  ws_off None: a generous zero-filled workspace and
    zero-filled outputs; an int: exactly esmb200_workspace_bytes at that offset past a 1024-aligned address, 0xFF
    everywhere, every buffer inside guard bands (checked here, with the absence of NaN).  Returns the outputs."""
    L = _lib(); lib = L.load()
    B, T, E = x0.shape
    H, F = m.layers[0].self_attn.num_heads, m.layers[0].fc1.weight.shape[0]
    prec = m.layers[0].precision
    nbytes = lib.esmb200_workspace_bytes(E, H, F, B, T, prec)
    exact = ws_off is not None
    G = fr.GUARD
    if exact:
        raw = torch.full((2 * G + 2048 + nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
        base = raw.data_ptr()
        start = ((base + G + 1023) // 1024) * 1024 - base + ws_off
        ws_ptr, ws_bytes = base + start, nbytes
    else:
        raw = torch.zeros(nbytes + (1 << 20), dtype=torch.uint8, device="cuda")
        ws_ptr, ws_bytes = raw.data_ptr(), raw.numel()

    bufs = []

    def out(shape, zero=False):
        if not exact:
            return torch.zeros(shape, device="cuda")
        t, b = fr.guarded(shape, torch.float32, "cuda")
        if zero:
            t.zero_()
        bufs.append(b)
        return t

    x = out((B, T, E))
    x.copy_(x0)
    reprs = [out((B, T, E)) for _ in range(NL)]
    attn = out((B, NL, H, T, T))
    contact = prec != 1  # fp32x3 ignores the job (esmb200.h)
    lo, hi = 1, T - 1
    S, nt = hi - lo, (T + 127) // 128
    res = {}
    if contact:
        w = torch.randn(NL, H, generator=torch.Generator().manual_seed(7)).cuda()
        acc, row, col = out((B, S, S), zero=True), out((NL, B, H, 4 * nt, S)), out((NL, B, H, 4 * nt, S))
        job = L.ContactJob()
        job.weights, job.keep, job.acc, job.row_part, job.col_part = (w.data_ptr(), keep.data_ptr(), acc.data_ptr(),
                                                                      row.data_ptr(), col.data_ptr())
        job.lo, job.hi = lo, hi
        res.update(acc=acc, row=row, col=col)
    cos, sin = m._rope_tables(T)
    handles = (ctypes.c_void_p * NL)(*[layer.handle() for layer in m.layers])
    rp = (ctypes.c_void_p * NL)(*[t.data_ptr() for t in reprs])
    ap = (ctypes.c_void_p * NL)(*[attn[:, i].data_ptr() for i in range(NL)])
    L.check(lib.esmb200_stack_forward(handles, NL, P(x), P(pad), B, T, P(cos), P(sin), rp, ap, NL * H * T * T, flags,
                                      ctypes.byref(job) if contact else None, ctypes.c_void_p(ws_ptr), ws_bytes,
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    res.update(x=x, reprs=reprs, attn=attn)
    if exact:
        outside = torch.cat([raw[:start], raw[start + nbytes:]])
        assert int((outside != 0xFF).sum()) == 0, "workspace write outside esmb200_workspace_bytes"
        assert all(fr.guard_changes(b) == 0 for b in bufs), "output write outside its tensor"
        for k in ("x", "attn", "acc", "row", "col"):
            if k in res:
                assert not bool(res[k].isnan().any()), f"{k} not fully written"
        assert not any(bool(r.isnan().any()) for r in reprs), "representation not fully written"
    return res


def same(a, b):
    for k in a:
        if k == "reprs":
            assert all(torch.equal(u, v) for u, v in zip(a[k], b[k])), k
        else:
            assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("shape,precision,T", CASES, ids=[f"{s}-{PRECISIONS[p]}-T{T}" for s, p, T in CASES])
def test_exact_workspace_and_every_output_written(shape, precision, T):
    m = model_for(shape, precision)
    E = SHAPES[shape][0]
    x0, pad, keep = inputs(E, T, [T, T - 13, T // 2], seed=T + E)
    ref = {f: run(m, x0, pad, keep, flags=f) for f in (0, 1)}
    for off, flags in ((0, 1), (16, 0), (1008, 1)):
        got = run(m, x0, pad, keep, flags=flags, ws_off=off)
        same(got, ref[flags])
    print(f"PARITY stack exact workspace {shape} {PRECISIONS[precision]} T={T}: bit-identical, guards intact",
          flush=True)


def seq_view(res, b, T, n):
    """Sequence b's share of run `res`, cut to the first T positions (the contact accumulators to T - 2 crop indices:
    every entry past the keep mask is zero, checked by the caller)."""
    v = {"x": res["x"][b, :T], "attn": res["attn"][b, :, :, :T, :T]}
    for i, r in enumerate(res["reprs"]):
        v[f"repr{i}"] = r[b, :T]
    if "acc" in res:
        S, nt = T - 2, (T + 127) // 128
        v["acc"] = res["acc"][b, :S, :S]
        v["row"] = res["row"][:, b, :, :4 * nt, :S]
        v["col"] = res["col"][:, b, :, :4 * nt, :S]
    return v


def rest_is_zero(res, b, T):
    """Beyond the first T positions (crop indices T - 2) a padded sequence's maps and contact accumulators are zero."""
    a = res["attn"][b].clone()
    a[:, :, :T, :T] = 0
    assert not bool(a.any()), "attention beyond the sequence"
    if "acc" in res:
        S, nt = T - 2, (T + 127) // 128
        t = res["acc"][b].clone()
        t[:S, :S] = 0
        assert not bool(t.any()), "acc"
        for k in ("row", "col"):
            t = res[k][:, b].clone()  # [layers, H, quarters, S]
            t[:, :, :4 * nt, :S] = 0
            assert not bool(t.any()), k


@pytest.mark.parametrize("shape,precision,T", CASES, ids=[f"{s}-{PRECISIONS[p]}-T{T}" for s, p, T in CASES])
def test_batch_isolation_and_padded_values(shape, precision, T):
    m = model_for(shape, precision)
    E = SHAPES[shape][0]
    lengths = [T, T - 30, 40, T - 1]
    x0, pad, keep = inputs(E, T, lengths, seed=3 * T + E)
    fwd = run(m, x0, pad, keep)
    rev = run(m, x0.flip(0).contiguous(), pad.flip(0).contiguous(), keep.flip(0).contiguous())
    g = torch.Generator().manual_seed(T)
    for b, n in enumerate(lengths):
        want = seq_view(fwd, b, T, n)
        same(seq_view(rev, 3 - b, T, n), want)                                       # index b of 4 -> index 3 - b
        alone = run(m, x0[b:b + 1].contiguous(), pad[b:b + 1].contiguous(), keep[b:b + 1].contiguous())
        same(seq_view(alone, 0, T, n), want)                                         # alone at T
        xl = torch.cat([x0[b:b + 1], torch.randn(1, 64, E, generator=g).cuda()], 1).contiguous()
        pl = torch.cat([pad[b:b + 1], torch.ones(1, 64, dtype=torch.uint8, device="cuda")], 1).contiguous()
        kl = torch.cat([keep[b:b + 1], torch.zeros(1, 64, dtype=torch.uint8, device="cuda")], 1).contiguous()
        longer = run(m, xl, pl, kl)
        same(seq_view(longer, 0, T, n), want)                                        # trailing-padded to T + 64
        rest_is_zero(longer, 0, T)
    # padded-value invariance: x changed only at padded positions (large values, outliers included), flags 0 so that
    # the padded query rows' maps are written too; valid rows and valid x valid attention entries must not move
    x1 = x0.clone()
    noise = torch.randn(x0.shape, generator=g).cuda() * 50
    noise[:, :, 3] = 1e4
    x1 = torch.where(pad.bool()[:, :, None], noise, x1)
    a0, a1 = run(m, x0, pad, keep, flags=0), run(m, x1, pad, keep, flags=0)
    for b, n in enumerate(lengths):
        assert torch.equal(a0["x"][b, :n], a1["x"][b, :n]), b
        assert all(torch.equal(r0[b, :n], r1[b, :n]) for r0, r1 in zip(a0["reprs"], a1["reprs"])), b
        assert torch.equal(a0["attn"][b, :, :, :n, :n], a1["attn"][b, :, :, :n, :n]), b
        if "acc" in a0:
            assert torch.equal(a0["acc"][b], a1["acc"][b]), b
    print(f"PARITY stack isolation {shape} {PRECISIONS[precision]} T={T}: bit-identical alone, at index 0/3, "
          f"padded to T+64, and under padded-value changes", flush=True)
