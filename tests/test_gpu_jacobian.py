"""GPU: the categorical Jacobian (esm_b200.jacobian, esmb200_jacobian_contacts).

  1. the contact kernel against the float64 definition on the same fp32 J, element-wise within a bound derived from
     the summation lengths, at every tile and grid edge of its kernels, with a large term constant along each centred
     axis, and past 2^31 elements of J, the output and scratch poisoned first; an all-zero J; bit-reproducibility;
  2. batching is exact: J equals a loop of the public forward, for every max_tokens, and identity copies give f_wt;
  3. against the unmodified reference (oracle/_ref) in float64 on the CPU;
  4. cpu_offload() and model.half();
  5. full size: 650M, L = 200;
  6. the command line end to end.
Every gated comparison prints a PARITY line.
"""
import argparse
import math
import os
import sys
import tempfile

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # jacobian_refs, variant_fixtures, esm1b_weights

from jacobian_refs import contacts_f64, contacts_f64_chunked  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
AA = "LAGVSERTIDPKQNFYMHWC"
U32 = 2.0 ** -24  # fp32 unit roundoff: the output rounding
U64 = 2.0 ** -53  # fp64 unit roundoff: every sum of the kernel


# ---- 1. the kernel against float64 --------------------------------------------------------------------------------
# A term constant along the named axes, 100x the substitution effects: the centring along them must cancel it.
OFFSET_SHAPES = {"i,a": lambda L: (1, 1, L, 20), "i": lambda L: (1, 20, L, 20), "a": lambda L: (L, 1, L, 20),
                 "j": lambda L: (L, 20, 1, 20), "b": lambda L: (L, 20, L, 1)}


def _random_jac(L, seed, offset=0.0, axes="i,a"):
    g = torch.Generator(device="cuda").manual_seed(seed)
    jac = torch.randn((L, 20, L, 20), device="cuda", generator=g).mul_(8)
    if offset:
        jac += torch.randn(OFFSET_SHAPES[axes](L), device="cuda", generator=g) * offset
    return jac


def _poisoned_contacts(jac):
    """esmb200_jacobian_contacts through the C ABI with the output filled with NaN and the scratch with 0xFF bytes
    (NaN as fp64), so that an entry no kernel writes, or a scratch value read before it is written, shows."""
    from esm_b200 import _lib
    lib = _lib.load()
    L = jac.shape[0]
    n = lib.esmb200_jacobian_scratch_bytes(L)
    scratch = torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda")
    out = torch.full((L, L), float("nan"), device="cuda")
    _lib.check(lib.esmb200_jacobian_contacts(jac.data_ptr(), L, scratch.data_ptr(), n, out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream))
    return out


def _gate(C, jac, label, rows=None):
    """C [L,L] from the kernel against contacts_f64 on the same fp32 J (contacts_f64_chunked in slabs of `rows` values
    of i, when given). The kernel reads J exactly into fp64 and takes every sum there: S_i and S_j over L terms, S over
    L^2, a block's centring and norm over 20 and 400, the APC sums over L and L^2. A sequential sum of n terms is off by
    at most n U64 times the sum of their magnitudes, so relative to max|J| (the marginals and the centred block) and
    max N (the APC terms) every step stays within (L^2 + 400) U64, a few such steps compose, hence
    64 (L^2 + 400) U64 (max|J| + max N). The output rounding adds U32 |C|. The bound must be no looser than
    1e-5 max N."""
    L = jac.shape[0]
    if rows is None:
        want = contacts_f64(jac)
        jmax = float(jac.abs().max())
        jc = jac.double()
        for axis in range(4):
            jc = jc - jc.mean(axis, keepdim=True)
        nmax = float(jc.pow(2).sum((1, 3)).sqrt().max())
        del jc
    else:
        want, nmax, jmax = contacts_f64_chunked(jac, rows)
    f64 = 64 * (L * L + 400) * U64 * (jmax + nmax)
    bound = U32 * want.abs() + f64
    err = (C.double() - want).abs()
    worst = float((err / bound).max())
    print(f"PARITY jacobian_contacts {label} L={L}: max_abs_err={float(err.max()):.3e} max N={nmax:.4g} "
          f"max|C|={float(want.abs().max()):.4g} err/bound={worst:.3e} bound/maxN={float(bound.max()) / nmax:.3e}")
    assert float(bound.max()) <= 1e-5 * nmax
    assert worst <= 1.0  # also false for a NaN


# 15, 16: pass 1's 16-row staging; 63, 65, 129: its 64-wide j tiles; 255, 256, 257: the 256-column blocks of the APC
# sums; 512, 513: exactly the APC kernel's 1024 blocks, and one row past them (its grid-stride loop)
@pytest.mark.parametrize("L", [2, 3, 15, 16, 17, 63, 64, 65, 129, 255, 256, 257, 300, 512, 513, 1022])
def test_contact_kernel_matches_float64(L):
    from esm_b200 import jacobian
    jac = _random_jac(L, seed=L)
    before = jac.clone()
    C = _poisoned_contacts(jac)
    assert torch.equal(jac, before), "J must be read only"
    _gate(C, jac, "random")
    got = jacobian.jacobian_contacts(jac)
    assert got.dtype == torch.float32 and got.shape == (L, L)
    assert torch.equal(got, C), "two runs must be bit-identical"


@pytest.mark.parametrize("axes", list(OFFSET_SHAPES))
@pytest.mark.parametrize("L", [17, 300])
def test_contact_kernel_cancels_a_large_common_offset(L, axes):
    """A term constant along `axes` only (a wild-type-like term per (j, b) for "i,a"), 100x the substitution effects:
    the fp64 centring along those axes must cancel it."""
    jac = _random_jac(L, seed=100 + L + 1000 * list(OFFSET_SHAPES).index(axes), offset=800.0, axes=axes)
    _gate(_poisoned_contacts(jac), jac, f"offset along {axes}")


def test_contact_kernel_past_2_31_jacobian_elements():
    """L = 2400: J holds 2.30e9 elements (9.2 GB), so an index formed in 32 bits anywhere would go wrong. The float64
    reference is taken one 64-row slab of i at a time; the peak is J, the scratch and one slab's float64 copies."""
    import time
    L = 2400
    assert L * 20 * L * 20 > 2 ** 31
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    jac = _random_jac(L, seed=L)
    C = _poisoned_contacts(jac)
    _gate(C, jac, "random past 2^31 elements", rows=64)
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 1e9
    print(f"PARITY jacobian_contacts L={L}: J {jac.numel() / 1e9:.2f}e9 elements, peak {peak:.1f} GB, "
          f"wall {time.perf_counter() - t0:.1f} s")
    assert peak <= jac.numel() * 4 / 1e9 + 4


def test_contact_kernel_all_zero_jacobian_is_nan_where_the_definition_is():
    from esm_b200 import jacobian
    jac = torch.zeros((5, 20, 5, 20), device="cuda")
    C = jacobian.jacobian_contacts(jac).cpu()
    want = contacts_f64(jac).cpu()
    off = ~torch.eye(5, dtype=torch.bool)
    print(f"PARITY jacobian_contacts zero L=5: NaN off the diagonal {bool(C[off].isnan().all())}")
    assert bool(want[off].isnan().all()) and bool(C[off].isnan().all())
    assert bool((C.diagonal() == 0).all()) and bool((want.diagonal() == 0).all())


def test_contact_kernel_argument_checks():
    from esm_b200 import _lib
    lib = _lib.load()
    jac = torch.zeros((4, 20, 4, 20), device="cuda")
    out = torch.empty((4, 4), device="cuda")
    n = lib.esmb200_jacobian_scratch_bytes(4)
    scratch = torch.empty(n, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert lib.esmb200_jacobian_contacts(jac.data_ptr(), 1, scratch.data_ptr(), n, out.data_ptr(), s) == -1
    assert lib.esmb200_jacobian_contacts(jac.data_ptr(), 4, scratch.data_ptr(), n - 1, out.data_ptr(), s) == -1
    assert lib.esmb200_jacobian_contacts(None, 4, scratch.data_ptr(), n, out.data_ptr(), s) == -1
    assert lib.esmb200_jacobian_contacts(jac.data_ptr(), 4, scratch.data_ptr(), n, out.data_ptr(), s) == 0


# ---- fixture models -----------------------------------------------------------------------------------------------
def _protein(n, seed):
    g = torch.Generator().manual_seed(seed)
    seq = [AA[int(k)] for k in torch.randint(0, 20, (n,), generator=g)]
    seq[n // 3] = "X"  # a non-canonical wild type: all 20 copies run there
    return "".join(seq)


def _fixture_model(name, tmp):
    import variant_fixtures as vf
    from esm_b200 import pretrained
    model, alphabet = pretrained.load_model_and_alphabet(vf.write_checkpoint(name, vf.MODELS[name], tmp))
    return model.eval(), alphabet


@pytest.fixture(scope="module")
def fixtures():
    with tempfile.TemporaryDirectory() as tmp:
        yield {n: _fixture_model(n, tmp) for n in ("esm2_t2_tiny", "esm1b_t2_tiny")}


# ---- 2. batching is exact -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", [("esm2_t2_tiny", 48), ("esm1b_t2_tiny", 61)])
def test_jacobian_equals_the_public_forward_for_every_chunk_size(fixtures, name, n):
    from esm_b200 import jacobian
    model, alphabet = fixtures[name]
    model = model.cuda()
    tokens = alphabet.get_batch_converter()([("p", _protein(n, seed=n))])[2].cuda()
    T, L = tokens.shape[1], n
    out = jacobian.categorical_jacobian(model, tokens, max_tokens=1 << 30, return_jacobian=True)
    J = out["jacobian"]
    assert J.shape == (L, 20, L, 20) and J.dtype == torch.float32
    assert out["contacts"].shape == (L, L) and out["contacts"].dtype == torch.float32
    assert torch.equal(out["contacts"], jacobian.jacobian_contacts(J))
    wt = model(tokens)["logits"][0, 1:L + 1, 4:24]
    mismatches, identities = 0, 0
    for i in range(L):
        for a in range(20):
            if int(tokens[0, 1 + i]) == 4 + a:
                identities += 1
                assert bool((J[i, a] == 0).all()) and not bool(torch.signbit(J[i, a]).any()), (i, a)
                continue
            x = tokens.clone()
            x[0, 1 + i] = 4 + a
            want = model(x)["logits"][0, 1:L + 1, 4:24] - wt
            mismatches += int(not torch.equal(J[i, a], want))
    print(f"PARITY jacobian batching {name} L={L}: {20 * L - identities} copies, {mismatches} rows differ from the "
          f"public forward loop, max|J|={float(J.abs().max()):.4g}")
    assert identities == L - 1 and mismatches == 0  # one residue is X
    for copies in (1, 7):
        assert torch.equal(jacobian.categorical_jacobian(model, tokens, max_tokens=copies * T,
                                                         return_jacobian=True)["jacobian"], J), copies


def test_a_chunk_with_identity_copies_returns_the_wild_type(fixtures):
    from esm_b200 import jacobian
    model, alphabet = fixtures["esm2_t2_tiny"]
    model = model.cuda()
    seq = _protein(40, seed=3)
    tokens = alphabet.get_batch_converter()([("p", seq)])[2].cuda()
    L = len(seq)
    wt = model(tokens)["logits"][0, 1:L + 1, 4:24]
    flat = torch.arange(20 * L, device="cuda")
    ident = flat[tokens[0, 1 + flat // 20] == 4 + flat % 20]
    mixed = torch.cat([flat[:25], ident])  # substitutions and identities in one chunk
    rows = jacobian._substitution_rows(model, tokens, mixed, 4)
    for k in range(25, mixed.numel()):
        assert torch.equal(rows[k], wt), int(mixed[k])


# ---- 3. against the reference in float64 ----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def esm_ref():
    if not os.path.isdir(os.path.join(REF, "esm")):
        pytest.fail("oracle/_ref/esm is missing: build() copies the reference there (oracle/reference.py)")
    sys.path.insert(0, REF)
    try:
        import esm  # the reference
        yield esm
    finally:
        sys.path.remove(REF)


def _reference_jacobian(ref, tokens):
    """J, F (the stacked residue logits of the copies) and f_wt by the definition, float64 on the CPU."""
    T = tokens.shape[1]
    L = T - 2
    with torch.no_grad():
        wt = ref(tokens)["logits"][0, 1:L + 1, 4:24]
        batch = tokens.repeat(20 * L, 1)
        flat = torch.arange(20 * L)
        batch[flat, flat // 20 + 1] = flat % 20 + 4
        keep = tokens[0, 1 + flat // 20] != 4 + flat % 20
        F = torch.cat([ref(batch[s:s + 256])["logits"][:, 1:L + 1, 4:24] for s in range(0, 20 * L, 256)])
    J = (F - wt).view(L, 20, L, 20)
    J[~keep.view(L, 20)] = 0
    return J, F[keep], wt, int(keep.sum())


@pytest.mark.parametrize("precision", ["fp16", "fp32x3"])
@pytest.mark.parametrize("name", ["esm2_t2_tiny", "esm1b_t2_tiny"])
def test_against_the_reference_in_float64(esm_ref, fixtures, name, precision):
    import variant_fixtures as vf
    from esm_b200 import jacobian
    model, alphabet = fixtures[name]
    cfg = vf.MODELS[name]
    if cfg["kind"] == "esm2":
        ref = esm_ref.ESM2(num_layers=cfg["layers"], embed_dim=cfg["embed_dim"],
                           attention_heads=cfg["attention_heads"],
                           alphabet=esm_ref.Alphabet.from_architecture("ESM-1b"), token_dropout=cfg["token_dropout"])
    else:
        args = argparse.Namespace(**vars(vf.model_args(cfg)), emb_layer_norm_before=cfg["emb_layer_norm_before"])
        ref = esm_ref.ProteinBertModel(args, esm_ref.Alphabet.from_architecture("roberta_large"))
    ref.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()}, strict=True)
    ref = ref.double().eval()
    seq = _protein(40, seed=7)
    tokens = alphabet.get_batch_converter()([("p", seq)])[2]
    J64, F64, wt64, n_copies = _reference_jacobian(ref, tokens)
    model = model.cuda().set_precision(precision)
    try:
        out = jacobian.categorical_jacobian(model, tokens.cuda(), return_jacobian=True)
    finally:
        model.set_precision("fp16")
    J = out["jacobian"].double().cpu()
    c = 4e-3 if precision == "fp16" else 4e-4
    scale = float(F64.norm()) + math.sqrt(n_copies) * float(wt64.norm())
    j_err = float((J - J64).norm()) / scale
    C64 = contacts_f64(J64)
    c_err = float((out["contacts"].double().cpu() - C64).norm() / C64.norm())
    c_gate = 1e-2 if precision == "fp16" else 1e-3
    print(f"PARITY jacobian reference_f64 {name} {precision} L={len(seq)}: J err/(|F|+sqrt(n)|f_wt|)={j_err:.3e} "
          f"(gate {c:.0e}), |J - J64|/|J64|={float((J - J64).norm() / J64.norm()):.3e}, "
          f"contacts rel_fro={c_err:.3e} (gate {c_gate:.0e})")
    assert j_err <= c
    assert c_err <= c_gate


# ---- 4. cpu_offload() and model.half() -----------------------------------------------------------------------------
def test_cpu_offload_is_bit_identical_and_half_returns_fp32(tmp_path):
    from esm_b200 import jacobian
    model, alphabet = _fixture_model("esm2_t2_tiny", str(tmp_path))  # its own copy: half() rounds the weights
    model = model.cuda()
    tokens = alphabet.get_batch_converter()([("p", _protein(33, seed=11))])[2].cuda()
    want = jacobian.categorical_jacobian(model, tokens, return_jacobian=True)
    model.cpu_offload()
    try:
        got = jacobian.categorical_jacobian(model, tokens, max_tokens=5 * tokens.shape[1], return_jacobian=True)
    finally:
        model.cuda()
    assert torch.equal(got["jacobian"], want["jacobian"]) and torch.equal(got["contacts"], want["contacts"])
    half = jacobian.categorical_jacobian(model.half(), tokens, return_jacobian=True)
    assert half["jacobian"].dtype == torch.float32 and half["contacts"].dtype == torch.float32
    r = float((half["contacts"] - want["contacts"]).norm() / want["contacts"].norm())
    print(f"PARITY jacobian half() esm2_t2_tiny: contacts rel_fro={r:.3e} vs the fp32 model; cpu_offload bit-identical")
    assert bool(half["contacts"].isfinite().all()) and r <= 0.1


# ---- 5. full size ----------------------------------------------------------------------------------------------------
def test_650M_sampled_rows_equal_the_public_forward():
    from esm_b200 import jacobian, pretrained
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        model, alphabet = pretrained.load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=True,
                                                             device="cuda")
    model = model.eval().cuda()
    L = 200
    tokens = alphabet.get_batch_converter()([("p", _protein(L, seed=200))])[2].cuda()
    J = jacobian.categorical_jacobian(model, tokens, return_jacobian=True)["jacobian"]
    wt = model(tokens)["logits"][0, 1:L + 1, 4:24]
    g = torch.Generator().manual_seed(5)
    picks = [(int(i), int(a)) for i, a in zip(torch.randint(0, L, (60,), generator=g),
                                             torch.randint(0, 20, (60,), generator=g))
             if int(tokens[0, 1 + int(i)]) != 4 + int(a)][:50]
    assert len(picks) == 50
    bad = 0
    for i, a in picks:
        x = tokens.clone()
        x[0, 1 + i] = 4 + a
        bad += int(not torch.equal(J[i, a], model(x)["logits"][0, 1:L + 1, 4:24] - wt))
    print(f"PARITY jacobian 650M L={L} fp16: {bad} of 50 sampled rows differ from the public forward, "
          f"max|J|={float(J.abs().max()):.4g}")
    assert bad == 0


# ---- 6. the command line ---------------------------------------------------------------------------------------------
def test_cli_end_to_end(tmp_path):
    import variant_fixtures as vf
    from esm_b200 import jacobian, jacobian_cli, pretrained
    path = vf.write_checkpoint("esm2_t2_tiny", vf.MODELS["esm2_t2_tiny"], str(tmp_path))
    seqs = {"first": _protein(30, seed=1), "short": "M", "third": _protein(45, seed=2)}
    (tmp_path / "s.fa").write_text("".join(f">{k}\n{v}\n" for k, v in seqs.items()))
    out_dir = tmp_path / "out"
    args = jacobian_cli.create_parser().parse_args([path, str(tmp_path / "s.fa"), str(out_dir), "--save-jacobian",
                                                    "--max-tokens", "500"])
    assert jacobian_cli.run(args) == 2
    assert not (out_dir / "short.pt").exists()
    model, alphabet = pretrained.load_model_and_alphabet(path)
    model = model.eval().cuda()
    for label in ("first", "third"):
        got = torch.load(out_dir / f"{label}.pt")
        tokens = alphabet.get_batch_converter()([(label, seqs[label])])[2].cuda()
        want = jacobian.categorical_jacobian(model, tokens, return_jacobian=True)
        assert got["label"] == label and not got["contacts"].is_cuda
        assert torch.equal(got["contacts"], want["contacts"].cpu())
        assert torch.equal(got["jacobian"], want["jacobian"].cpu())
    print("PARITY jacobian cli: 2 files equal the API's results bit for bit, the 1-residue record skipped")
