"""Generates tests/golden/variants.json by running the UNMODIFIED reference script
examples/variant-prediction/predict.py (from /root/reference) on the CPU, on the small models of
tests/variant_fixtures.py written as local checkpoints.

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_variants.py

predict.py needs four things this container does not give it, supplied here without touching the script:
  * Biopython: a stub `Bio.SeqIO` whose parse(path, "fasta") yields records with .description and .seq;
  * a GPU: predict.py calls `.cuda()` on the tokens even with --nogpu (predict.py:142,175,194,211), so
    torch.Tensor.cuda is patched to return the tensor itself;
  * torch.load(weights_only=True) (the default) refuses the argparse.Namespace in the checkpoints:
    torch.serialization.safe_globals([Namespace]);
  * checkpoints: each model is written as a .pt file with the "-contact-regression.pt" companion that the reference's
    local loader expects (pretrained.py:67-77).
The fixture stores the model configs, seeds and state-dict checksums (weights are rebuilt where the tests run), the
input texts (sequence, DMS table, a3m) and predict.py's output tables.
"""
import json
import os
import random
import sys
import tempfile
import types
from argparse import Namespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))  # tests/
REFERENCE = "/root/reference"
sys.path.insert(0, REFERENCE)
sys.path.insert(0, os.path.join(REFERENCE, "examples", "variant-prediction"))

import variant_fixtures as vf  # noqa: E402  (tests/variant_fixtures.py)

AA = "ACDEFGHIKLMNPQRSTVWY"
OFFSET_IDX = 1          # mutation positions are 1-based in the table
SEED = 2024


def _stub_biopython():
    class Record:
        def __init__(self, description, seq):
            self.description, self.seq = description, seq

    def parse(path, fmt):
        assert fmt == "fasta"
        title, lines = None, []
        with open(path) as f:
            for line in f:
                if line.startswith(">"):
                    if title is not None:
                        yield Record(title, "".join(lines))
                    title, lines = line[1:].rstrip(), []
                elif title is not None:
                    lines.append(line.strip())
        if title is not None:
            yield Record(title, "".join(lines))

    bio = types.ModuleType("Bio")
    seqio = types.ModuleType("Bio.SeqIO")
    seqio.parse = parse
    bio.SeqIO = seqio
    sys.modules["Bio"] = bio
    sys.modules["Bio.SeqIO"] = seqio


def make_inputs():
    rng = random.Random(SEED)
    L = 52
    sequence = "".join(rng.choice(AA) for _ in range(L))
    idxs = [0, L - 1] + rng.sample(range(1, L - 1), 36)
    targets = {0: "W", L - 1: "X", idxs[2]: "B", idxs[3]: "Z"}  # X, B, Z: non-standard residue letters
    rows = []
    for n, i in enumerate(idxs):
        mt = targets.get(i) or rng.choice([a for a in AA if a != sequence[i]])
        note = ["", "surface", "core, buried", "loop", "helix 2"][n % 5]
        rows.append((f"{sequence[i]}{i + OFFSET_IDX}{mt}", note, str(rng.randint(0, 3))))
    dms = "mutant,note,replicate\n" + "".join(
        ",".join(f'"{c}"' if "," in c else c for c in r) + "\n" for r in rows)
    # a3m: the query first, then aligned rows with lowercase insertions, '.' and gaps
    a3m = [f">query {L} residues\n{sequence}\n"]
    for r in range(9):
        cols = []
        for i, a in enumerate(sequence):
            x = rng.random()
            cols.append("-" if x < 0.1 else (rng.choice(AA) if x < 0.4 else a))
            if rng.random() < 0.05:
                cols.append(rng.choice(AA).lower() + ("." if rng.random() < 0.5 else ""))
        seq = "".join(cols)
        a3m.append(f">hit{r} score={rng.randint(10, 99)} desc with spaces\n{seq[:40]}\n{seq[40:]}\n")
    return sequence, dms, "".join(a3m)


def main():
    _stub_biopython()
    torch.Tensor.cuda = lambda self, *a, **k: self
    import predict  # noqa: E402  (the reference script, unmodified)

    torch.set_num_threads(8)
    sequence, dms, a3m = make_inputs()
    fixture = {"offset_idx": OFFSET_IDX, "msa_samples": 7, "sequence": sequence, "dms_csv": dms, "a3m": a3m,
               "models": {}, "outputs": {},
               "reference": "facebookresearch/esm @ 2b36991 (fair-esm 2.0.1) examples/variant-prediction/predict.py, "
                            "torch %s, CPU fp32" % torch.__version__}
    with tempfile.TemporaryDirectory() as tmp, torch.serialization.safe_globals([Namespace]):
        dms_path = os.path.join(tmp, "dms.csv")
        msa_path = os.path.join(tmp, "msa.a3m")
        open(dms_path, "w").write(dms)
        open(msa_path, "w").write(a3m)
        for name, cfg in vf.MODELS.items():
            fixture["models"][name] = dict(cfg, state_dict_checksum=vf.checksum(vf.state_dict(cfg)))
            ckpt = vf.write_checkpoint(name, cfg, tmp)
            strategies = ["masked-marginals"] if cfg["kind"] == "msa" else \
                ["wt-marginals", "masked-marginals", "pseudo-ppl"]
            for strategy in strategies:
                out = os.path.join(tmp, f"{name}-{strategy}.csv")
                argv = ["--model-location", ckpt, "--sequence", sequence, "--dms-input", dms_path, "--dms-output", out,
                        "--offset-idx", str(OFFSET_IDX), "--scoring-strategy", strategy, "--nogpu"]
                if cfg["kind"] == "msa":
                    argv += ["--msa-path", msa_path, "--msa-samples", str(fixture["msa_samples"])]
                predict.main(predict.create_parser().parse_args(argv))
                text = open(out).read()
                # the score column is named by the location string: store it relative to the checkpoint directory
                fixture["outputs"][f"{name}/{strategy}"] = text.replace(ckpt, name + ".pt")
                print(name, strategy, "done")
    path = os.path.join(HERE, "variants.json")
    with open(path, "w") as f:
        json.dump(fixture, f, indent=1)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
