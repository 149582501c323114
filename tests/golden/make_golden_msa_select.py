"""Writes tests/golden/msa_select.json: the rows that greedy_select of facebookresearch/esm's
examples/contact_prediction.ipynb (the "MSA Transformer" section) returns, for

  * the notebook's three alignments (tests/golden/msa/{1a3a,5ahw,1xcr}_1_A.a3m.gz, gzip copies of examples/data) at
    num_seqs 64, 128 and 500, in both modes;
  * seeded tie-heavy alignments of 2 or 3 symbols with 1, 3, 7 or 10 columns, with num_seqs past 8, 128 and 256 (the
    edges of numpy's pairwise summation);
  * num_seqs >= N, num_seqs 0 and 1, and a single row.

The function is read out of the notebook when this script runs and executed as it stands; nothing of it is copied
here. Alignments are read as the notebook reads them (esm_b200.variants.read_msa: the whole header line as the
description, insertions removed). Each alignment is stored once, with the selected indices of every (num_seqs, mode).

    python tests/golden/make_golden_msa_select.py PATH_TO_A_FACEBOOKRESEARCH_ESM_CHECKOUT    (CPU, numpy and scipy)
"""
import json
import os
import sys
from typing import List, Tuple

import numpy as np
from scipy.spatial.distance import cdist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))  # msa_select_refs
OUT = os.path.join(HERE, "msa_select.json")
ALIGNMENTS = ["1a3a_1_A", "5ahw_1_A", "1xcr_1_A"]


def notebook_greedy_select(reference: str):
    with open(os.path.join(reference, "examples", "contact_prediction.ipynb")) as f:
        cells = json.load(f)["cells"]
    src = next("".join(c["source"]) for c in cells if "def greedy_select" in "".join(c["source"]))
    namespace = {"np": np, "cdist": cdist, "List": List, "Tuple": Tuple}
    exec(src, namespace)
    return namespace["greedy_select"]


def synthetic_cases():
    g = np.random.default_rng(2024)
    cases = []
    for symbols, C, N, ks in [(2, 1, 40, [9, 39]), (3, 3, 150, [9, 130]), (2, 7, 300, [17, 129, 260]),
                              (3, 10, 320, [8, 136, 257, 300]), (2, 10, 140, [128, 129]), (3, 7, 30, [30, 31, 50])]:
        rows = ["".join(g.choice(list("ACD"[:symbols]), C)) for _ in range(N)]
        cases.append((rows, ks))
    cases.append((["AC-", "AD-", "CC-"], [0, 1, 2, 3, 4]))
    cases.append((["MKV"], [0, 1, 5]))
    return cases


def main(reference: str):
    import msa_select_refs as ref
    greedy_select = notebook_greedy_select(reference)

    def results(msa, ks):
        index = {id(r): i for i, r in enumerate(msa)}
        return [{"num_seqs": k, "mode": mode, "selected": [index[id(r)] for r in greedy_select(msa, k, mode)]}
                for k in ks for mode in ("max", "min")]

    out = {"source": "facebookresearch/esm examples/contact_prediction.ipynb, greedy_select (executed unchanged); "
                     "selected: the indices of the returned rows in the input, in the returned order",
           "alignments": [], "synthetic": []}
    for name in ALIGNMENTS:
        file = f"msa/{name}.a3m.gz"
        out["alignments"].append({"file": file, "results": results(ref.read_golden_a3m(file), (64, 128, 500))})
    for rows, ks in synthetic_cases():
        out["synthetic"].append({"rows": rows, "results": results([(str(i), r) for i, r in enumerate(rows)], ks)})
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"))
        f.write("\n")
    print(OUT, sum(len(a["results"]) for a in out["alignments"] + out["synthetic"]), "cases")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
