"""A vectorised numpy restatement of greedy_select from the reference's examples/contact_prediction.ipynb, the
definition in include/esmb200.h at esmb200_msa_greedy_select. It returns the picked rows in selection order.

The notebook scores the candidates with np.delete(pairwise_distances, indices, axis=1).mean(0). np.delete along axis 1
returns an F-contiguous array, so mean(0) reduces along the contiguous axis with numpy's pairwise summation, whose
tree depends only on the number of terms t: it vectorises over the candidates."""
import gzip
import json
import os
import tempfile

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def read_golden_a3m(file):
    """[(description, sequence)] of a gzipped a3m file under tests/golden, read by esm_b200.variants.read_msa."""
    from esm_b200 import variants
    with tempfile.TemporaryDirectory() as tmp, gzip.open(os.path.join(GOLDEN, file), "rb") as f:
        path = os.path.join(tmp, "msa.a3m")
        with open(path, "wb") as out:
            out.write(f.read())
        return variants.read_msa(path, None)


def fixture_cases():
    """(alignment, num_seqs, mode, selected) for every case of tests/golden/msa_select.json."""
    with open(os.path.join(GOLDEN, "msa_select.json")) as f:
        fx = json.load(f)
    out = []
    for a in fx["alignments"] + fx["synthetic"]:
        msa = read_golden_a3m(a["file"]) if "file" in a else [(str(i), r) for i, r in enumerate(a["rows"])]
        out += [(msa, r["num_seqs"], r["mode"], r["selected"]) for r in a["results"]]
    return out


def pairwise_sum(a):
    """numpy's pairwise_sum of each column of a float64 [n, M], in numpy's order."""
    n = a.shape[0]
    if n < 8:
        res = np.zeros(a.shape[1])
        for i in range(n):
            res = res + a[i]
        return res
    if n <= 128:
        r = a[:8].copy()
        i = 8
        while i < n - n % 8:
            r = r + a[i:i + 8]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(n - n % 8, n):
            res = res + a[i]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


def as_rows(msa):
    """The notebook's byte array of an alignment [(description, sequence)]: uint8 [N, C]. Ragged rows raise
    ValueError."""
    return np.array([list(seq) for _, seq in msa], dtype=np.bytes_).view(np.uint8)


def greedy_order(rows, k, mode="max", shortcut=True):
    """The notebook's picks for uint8 rows [N, C], in selection order (the notebook returns them sorted). N <= k
    returns every row, as the notebook (and esm_b200.msa_select) does without a selection; shortcut=False instead runs
    the loop up to k = N, whose last step has a single candidate, as the C ABI does when called with k = N."""
    assert mode in ("max", "min")
    rows = np.asarray(rows, dtype=np.uint8)
    N, C = rows.shape
    if shortcut and N <= k:
        return list(range(N))
    assert k <= N
    sel = [0]
    picked = np.zeros(N, dtype=bool)
    picked[0] = True
    d = np.empty((max(k - 1, 0), N))
    for t in range(1, k):
        d[t - 1] = (rows != rows[sel[-1]]).sum(1) / C
        score = pairwise_sum(d[:t]) / t
        score[picked] = -np.inf if mode == "max" else np.inf
        j = int(np.argmax(score) if mode == "max" else np.argmin(score))
        sel.append(j)
        picked[j] = True
    return sel
