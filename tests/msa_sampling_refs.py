"""Numpy restatement of the alignment sampler's definition (esm_b200.sampling.msa_gibbs) on top of sampling_refs: the
entry index of an alignment, the 20-bit visiting order and block partition of a sweep, the uniforms of a token set of
up to 32 ids, and the Gumbel-max draw of a block in float64."""
from __future__ import annotations

import numpy as np

import sampling_refs as sr

ENTRY_BITS = 20


def entry_token(p, C):
    """(row, column) of entry p in an alignment of C columns whose column 0 is <cls>."""
    p = np.asarray(p, dtype=np.int64)
    return p // (C - 1), 1 + p % (C - 1)


def msa_order_keys(entries, chains, sweep, seed):
    """keys [len(chains), n] int64 = R(sweep, c, p, 0).x * 2^20 + p."""
    p = np.asarray(entries, dtype=np.int64)[None, :]
    c = np.asarray(chains, dtype=np.int64)[:, None]
    x = sr.philox4x32_10(sweep, c, p, 0, seed)[0]
    return x.astype(np.int64) * (1 << ENTRY_BITS) + p


def msa_sweep_blocks(entries, chain, sweep, seed, block):
    """The blocks of one sweep of one chain: the designable entries sorted by their keys, cut into runs of
    min(block, n)."""
    keys = msa_order_keys(entries, [chain], sweep, seed)[0]
    order = np.sort(keys) % (1 << ENTRY_BITS)
    k = min(block, len(order))
    return [order[i:i + k] for i in range(0, len(order), k)]


def set_uniforms(step, chains, entries, seed, n_set):
    """u [n, n_set] fp32 of n rows (chain, entry): u_a = word a mod 4 of R(step, chain, p, 1 + a div 4)."""
    chains = np.asarray(chains, dtype=np.int64)[:, None]
    entries = np.asarray(entries, dtype=np.int64)[:, None]
    words = sr.philox4x32_10(step, chains, entries, np.arange(1, 9)[None, :], seed)  # 4 arrays of [n, 8]
    return sr.uniform(np.stack(words, -1).reshape(len(entries), 32)[:, :n_set])


def draw_f64(z, step, chains, entries, seed):
    """Float64 Gumbel-max scores and a* of fp32 tempered logits z [n, n_set] for rows (chain, entry)."""
    return sr.gumbel_max_f64(z, set_uniforms(step, chains, entries, seed, np.shape(z)[-1]))
