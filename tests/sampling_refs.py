"""Numpy restatement of the sampler's definition (esm_b200/sampling.py): Philox4x32-10, the uniform map, the entry
index of a layout, the visiting order and block partition of a sweep, the uniforms of a token set of up to 32 ids, and
the Gumbel-max draw in float64. The CPU tests pin it against the toolkit's Philox known answers and the definition's
properties; the GPU tests gate the kernels, gibbs and msa_gibbs against it."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, key):
    """R(c0, c1, c2, c3) for uint32 counter words (scalars or broadcastable arrays) and a 64-bit seed, key (seed mod
    2^32, seed >> 32). Returns four uint32 arrays (x, y, z, w), as curand_Philox4x32_10 computes them."""
    c = [np.asarray(v, dtype=np.uint64) & MASK for v in (c0, c1, c2, c3)]
    c = np.broadcast_arrays(*c)
    c = [v.copy() for v in c]
    k0, k1 = np.uint64(int(key) & 0xFFFFFFFF), np.uint64(int(key) >> 32)
    for r in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]  # 32 x 32 -> 64-bit products, exact in uint64
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        if r < 9:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return tuple(v.astype(np.uint32) for v in c)


def uniform(r):
    """u = ((r >> 8) + 0.5) * 2^-24 rounded toward zero to fp32: (2j + 1) 2^-25 below 2^23 (exact), j 2^-24 above."""
    j = np.asarray(r, dtype=np.uint64) >> np.uint64(8)
    exact = (2 * j.astype(np.float64) + 1) * 2.0 ** -25
    return np.where(j < (1 << 23), exact, j.astype(np.float64) * 2.0 ** -24).astype(np.float32)


def entry_token(p, C):
    """(row, column) of entry p in an alignment of C columns whose column 0 is <cls>."""
    p = np.asarray(p, dtype=np.int64)
    return p // (C - 1), 1 + p % (C - 1)


def order_keys(entries, chains, sweep, seed):
    """keys [len(chains), n] int64 = R(sweep, c, p, 0).x * 2^20 + p."""
    p = np.asarray(entries, dtype=np.int64)[None, :]
    c = np.asarray(chains, dtype=np.int64)[:, None]
    x = philox4x32_10(sweep, c, p, 0, seed)[0]
    return x.astype(np.int64) * (1 << 20) + p


def sweep_blocks(entries, chain, sweep, seed, block):
    """The blocks of one sweep of one chain: the designable entries sorted by their keys, cut into runs of
    min(block, n)."""
    keys = order_keys(entries, [chain], sweep, seed)[0]
    order = np.sort(keys) % (1 << 20)
    k = min(block, len(order))
    return [order[i:i + k] for i in range(0, len(order), k)]


def uniforms(step, chains, entries, seed, n_set):
    """u [n, n_set] fp32 of n rows (chain, entry): u_a = word a mod 4 of R(step, chain, p, 1 + a div 4)."""
    chains = np.asarray(chains, dtype=np.int64)[:, None]
    entries = np.asarray(entries, dtype=np.int64)[:, None]
    words = philox4x32_10(step, chains, entries, np.arange(1, 9)[None, :], seed)  # 4 arrays of [n, 8]
    return uniform(np.stack(words, -1).reshape(len(entries), 32)[:, :n_set])


def draw_f64(z, step, chains, entries, seed):
    """Float64 Gumbel-max scores and a* of fp32 tempered logits z [n, n_set] for rows (chain, entry)."""
    return gumbel_max_f64(z, uniforms(step, chains, entries, seed, np.shape(z)[-1]))


def gumbel_max_f64(z, u):
    """Float64 Gumbel-max scores z + g, g = -log(-log(u)), and a* (the first maximum). z [..., n_set], u likewise."""
    score = np.asarray(z, dtype=np.float64) - np.log(-np.log(np.asarray(u, dtype=np.float64)))
    return score, np.argmax(score, axis=-1)


def top_two_gap(score):
    """Per row, the best score minus the second best."""
    s = np.sort(score, axis=-1)
    return s[..., -1] - s[..., -2]


def log_softmax_f64(z):
    """log_softmax of z along the last axis in float64."""
    z = np.asarray(z, dtype=np.float64)
    m = z.max(-1, keepdims=True)
    return (z - m) - np.log(np.exp(z - m).sum(-1, keepdims=True))
