"""Restatement of the training negatives: the device draw of nr_sample_negatives (include/newsrec_b200.h) in NumPy, and
the reference's balancing rule (parse_behaviors in src/data_preprocess.py:52-67) in plain Python.

The reference pairs, per impression, each positive in file order with the next K = negative_sampling_ratio negatives of
ONE shuffle of the impression's negatives, until the positives run out or fewer than K negatives remain: min(P, N // K)
rows, no negative in two rows of an impression, the same negatives in every epoch.  The device draw keeps that rule and
redraws the shuffle per (seed, epoch): the negatives sorted by (h_j, j), h_j the high 32 bits of a chained splitmix64 hash
of (seed, epoch, impression, j).  `draw` is what the kernel must write, bit for bit; `reference_balance` is the host
baseline of tools/negsample_bench.py and the structure the minted fixture (tests/golden/negsample/) is checked against.
"""
from __future__ import annotations

import random

import numpy as np

M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15


def hash_step(x, v):
    """One link of the chain: splitmix64's finaliser of (x ^ v) + golden ratio, all uint64 (NumPy arrays or ints)."""
    with np.errstate(over="ignore"):
        z = (np.uint64(x) ^ np.uint64(v)) + np.uint64(GOLDEN)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def negative_order(seed, epoch, i, n):
    """Ordinals 0..n-1 of impression i's negatives in drawn order: ascending (h_j, j)."""
    x = hash_step(hash_step(hash_step(0, seed & M64), epoch & M64), i & M64)
    j = np.arange(n, dtype=np.uint64)
    h = hash_step(x, j) >> np.uint64(32)
    return np.lexsort((j, h)).astype(np.int64)


def balanced_rows(labels, imp_offsets, K):
    """(n_imp,) int64 rows per impression: min(P, N // K) over labels 1 (positive) and 0 (negative)."""
    imp = np.repeat(np.arange(len(imp_offsets) - 1), np.diff(imp_offsets))
    P = np.bincount(imp, weights=labels == 1, minlength=len(imp_offsets) - 1).astype(np.int64)
    N = np.bincount(imp, weights=labels == 0, minlength=len(imp_offsets) - 1).astype(np.int64)
    return np.minimum(P, N // K)


def draw(cand_rows, labels, imp_offsets, K, seed, epoch):
    """(row_offsets (n_imp + 1,), candidates (R, 1 + K)) int64: the candidate columns nr_sample_negatives writes."""
    cand_rows, labels, imp_offsets = np.asarray(cand_rows), np.asarray(labels), np.asarray(imp_offsets, np.int64)
    rows = balanced_rows(labels, imp_offsets, K)
    row_offsets = np.concatenate([[0], np.cumsum(rows)]).astype(np.int64)
    out = np.zeros((int(row_offsets[-1]), 1 + K), np.int64)
    for i in np.flatnonzero(rows):
        c = cand_rows[imp_offsets[i]:imp_offsets[i + 1]]
        lab = labels[imp_offsets[i]:imp_offsets[i + 1]]
        pos, neg = c[lab == 1], c[lab == 0]
        R = int(rows[i])
        picked = neg[negative_order(seed, epoch, int(i), len(neg))[:R * K]]
        out[row_offsets[i]:row_offsets[i + 1], 0] = pos[:R]
        out[row_offsets[i]:row_offsets[i + 1], 1:] = picked.reshape(R, K)
    return row_offsets, out


def reference_balance(impressions, K, rng=random):
    """The reference's loop (data_preprocess.py:52-67) over impression token lists ("N123-1", ...): per impression the
    list of rows [positive, K negatives], the negatives shuffled once with `rng` (a random.Random or the module)."""
    out = []
    for items in impressions:
        pos = [x for x in items if x.endswith("1")]
        neg = [x for x in items if x.endswith("0")]
        rng.shuffle(neg)
        out.append([[pos[p]] + neg[p * K:(p + 1) * K] for p in range(min(len(pos), len(neg) // K))])
    return out
