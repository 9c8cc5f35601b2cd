"""NumPy fp64 restatement of the evaluator's per-impression metrics (reference src/evaluate.py:25-46, 160-168).

TEST INFRASTRUCTURE ONLY (see newsrec_oracle.py).  No scikit-learn: the GPU machines may not have it.

The reference computes, per impression, sklearn's ``roc_auc_score`` and NumPy ``mrr_score`` / ``ndcg_score`` over
``np.argsort(y_score)[::-1]``.  NumPy's default sort is not stable, so where tied candidates carry different labels the
reference's MRR / nDCG depend on the sort's internals.  This restatement pins the stable reading of the same expression,
``np.argsort(s, kind="stable")[::-1]`` (among equal scores the later candidate ranks first), as ``nr_impression_metrics``
does.  AUC is the Mann-Whitney form (what ``roc_auc_score`` computes, ties counted half), in integers.

Degenerate impressions follow the reference with scikit-learn 1.9: a non-finite score makes sklearn raise (all four NaN);
no negative makes AUC NaN (sklearn warns) while MRR / nDCG stay defined; no positive makes all four NaN.
"""
from __future__ import annotations

import numpy as np


def single_impression(scores, labels):
    """(auc, mrr, ndcg5, ndcg10) of one impression, fp64."""
    s = np.asarray(scores, dtype=np.float64)
    y = np.asarray(labels, dtype=np.int64)
    nan = (np.nan,) * 4
    if not np.isfinite(s).all():
        return nan
    P = int(y.sum())
    N = len(y) - P
    if P == 0:
        return nan
    neg = np.sort(s[y == 0])
    sp = s[y == 1]
    below = np.searchsorted(neg, sp, side="left")
    level = np.searchsorted(neg, sp, side="right") - below
    auc = float(np.sum(2 * below + level)) / (2.0 * P * N) if N > 0 else np.nan
    gains = y[np.argsort(s, kind="stable")[::-1]]
    places = np.flatnonzero(gains)                     # 0-based positions of the positives in the descending order
    mrr = float(np.sum(1.0 / (places + 1.0))) / P
    disc = 1.0 / np.log2(np.arange(10) + 2.0)

    def ndcg(k):
        return float(np.sum(disc[places[places < k]])) / float(np.sum(disc[:min(P, k)]))

    return auc, mrr, ndcg(5), ndcg(10)


def impression_metrics(scores, labels, offsets):
    """(n_impressions, 4) fp64: the metrics of scores[offsets[s]:offsets[s+1]] with the labels at the same positions."""
    scores, labels, offsets = np.asarray(scores), np.asarray(labels), np.asarray(offsets)
    out = np.empty((len(offsets) - 1, 4), dtype=np.float64)
    for i in range(len(offsets) - 1):
        a, b = offsets[i], offsets[i + 1]
        out[i] = single_impression(scores[a:b], labels[a:b])
    return out


def cross_label_ties(scores, labels, offsets):
    """(n_impressions,) bool: some score is shared by a positive and a negative candidate (the reference's MRR / nDCG
    are then decided by NumPy's unstable sort)."""
    scores, labels, offsets = np.asarray(scores, dtype=np.float64), np.asarray(labels), np.asarray(offsets)
    out = np.zeros(len(offsets) - 1, dtype=bool)
    for i in range(len(offsets) - 1):
        a, b = offsets[i], offsets[i + 1]
        s, y = scores[a:b], labels[a:b]
        out[i] = bool(np.intersect1d(s[y == 1], s[y == 0]).size)
    return out
