"""NumPy / Python restatement of the test-set prediction file (newsrec_b200.predict): ranks of every impression and the
text of prediction.txt.  Test infrastructure only.

The rank of candidate i is its 1-based position in ``np.argsort(s, kind="stable")[::-1]``: descending score, among equal
scores the later candidate first, -0 == +0 -- the order oracle/ranking_metrics.py pins for MRR / nDCG, so MRR recomputed
from these ranks is that oracle's MRR."""
from __future__ import annotations

import numpy as np


def single_ranks(scores):
    """(n,) int64 1-based ranks of one impression's scores (finite)."""
    s = np.asarray(scores, dtype=np.float64)  # fp32 -> fp64 is exact; -0.0 and 0.0 compare equal, so the stable sort ties them
    order = np.argsort(s, kind="stable")[::-1]
    ranks = np.empty(len(s), np.int64)
    ranks[order] = np.arange(1, len(s) + 1)
    return ranks


def impression_ranks(scores, offsets):
    """(n_cand,) int64: the ranks of scores[offsets[s]:offsets[s+1]] within each impression."""
    scores, offsets = np.asarray(scores), np.asarray(offsets)
    out = np.empty(len(scores), np.int64)
    for a, b in zip(offsets[:-1], offsets[1:]):
        out[a:b] = single_ranks(scores[a:b])
    return out


def prediction_text(ids, ranks, offsets):
    """The bytes of prediction.txt: one "<id> [r1,...,rn]\\n" per impression."""
    return "".join(f"{i} [{','.join(map(str, ranks[a:b]))}]\n" for i, a, b in zip(ids, offsets[:-1], offsets[1:])).encode()
