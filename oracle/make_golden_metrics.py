"""Mint tests/golden/eval_metrics.npz from the LIVE reference metric function (build container only).

    python oracle/make_golden_metrics.py

Imports ``calculate_single_user_metric`` from the unmodified reference ``src/evaluate.py`` (sklearn ``roc_auc_score`` +
NumPy ``mrr_score`` / ``ndcg_score``) and evaluates it, exactly as the reference's process pool does, on seeded fp32
impressions chosen for their edges: lengths 1 .. 1500 (longer than the kernel's shared-memory chunk), one class only,
non-finite scores, ties within one label, ties across labels, -0 / +0.  Kept apart from make_golden.py so that minting
this fixture does not re-mint the model fixtures.

Writes scores (fp32, back to back), labels (uint8), offsets (int64), ref (n, 4) fp64 -- the reference's values --,
cross_tie (bool: a score shared by a positive and a negative; there the reference's MRR / nDCG depend on NumPy's
unstable sort) and the scikit-learn / NumPy versions.
"""
from __future__ import annotations

import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ranking_metrics  # noqa: E402

REF_SRC = "/root/reference/src"
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "eval_metrics.npz")


def segments(rng):
    """[(scores fp32, labels uint8)] -- every edge the issue of the evaluator names, plus seeded random impressions."""
    segs = []

    def rand(n, p_pos=0.2, levels=None):
        s = (rng.integers(0, levels, n) if levels else rng.standard_normal(n)).astype(np.float32)
        y = (rng.random(n) < p_pos).astype(np.uint8)
        if n >= 2 and y.sum() == 0:
            y[rng.integers(n)] = 1
        if n >= 2 and y.sum() == n:
            y[rng.integers(n)] = 0
        return s, y

    for n in (1, 2, 5, 16, 17, 37, 100, 300, 1500):
        for _ in range(3):
            segs.append(rand(n))
    segs.append((np.array([0.3, -1.0, 2.0], np.float32), np.array([1, 1, 1], np.uint8)))            # all positive
    segs.append((np.array([0.3, -1.0, 2.0, 0.1], np.float32), np.array([0, 0, 0, 0], np.uint8)))    # all negative
    segs.append((np.array([0.3, np.nan, 2.0], np.float32), np.array([1, 0, 0], np.uint8)))          # NaN score
    segs.append((np.array([0.3, np.inf, 2.0], np.float32), np.array([0, 1, 0], np.uint8)))          # inf score
    segs.append((np.array([-np.inf, 0.5], np.float32), np.array([1, 0], np.uint8)))
    segs.append((np.array([1.0, 1.0, 0.5, 0.5, 0.2], np.float32), np.array([1, 1, 0, 0, 0], np.uint8)))  # ties within a label
    segs.append((np.array([0.5, 0.5, 0.5, 0.1], np.float32), np.array([0, 1, 1, 0], np.uint8)))     # ties across labels
    segs.append((np.array([0.7, 0.7], np.float32), np.array([1, 0], np.uint8)))
    segs.append((np.array([0.0, -0.0, 1.0, -1.0], np.float32), np.array([1, 0, 0, 0], np.uint8)))   # -0 / +0
    segs.append((np.array([-0.0, 0.0, -2.0], np.float32), np.array([0, 1, 0], np.uint8)))
    for n in (5, 16, 37, 100, 300):                                                                    # many ties
        for _ in range(3):
            segs.append(rand(n, p_pos=0.3, levels=4))
    segs.append(rand(1500, p_pos=0.1, levels=6))
    for _ in range(40):                                                                                # MIND-like
        segs.append(rand(int(rng.integers(2, 80)), p_pos=0.1))
    return segs


def main():
    assert os.path.isdir(REF_SRC), "the reference is only mounted in the build container"
    sys.path.insert(0, REF_SRC)
    import sklearn
    from evaluate import calculate_single_user_metric  # the reference's own metric function

    segs = segments(np.random.default_rng(2024))
    ref = np.empty((len(segs), 4), np.float64)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")  # one-class UndefinedMetricWarning, 0/0 RuntimeWarning: the values are the point
        for i, (s, y) in enumerate(segs):
            # what the reference's scoring loop hands the pool: labels as ints, scores as fp32 .tolist()
            ref[i] = calculate_single_user_metric(([int(v) for v in y], s.tolist()))
    scores = np.concatenate([s for s, _ in segs]).astype(np.float32)
    labels = np.concatenate([y for _, y in segs]).astype(np.uint8)
    offsets = np.concatenate([[0], np.cumsum([len(s) for s, _ in segs])]).astype(np.int64)
    cross = ranking_metrics.cross_label_ties(scores, labels, offsets)
    np.savez_compressed(OUT, scores=scores, labels=labels, offsets=offsets, ref=ref, cross_tie=cross,
                        versions=np.array(f"scikit-learn={sklearn.__version__} numpy={np.__version__}"))
    print(f"{len(segs)} impressions ({cross.sum()} with cross-label ties, {np.isnan(ref).any(1).sum()} with NaN) -> {OUT} "
          f"({os.path.getsize(OUT) / 1024:.0f} KB)")


if __name__ == "__main__":
    main()
