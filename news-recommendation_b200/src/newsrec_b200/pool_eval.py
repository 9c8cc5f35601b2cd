"""Retrieval metrics over the whole news pool on the device: for every held-out click of a labelled split, its position among
all news of ``news_parsed.tsv`` under the model's click score, and recall@K, nDCG@K and MRR of those positions.

``evaluate`` measures how an impression's few dozen candidates are ordered.  A two-tower retriever is asked a different
question: does the news the user clicked come near the top of the whole pool?  Per impression i of ``behaviors.tsv``:

1. P_i      its positives (label 1, a news listed twice counted once); an impression without a positive is skipped;
2. X_i      its user's history when ``exclude_clicked`` (the user is its distinct history, as in ``evaluate``);
3. ranks    r_p of every p in P_i among the pool without X_i and P_i (``ops.pool_ranks``, nr_pool_ranks: the scores
            nr_topk_dot computes, higher first, equal scores by lower row), in chunks of ``chunk_impressions``;
4. position c_p = r_p + |{q in P_i : (s_q, q) before (s_p, p)}|: p's place in the list ``recommend`` would write for
            that user with k = infinity;
5. metrics  recall@K = |{p : c_p < K}| / |P_i|,  nDCG@K = sum_{c_p < K} 1 / log2(c_p + 2) / sum_{j < min(|P_i|, K)} 1 / log2(j + 2),
            MRR = 1 / (1 + min_p c_p), fp64 means over the counted impressions.

Device memory is bounded by the chunk and the pool, and the result does not depend on the chunk.  The click predictor must be
a dot product of a user vector and a news vector: NRMS, NAML, LSTUR, TANR and Exp1.

    python -m newsrec_b200.pool_eval --directory data/val [--ks 5,10,20,50,100] [--keep-clicked]
                                     [--checkpoint PATH | --checkpoint-dir DIR] [--user2int data/train/user2int.tsv]
                                     [--chunk-impressions N] [--set KNOB=VALUE ...]
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

from . import NewsrecError
from .evaluate import build_tables, new_flag, news_matrix, read_behaviors, user_vectors, _gather
from .recommend import _REFUSED, _Users, exclusion_csr

DEFAULT_KS = (5, 10, 20, 50, 100)
DEFAULT_CHUNK = 65536


def check_request(model, directory, ks):
    """Everything evaluate_pool() refuses before any device work: a K that is not a positive integer, a family whose click
    predictor is not a dot product, a split without behaviors.tsv or news_parsed.tsv, a split without labels."""
    ks = tuple(ks)
    if not ks or any(isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1 for k in ks):
        raise NewsrecError(f"evaluate_pool: ks={ks!r} must be positive integers")
    name = type(model).__name__
    if name in _REFUSED:
        raise NewsrecError(f"evaluate_pool: {name} is not supported: {_REFUSED[name]}")
    for f in ("behaviors.tsv", "news_parsed.tsv"):
        if not os.path.isfile(os.path.join(directory, f)):
            raise FileNotFoundError(f"evaluate_pool: {os.path.join(directory, f)} not found")
    beh = read_behaviors(directory)
    if any("-" not in item for imp in beh["impressions"].tolist() for item in str(imp).split()):
        raise NewsrecError(f"evaluate_pool: {directory}/behaviors.tsv has unlabelled impressions (a test split?): "
                           "retrieval metrics need the clicks")


def positives(cand, labels, seg_offsets):
    """(imp, rows): the impressions with at least one positive and, per impression, its distinct positive rows ascending, as
    CSR (imp (S,) int64 indices into the impressions, rows, offsets (S + 1,))."""
    seg = np.repeat(np.arange(len(seg_offsets) - 1, dtype=np.int64), np.diff(seg_offsets))
    pos = labels == 1
    key = np.unique(np.stack([seg[pos], cand[pos]], axis=1), axis=0) if pos.any() else np.zeros((0, 2), np.int64)
    imp, first = np.unique(key[:, 0], return_index=True)
    offsets = np.append(first, len(key)).astype(np.int64)
    return imp.astype(np.int64), key[:, 1].astype(np.int64), offsets


def positions(rank, score, rows, offsets):
    """c_p of every positive (step 4): its rank among the pool plus the positives of its impression that come before it
    (higher score, then lower row).  rank, score and rows in CSR order over the counted impressions (offsets)."""
    seg = np.repeat(np.arange(len(offsets) - 1, dtype=np.int64), np.diff(offsets))
    order = np.lexsort((rows, -np.asarray(score, np.float64), seg))
    before = np.empty(len(rows), np.int64)
    before[order] = np.arange(len(rows), dtype=np.int64) - offsets[seg[order]]
    return np.asarray(rank, np.int64) + before


def metrics(c, offsets, ks):
    """The dict evaluate_pool returns from the positions c (CSR over the counted impressions): recall@K and nDCG@K per K, and
    MRR, each an fp64 mean over the impressions."""
    S = len(offsets) - 1
    n_pos = np.diff(offsets)
    seg = np.repeat(np.arange(S, dtype=np.int64), n_pos)
    ideal_prefix = np.cumsum(1.0 / np.log2(np.arange(max(int(n_pos.max(initial=0)), 1)) + 2.0))
    out = {}
    for k in ks:
        hit = c < k
        gain = np.where(hit, 1.0 / np.log2(c + 2.0), 0.0)
        out[f"recall@{k}"] = np.float64(np.mean(np.bincount(seg, hit.astype(np.float64), S) / n_pos)) if S else np.float64(np.nan)
        out[f"ndcg@{k}"] = np.float64(np.mean(np.bincount(seg, gain, S) / ideal_prefix[np.minimum(n_pos, k) - 1])) if S else np.float64(np.nan)
    first = np.full(S, np.iinfo(np.int64).max)
    np.minimum.at(first, seg, c)
    out["mrr"] = np.float64(np.mean(1.0 / (1.0 + first))) if S else np.float64(np.nan)
    out["impressions"] = int(S)
    return out


def pool_positions(model, directory, *, exclude_clicked=True, max_count=sys.maxsize, user2int_path="data/train/user2int.tsv",
                   chunk_impressions=DEFAULT_CHUNK):
    """Steps 1-3 of the module: (imp, rows, offsets, rank, score) -- the counted impressions, their positive rows (CSR) and
    each positive's rank and score, on the host."""
    import torch
    from .ops import pool_ranks
    if chunk_impressions < 1:
        raise ValueError(f"evaluate_pool: chunk_impressions={chunk_impressions}")
    with torch.no_grad():
        news_index, matrix = news_matrix(model, directory)
        pad = news_index["PADDED_NEWS"]
        t = build_tables(directory, news_index, model.config.num_clicked_news_a_user, max_count, user2int_path)
        if (t.labels > 1).any():
            raise ValueError("evaluate_pool: a label other than 0 or 1")
        imp, rows, offsets = positives(t.cand, t.labels, t.seg_offsets)
        pool = matrix[:pad]
        flag = new_flag(matrix.device)
        rank, score = np.zeros(len(rows), np.int64), np.zeros(len(rows), np.float32)
        for a in range(0, len(imp), chunk_impressions):
            b = min(len(imp), a + chunk_impressions)
            who, inv = np.unique(t.seg_user[imp[a:b]], return_inverse=True)
            uv = user_vectors(model, _Users(t.user[who], t.history[who], t.history_length[who]), matrix, flag)
            queries = _gather(inv.astype(np.int64), uv, flag)
            excl = None, None
            if exclude_clicked:
                xr, xo = exclusion_csr(t.history[t.seg_user[imp[a:b]]], pad)
                excl = torch.from_numpy(xr), torch.from_numpy(xo)
            lo, hi = offsets[a], offsets[b]
            r, s = pool_ranks(queries, pool, torch.from_numpy(rows[lo:hi]), torch.from_numpy(offsets[a:b + 1] - lo), *excl)
            if int(flag.item()):
                raise IndexError("evaluate_pool: a history row is outside the news table")
            rank[lo:hi], score[lo:hi] = r.cpu().numpy(), s.cpu().numpy()
    return imp, rows, offsets, rank, score


def evaluate_pool(model, directory, ks=DEFAULT_KS, *, exclude_clicked=True, max_count=sys.maxsize,
                  user2int_path="data/train/user2int.tsv", chunk_impressions=DEFAULT_CHUNK):
    """{"recall@K": ..., "ndcg@K": ... for each K, "mrr": ..., "impressions": n} over the impressions of directory/behaviors.tsv
    with at least one click (the first max_count - 1 rows, as evaluate).  Runs under torch.no_grad() on the model as given
    (call .eval() first).  A non-finite score raises ValueError, a history row outside the news table IndexError."""
    check_request(model, directory, ks)
    _, rows, offsets, rank, score = pool_positions(model, directory, exclude_clicked=exclude_clicked, max_count=max_count,
                                                   user2int_path=user2int_path, chunk_impressions=chunk_impressions)
    return metrics(positions(rank, score, rows, offsets), offsets, tuple(int(k) for k in ks))


def parse_ks(text):
    ks = []
    for x in text.split(","):
        try:
            k = int(x)
        except ValueError:
            k = 0
        if k < 1:
            raise ValueError(f"--ks: {x!r} is not a positive integer")
        ks.append(k)
    return tuple(ks)


def parse_args(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--directory", default="./data/val", help="labelled split: news_parsed.tsv (the pool) and behaviors.tsv")
    ap.add_argument("--ks", default=",".join(map(str, DEFAULT_KS)), help="comma-separated cut-offs of recall@K and nDCG@K")
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--checkpoint", help="a checkpoint file (a dict with model_state_dict, as the trainer saves)")
    g.add_argument("--checkpoint-dir", help="load its latest ckpt-<n>.pth (default: ./checkpoint/<MODEL_NAME>)")
    ap.add_argument("--keep-clicked", action="store_true", help="rank a user's clicked news as part of the pool")
    ap.add_argument("--user2int", default="./data/train/user2int.tsv")
    ap.add_argument("--chunk-impressions", type=int, default=DEFAULT_CHUNK, help="impressions ranked per device pass")
    ap.add_argument("--set", action="append", default=[], metavar="KNOB=VALUE",
                    help="override a knob of the selected <MODEL_NAME>Config (repeatable)")
    args = ap.parse_args(argv)
    try:
        args.ks = parse_ks(args.ks)
    except ValueError as e:
        ap.error(str(e))
    if args.chunk_impressions < 1:
        ap.error("--chunk-impressions must be at least 1")
    return args


def main(argv=None):
    from .predict import load_model
    args = parse_args(argv)
    name, path, model = load_model(args.checkpoint, args.checkpoint_dir, args.set)
    out = evaluate_pool(model, args.directory, args.ks, exclude_clicked=not args.keep_clicked, user2int_path=args.user2int,
                        chunk_impressions=args.chunk_impressions)
    print(json.dumps({"model": name, "checkpoint": path, **out}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
