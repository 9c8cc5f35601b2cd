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

Device memory is bounded by the chunk and the pool, and the result does not depend on the chunk.  NRMS, NAML, LSTUR, TANR and
Exp1 are ranked under the dot product of user and news vectors; Hi-Fi Ark and DKN under their DNN click predictor, through
their models' ``pool_user_vector`` and ``ops.pool_ranks(..., dnn=)`` (nr_pool_ranks_archive: the scores nr_topk_archive
computes).  A model of those two families without ``pool_user_vector`` is refused.

``evaluate_lists`` (``--lists``) evaluates the k-lists ``recommend`` writes instead, plain, capped (``max_per_category``) or
MMR re-ranked (``mmr_lambda``), over the same impressions: where each click lands in its user's list (recall@K, nDCG@K,
MRR) and how the lists look (intra-list similarity, distinct categories, catalog coverage, exposure Gini), the similarity
statistics from one kernel (``ops.list_stats``, nr_list_stats).

Live news only (``max_age_hours=H``, ``--max-age-hours H``, both modes): each impression only ranks and lists the news first
shown in ``behaviors.tsv`` within H hours before its own time (``window``: the definition and the time order the device
work runs in), so the numbers are the ones a feed serving live news would see; without it every news of the split is in
every impression's pool, future and stale news included.  A click first shown before the window is still ranked, against
the window's news.  The result adds ``max_age_hours``, ``pool_size_mean`` (the mean eligible pool over the counted
impressions) and ``targets_outside_window`` (the clicks first shown before their impression's window); with ``--lists``
coverage and Gini are taken over the news eligible for at least one counted impression, ``n_pool`` of them.  Each chunk's
impressions are sorted by time, so a block of 64 shares nearly one window; the result does not depend on the chunk.

    python -m newsrec_b200.pool_eval --directory data/val [--ks 5,10,20,50,100] [--keep-clicked] [--max-age-hours H]
                                     [--checkpoint PATH | --checkpoint-dir DIR] [--user2int data/train/user2int.tsv]
                                     [--chunk-impressions N] [--set KNOB=VALUE ...]
                                     [--lists [--k 10] [--max-per-category M [--diversify-by {category,subcategory}]
                                                        | --mmr-lambda X [--mmr-depth L]]]
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

from . import NewsrecError, window
from .evaluate import build_tables, new_flag, news_matrix, read_behaviors, read_news, _gather
from .recommend import (DIVERSIFY_FIELDS, MAX_K, _Users, add_diversify_args, add_window_arg, check_diversify_args,
                        check_window_arg, exclusion_csr, list_options, news_columns, pool_operands, refuse_family,
                        time_ordered)
from .recommend import check_request as check_list_request

DEFAULT_KS = (5, 10, 20, 50, 100)
DEFAULT_CHUNK = 65536


def check_request(model, directory, ks, max_age_hours=None):
    """Everything evaluate_pool() refuses before any device work: a K that is not a positive integer, a family whose click
    predictor is not a dot product, a max_age_hours that is not a real number > 0, a split without behaviors.tsv or
    news_parsed.tsv, a split without labels, and (with max_age_hours) a behaviors.tsv time that does not parse.  Returns
    window.load's (W, behaviors, times), or None without max_age_hours."""
    ks = tuple(ks)
    if not ks or any(isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 1 for k in ks):
        raise NewsrecError(f"evaluate_pool: ks={ks!r} must be positive integers")
    refuse_family("evaluate_pool", model)
    if max_age_hours is not None:
        window.max_age_seconds("evaluate_pool", max_age_hours)
    for f in ("behaviors.tsv", "news_parsed.tsv"):
        if not os.path.isfile(os.path.join(directory, f)):
            raise FileNotFoundError(f"evaluate_pool: {os.path.join(directory, f)} not found")
    require_labels("evaluate_pool", directory)
    return window.load("evaluate_pool", directory, max_age_hours)


def require_labels(who, directory):
    """Raises NewsrecError when directory/behaviors.tsv has an impression without labels."""
    beh = read_behaviors(directory)
    if any("-" not in item for imp in beh["impressions"].tolist() for item in str(imp).split()):
        raise NewsrecError(f"{who}: {directory}/behaviors.tsv has unlabelled impressions (a test split?): "
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
    return _positions(model, directory, None, exclude_clicked, max_count, user2int_path, chunk_impressions)[:5]


class _Window:
    """A windowed call's time order over the pool of news_ids and its counted impressions' ranges."""

    def __init__(self, win, news_ids, times_of_rows):
        W, beh, times = win
        self.W = W
        self.pw = window.pool_window(beh, times, news_ids)
        self.t = times[times_of_rows]
        self.lo, self.hi = self.pw.ranges(self.t, W)

    def stats(self, rows, offsets, max_age_hours):
        """The keys a windowed result adds: max_age_hours, pool_size_mean and targets_outside_window (the positives rows,
        CSR offsets, first shown before their impression's window)."""
        seg = np.repeat(np.arange(len(offsets) - 1, dtype=np.int64), np.diff(offsets))
        before = self.pw.to_time_order(rows) < self.lo[seg]
        return {"max_age_hours": float(max_age_hours),
                "pool_size_mean": float(np.mean(self.hi - self.lo)) if len(self.lo) else float("nan"),
                "targets_outside_window": int(np.count_nonzero(before))}

    def eligible_rows(self):
        """(n,) bool: the pool rows eligible for at least one counted impression."""
        n = len(self.pw.perm)
        d = np.zeros(n + 1, np.int64)
        np.add.at(d, self.lo, 1)
        np.add.at(d, self.hi, -1)
        out = np.zeros(n, bool)
        out[self.pw.perm] = np.cumsum(d[:n]) > 0
        return out


def _positions(model, directory, win, exclude_clicked, max_count, user2int_path, chunk_impressions):
    """pool_positions, and with win (window.load's) each impression ranked against the news live at its time; returns
    (imp, rows, offsets, rank, score, the _Window or None)."""
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
        w = None
        if win is not None:
            w = _Window(win, read_news(directory, [])[0], imp)
            pool, _ = time_ordered(w.pw, pool, {})
        flag = new_flag(matrix.device)
        rank, score = np.zeros(len(rows), np.int64), np.zeros(len(rows), np.float32)
        for a in range(0, len(imp), chunk_impressions):
            b = min(len(imp), a + chunk_impressions)
            lo, hi = offsets[a], offsets[b]
            sel, tgt, tgt_offsets, at, row_range = slice(a, b), rows[lo:hi], offsets[a:b + 1] - lo, slice(lo, hi), None
            if w is not None:  # by time within the chunk: a block of 64 impressions shares nearly one window
                order = np.argsort(w.t[a:b], kind="stable")
                sel = a + order
                gather, tgt_offsets = window.csr_take(offsets[a:b + 1] - lo, order)
                at = lo + gather
                tgt = w.pw.to_time_order(rows[at])
                row_range = torch.from_numpy(w.lo[sel]), torch.from_numpy(w.hi[sel])
            who, inv = np.unique(t.seg_user[imp[sel]], return_inverse=True)
            uv, dnn = pool_operands(model, _Users(t.user[who], t.history[who], t.history_length[who]), matrix, flag)
            queries = _gather(inv.astype(np.int64), uv.reshape(uv.shape[0], -1), flag).view(-1, *uv.shape[1:])
            excl = None, None
            if exclude_clicked:
                xr, xo = exclusion_csr(t.history[t.seg_user[imp[sel]]], pad)
                if w is not None:
                    xr = w.pw.to_time_order(xr)
                excl = torch.from_numpy(xr), torch.from_numpy(xo)
            r, s = pool_ranks(queries, pool, torch.from_numpy(tgt), torch.from_numpy(tgt_offsets), *excl, dnn=dnn,
                              row_range=row_range)
            if int(flag.item()):
                raise IndexError("evaluate_pool: a history row is outside the news table")
            rank[at], score[at] = r.cpu().numpy(), s.cpu().numpy()
    return imp, rows, offsets, rank, score, w


def evaluate_pool(model, directory, ks=DEFAULT_KS, *, exclude_clicked=True, max_count=sys.maxsize,
                  user2int_path="data/train/user2int.tsv", chunk_impressions=DEFAULT_CHUNK, max_age_hours=None):
    """{"recall@K": ..., "ndcg@K": ... for each K, "mrr": ..., "impressions": n} over the impressions of directory/behaviors.tsv
    with at least one click (the first max_count - 1 rows, as evaluate).  Runs under torch.no_grad() on the model as given
    (call .eval() first).  A non-finite score raises ValueError, a history row outside the news table IndexError.  With
    max_age_hours each impression's pool is the news live at its time, and the result adds max_age_hours, pool_size_mean
    and targets_outside_window (module docstring)."""
    win = check_request(model, directory, ks, max_age_hours)
    _, rows, offsets, rank, score, w = _positions(model, directory, win, exclude_clicked, max_count, user2int_path,
                                                  chunk_impressions)
    out = metrics(positions(rank, score, rows, offsets), offsets, tuple(int(k) for k in ks))
    if w is not None:
        out.update(w.stats(rows, offsets, max_age_hours))
    return out


# ---- the lists recommend writes ----
LIST_MAX_KS = 8  # cut-offs of one evaluate_lists call (nr_list_stats)


def list_ks(k, ks=None):
    """The cut-offs of evaluate_lists, ascending and distinct: by default the DEFAULT_KS below k, then k.  Raises
    NewsrecError on a K that is not an integer in [1, k] or on more than 8 distinct cut-offs."""
    if ks is None:
        return tuple(x for x in DEFAULT_KS if x < k) + (int(k),)
    ks = tuple(ks)
    if not ks or any(isinstance(x, bool) or not isinstance(x, (int, np.integer)) or not 1 <= x <= k for x in ks):
        raise NewsrecError(f"evaluate_lists: ks={ks!r} must be integers in [1, k] = [1, {k}]")
    ks = tuple(sorted(set(int(x) for x in ks)))
    if len(ks) > LIST_MAX_KS:
        raise NewsrecError(f"evaluate_lists: {len(ks)} distinct cut-offs; at most {LIST_MAX_KS}")
    return ks


def check_lists_request(model, directory, k, ks=None, max_per_category=None, diversify_by="category", mmr_lambda=None,
                        mmr_depth=None, max_age_hours=None):
    """Everything evaluate_lists() refuses, before any device work: every refusal of recommend.check_request (k, the cap, the
    field, the family, MMR, MMR together with a cap, missing files, the window), a bad ks (list_ks) and an unlabelled
    split.  Returns the cut-offs, or (cut-offs, window.load's) with max_age_hours."""
    win = check_list_request(model, directory, k, max_per_category, diversify_by, mmr_lambda, mmr_depth, who="evaluate_lists",
                             max_age_hours=max_age_hours)
    ks = list_ks(int(k), ks)
    require_labels("evaluate_lists", directory)
    return ks if max_age_hours is None else (ks, win)


def list_lengths(lists):
    """The number of entries before the first -1 of every row of lists (S, k)."""
    dead = np.asarray(lists) < 0
    return np.where(dead.any(1), dead.argmax(1), dead.shape[1]).astype(np.int64)


def gini(x):
    """Gini coefficient of the counts x (every item, zeros included): sum_i (2i - n - 1) x_(i) / (n sum x), x ascending, i
    from 1; NaN when sum x = 0.  The numerator is an exact integer sum."""
    x = np.sort(np.asarray(x, np.int64))
    n, total = len(x), int(x.sum())
    if total == 0:
        return np.float64(np.nan)
    w = 2 * np.arange(1, n + 1, dtype=np.int64) - n - 1
    return np.float64(int(np.dot(w, x))) / (np.float64(n) * np.float64(total))


def list_metrics(lists, rows, offsets, pair_sum, distinct, n_pool, ks, field=None, pool=None):
    """The dict evaluate_lists returns, from every counted impression's list and statistics at once:
    lists (S, k) int64 news rows (the entries before the first -1 are the list), rows / offsets the positives (CSR over the
    S impressions), pair_sum (S, len(ks)) fp64 and distinct (S, len(ks)) (or None) from ops.list_stats, n_pool the pool's
    size, ks the ascending cut-offs, field the name of distinct's column.  pool: None (coverage and Gini over all n_pool
    news), or an (n_pool,) bool mask of the news they are taken over, whose size is reported as n_pool."""
    lists = np.asarray(lists, np.int64)
    S, k = lists.shape
    n_pos = np.diff(offsets)
    seg = np.repeat(np.arange(S, dtype=np.int64), n_pos)
    L = list_lengths(lists)
    live = np.arange(k) < L[:, None]
    match = (lists[seg] == np.asarray(rows, np.int64)[:, None]) & live[seg]
    c = np.where(match.any(1), match.argmax(1), k)  # a positive outside the list sits at k: past every cut-off
    out = metrics(c, offsets, ks)
    del out["mrr"], out["impressions"]
    first = np.full(S, k, np.int64)
    np.minimum.at(first, seg, c)
    out[f"mrr@{k}"] = np.float64(np.mean(np.where(first < k, 1.0 / (1.0 + first), 0.0))) if S else np.float64(np.nan)
    for j, K in enumerate(ks):
        Kp = np.minimum(L, K)
        q = Kp >= 2
        out[f"ils@{K}"] = np.float64(np.mean(pair_sum[q, j] / (Kp[q] * (Kp[q] - 1) / 2.0))) if q.any() else np.float64(np.nan)
        if distinct is not None:
            out[f"distinct_{field}@{K}"] = np.float64(np.mean(np.asarray(distinct, np.float64)[:, j])) if S else np.float64(np.nan)
        exposure = np.bincount(lists[:, :K][live[:, :K]], minlength=n_pool)
        n_cov = n_pool
        if pool is not None:
            exposure, n_cov = exposure[pool], int(np.count_nonzero(pool))
        out[f"coverage@{K}"] = np.float64(np.count_nonzero(exposure)) / np.float64(n_cov) if n_cov else np.float64(np.nan)
        out[f"gini@{K}"] = gini(exposure)
        out[f"list_length@{K}"] = np.float64(np.mean(Kp)) if S else np.float64(np.nan)
    out["impressions"] = int(S)
    if pool is not None:
        out["n_pool"] = int(np.count_nonzero(pool))
    return out


def evaluate_lists(model, directory, k=10, ks=None, *, exclude_clicked=True, max_per_category=None, diversify_by="category",
                   mmr_lambda=None, mmr_depth=None, max_count=sys.maxsize, user2int_path="data/train/user2int.tsv",
                   chunk_impressions=DEFAULT_CHUNK, max_age_hours=None) -> dict:
    """Evaluate the k-lists recommend() writes, with the same k, exclusions and cap or MMR knobs, over the impressions
    evaluate_pool counts (at least one click; the first max_count - 1 rows; a positive listed twice counted once; the user
    of an impression is its distinct history).  Each distinct user of a chunk gets its list once (ops.top_k_scores through
    recommend.pool_operands) and its statistics once (ops.list_stats on the model's news vectors); both are gathered per
    impression.  With c_p the 0-based position of positive p in the list (absent: a miss), each an fp64 mean over the
    impressions:
        recall@K, ndcg@K     evaluate_pool's formulas with these c_p;   mrr@k  1 / (1 + min_p c_p), 0 when none is listed;
        ils@K                pair_sum / (K'(K' - 1) / 2) over the lists with K' = min(K, list length) >= 2 (NaN if none);
        distinct_<field>@K   distinct diversify_by values among the first K' (only when news_parsed.tsv has the column);
        coverage@K, gini@K   the share of pool news in some first-K list; the Gini coefficient of the per-news counts of
                             first-K lists holding them, over all pool news (NaN when nothing is listed);
        list_length@K        K';   impressions  the number of counted impressions.
    With exclude_clicked a positive that is in the user's history can never be listed, so it counts as a miss here, while
    evaluate_pool still ranks it.  Every mean is taken once, at the end, from the per-impression values, so the result does
    not depend on chunk_impressions, bit for bit.  Refusals (check_lists_request) come before any device work; a non-finite
    score raises ValueError, a history row outside the news table IndexError.  Runs under torch.no_grad() on the model as
    given (call .eval() first).  With max_age_hours each impression gets its own list, from the news live at its time;
    coverage and Gini are then over the news eligible for at least one counted impression (n_pool), and the result adds
    max_age_hours, pool_size_mean and targets_outside_window (module docstring)."""
    import torch
    from .ops import list_stats, top_k_scores
    ks = check_lists_request(model, directory, k, ks, max_per_category, diversify_by, mmr_lambda, mmr_depth, max_age_hours)
    win = None
    if max_age_hours is not None:
        ks, win = ks
    k = int(k)
    if chunk_impressions < 1:
        raise ValueError(f"evaluate_lists: chunk_impressions={chunk_impressions}")
    with torch.no_grad():
        news_index, matrix = news_matrix(model, directory)
        pad = news_index["PADDED_NEWS"]
        t = build_tables(directory, news_index, model.config.num_clicked_news_a_user, max_count, user2int_path)
        if (t.labels > 1).any():
            raise ValueError("evaluate_lists: a label other than 0 or 1")
        imp, rows, offsets = positives(t.cand, t.labels, t.seg_offsets)
        pool = matrix[:pad]
        opts = list_options("evaluate_lists", directory, matrix.device, max_per_category, diversify_by, mmr_lambda, mmr_depth)
        field = diversify_by if diversify_by in news_columns(directory) else None
        keys = None
        if field is not None:  # distinct counts only need equal keys to stay equal: any key width fits
            raw = read_news(directory, [field])[1][field]
            keys = torch.from_numpy(np.unique(raw, return_inverse=True)[1].reshape(-1).astype(np.int32)).to(matrix.device)
        flag = new_flag(matrix.device)
        S = len(imp)
        lists = np.full((S, k), -1, np.int64)
        pair_sum = np.zeros((S, len(ks)), np.float64)
        distinct = np.zeros((S, len(ks)), np.int64) if field is not None else None
        w = None
        if win is not None:
            w = _Window(win, read_news(directory, [])[0], imp)
            pool, opts = time_ordered(w.pw, pool, opts)
            if keys is not None:
                keys = keys.index_select(0, torch.from_numpy(w.pw.perm).to(keys.device))
        for a in range(0, S, chunk_impressions):
            b = min(S, a + chunk_impressions)
            if w is not None:
                _window_lists(model, t, imp, w, a, b, pad, matrix, pool, keys, flag, exclude_clicked, k, ks, opts,
                              lists, pair_sum, distinct)
                continue
            who, inv = np.unique(t.seg_user[imp[a:b]], return_inverse=True)
            inv = inv.reshape(-1)
            users, dnn = pool_operands(model, _Users(t.user[who], t.history[who], t.history_length[who]), matrix, flag)
            excl = None, None
            if exclude_clicked:
                xr, xo = exclusion_csr(t.history[who], pad)
                excl = torch.from_numpy(xr), torch.from_numpy(xo)
            idx, _ = top_k_scores(users, pool, k, *excl, dnn=dnn, **opts)  # reads its flags: synchronises
            ps, dc = list_stats(pool, idx, ks, categories=keys)
            if int(flag.item()):
                raise IndexError("evaluate_lists: a history row is outside the news table")
            lists[a:b] = idx.cpu().numpy()[inv]
            pair_sum[a:b] = ps.cpu().numpy()[inv]
            if distinct is not None:
                distinct[a:b] = dc.cpu().numpy()[inv]
    if w is None:
        return list_metrics(lists, rows, offsets, pair_sum, distinct, pad, ks, field)
    out = list_metrics(lists, rows, offsets, pair_sum, distinct, pad, ks, field, pool=w.eligible_rows())
    out.update(w.stats(rows, offsets, max_age_hours))
    return out


def _window_lists(model, t, imp, w, a, b, pad, matrix, pool, keys, flag, exclude_clicked, k, ks, opts, lists, pair_sum,
                  distinct):
    """evaluate_lists' chunk [a, b) with a window: one list per impression, from the news live at its time, on the pool in
    time order (pool, keys and opts permuted by time_ordered), sorted by time within the chunk; fills lists (pool rows),
    pair_sum and distinct at the impressions' own places."""
    import torch
    from .ops import list_stats, top_k_scores
    sel = a + np.argsort(w.t[a:b], kind="stable")
    who, inv = np.unique(t.seg_user[imp[sel]], return_inverse=True)
    users, dnn = pool_operands(model, _Users(t.user[who], t.history[who], t.history_length[who]), matrix, flag)
    users = users.index_select(0, torch.from_numpy(inv.reshape(-1).astype(np.int64)).to(users.device))
    excl = None, None
    if exclude_clicked:
        xr, xo = exclusion_csr(t.history[t.seg_user[imp[sel]]], pad)
        excl = torch.from_numpy(w.pw.to_time_order(xr)), torch.from_numpy(xo)
    row_range = torch.from_numpy(w.lo[sel]), torch.from_numpy(w.hi[sel])
    idx, _ = top_k_scores(users, pool, k, *excl, dnn=dnn, row_range=row_range, **opts)  # reads its flags: synchronises
    ps, dc = list_stats(pool, idx, ks, categories=keys)
    if int(flag.item()):
        raise IndexError("evaluate_lists: a history row is outside the news table")
    lists[sel] = w.pw.to_rows(idx).cpu().numpy()
    pair_sum[sel] = ps.cpu().numpy()
    if distinct is not None:
        distinct[sel] = dc.cpu().numpy()


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
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0],
                                 epilog="Every family is served: NRMS, NAML, LSTUR, TANR and Exp1 by the dot product of user and "
                                        "news vectors, Hi-Fi Ark and DKN by their DNN click predictor.")
    ap.add_argument("--directory", default="./data/val", help="labelled split: news_parsed.tsv (the pool) and behaviors.tsv")
    ap.add_argument("--ks", default=None,
                    help="comma-separated cut-offs of recall@K and nDCG@K (default 5,10,20,50,100; with --lists those below "
                         "--k, then --k)")
    g = ap.add_mutually_exclusive_group()
    g.add_argument("--checkpoint", help="a checkpoint file (a dict with model_state_dict, as the trainer saves)")
    g.add_argument("--checkpoint-dir", help="load its latest ckpt-<n>.pth (default: ./checkpoint/<MODEL_NAME>)")
    ap.add_argument("--keep-clicked", action="store_true", help="rank a user's clicked news as part of the pool")
    ap.add_argument("--user2int", default="./data/train/user2int.tsv")
    ap.add_argument("--chunk-impressions", type=int, default=DEFAULT_CHUNK, help="impressions ranked per device pass")
    ap.add_argument("--set", action="append", default=[], metavar="KNOB=VALUE",
                    help="override a knob of the selected <MODEL_NAME>Config (repeatable)")
    ap.add_argument("--lists", action="store_true",
                    help="evaluate the k-lists recommend writes (accuracy and diversity) instead of full-pool ranks")
    ap.add_argument("--k", type=int, default=None, help=f"with --lists: news per list, 1 .. {MAX_K} (default 10)")
    add_diversify_args(ap, None)
    add_window_arg(ap, "rank and list only the news first shown in behaviors.tsv within H hours before each impression "
                       "(inf: every news shown by then)")
    args = ap.parse_args(argv)
    check_window_arg(ap, args)
    if not args.lists:
        for name in ("k", "max_per_category", "diversify_by", "mmr_lambda", "mmr_depth"):
            if getattr(args, name) is not None:
                ap.error(f"--{name.replace('_', '-')} needs --lists")
    try:
        if args.ks is not None:
            args.ks = parse_ks(args.ks)
        elif not args.lists:
            args.ks = DEFAULT_KS
    except ValueError as e:
        ap.error(str(e))
    if args.chunk_impressions < 1:
        ap.error("--chunk-impressions must be at least 1")
    if args.lists:
        if args.k is None:
            args.k = 10
        if not 1 <= args.k <= MAX_K:
            ap.error(f"--k must be in [1, {MAX_K}]")
        check_diversify_args(ap, args)
        if args.diversify_by is None:
            args.diversify_by = DIVERSIFY_FIELDS[0]
        if args.ks is not None and max(args.ks) > args.k:
            ap.error(f"--ks: {max(args.ks)} is above --k {args.k}")
        try:
            args.ks = list_ks(args.k, args.ks)
        except NewsrecError as e:
            ap.error(str(e))
    return args


def main(argv=None):
    from .predict import load_model
    args = parse_args(argv)
    name, path, model = load_model(args.checkpoint, args.checkpoint_dir, args.set)
    if args.lists:
        out = evaluate_lists(model, args.directory, args.k, args.ks, exclude_clicked=not args.keep_clicked,
                             max_per_category=args.max_per_category, diversify_by=args.diversify_by,
                             mmr_lambda=args.mmr_lambda, mmr_depth=args.mmr_depth, user2int_path=args.user2int,
                             chunk_impressions=args.chunk_impressions, max_age_hours=args.max_age_hours)
    else:
        out = evaluate_pool(model, args.directory, args.ks, exclude_clicked=not args.keep_clicked, user2int_path=args.user2int,
                            chunk_impressions=args.chunk_impressions, max_age_hours=args.max_age_hours)
    print(json.dumps({"model": name, "checkpoint": path, **out}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
