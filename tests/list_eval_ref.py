"""Plain restatement of newsrec_b200.pool_eval.evaluate_lists' metrics, one impression at a time in fp64, and of
nr_list_stats' pair sums and distinct counts (include/newsrec_b200.h).

For impression i with list l_i (the entries before the first -1) and positives P_i, c_p = p's 0-based place in l_i or absent:
    recall@K   |{p : c_p < K}| / |P_i|
    ndcg@K     sum_{c_p < K} 1 / log2(c_p + 2) / sum_{j < min(|P_i|, K)} 1 / log2(j + 2)
    mrr@k      1 / (1 + min_p c_p), 0 when no positive is listed
    ils@K      mean cosine over the pairs of the first K' = min(K, |l_i|) entries, over the lists with K' >= 2
    distinct   distinct category keys among the first K'
    coverage   |news in some first-K list| / n_pool
    gini       sum_i (2i - n - 1) x_(i) / (n sum x) over the per-news exposure counts x, ascending, i from 1
    length     K'
each (but coverage and gini) a mean over the impressions."""
import math

import numpy as np


def live(row):
    out = []
    for r in row:
        if r < 0:
            break
        out.append(int(r))
    return out


def cosine_pairs(news, row):
    """sum over i < j of the fp64 cosine of news rows row[i] and row[j] (0 for a zero row)."""
    X = np.asarray(news, np.float32).astype(np.float64)[np.asarray(row, np.int64)] if len(row) else np.zeros((0, 1))
    nrm = np.linalg.norm(X, axis=1)
    Xn = np.divide(X, nrm[:, None], out=np.zeros_like(X), where=nrm[:, None] > 0)
    G = Xn @ Xn.T
    return float(sum(G[i, j] for j in range(len(row)) for i in range(j)))


def list_stats(news, lists, ks, categories=None):
    """(pair_sum (S, n_ks) fp64 of exact cosines, distinct (S, n_ks) int64 or None), nr_list_stats' contract."""
    S = len(lists)
    ps = np.zeros((S, len(ks)))
    dc = np.zeros((S, len(ks)), np.int64) if categories is not None else None
    for s, row in enumerate(lists):
        lv = live(row)
        for c, K in enumerate(ks):
            head = lv[:K]
            ps[s, c] = cosine_pairs(news, head)
            if dc is not None:
                dc[s, c] = len({int(categories[r]) for r in head})
    return ps, dc


def metrics(lists, positives, n_pool, ks, pair_sum, distinct=None, field="category"):
    """The evaluate_lists dict from lists (S, k), positives (S lists of distinct rows), pair_sum / distinct (S, n_ks)."""
    S, k = len(lists), len(lists[0]) if len(lists) else 0
    lv = [live(r) for r in lists]
    out = {}
    for K in ks:
        rec, nd = [], []
        for i in range(S):
            pos = positives[i]
            c = {p: lv[i].index(p) for p in pos if p in lv[i]}
            rec.append(sum(1 for p in pos if p in c and c[p] < K) / len(pos))
            ideal = sum(1 / math.log2(j + 2) for j in range(min(len(pos), K)))
            nd.append(sum(1 / math.log2(c[p] + 2) for p in pos if p in c and c[p] < K) / ideal)
        out[f"recall@{K}"] = float(np.mean(rec)) if S else math.nan
        out[f"ndcg@{K}"] = float(np.mean(nd)) if S else math.nan
    rr = []
    for i in range(S):
        places = [lv[i].index(p) for p in positives[i] if p in lv[i]]
        rr.append(1 / (1 + min(places)) if places else 0.0)
    out[f"mrr@{k}"] = float(np.mean(rr)) if S else math.nan
    for c, K in enumerate(ks):
        Kp = [min(K, len(x)) for x in lv]
        ils = [pair_sum[i][c] / (Kp[i] * (Kp[i] - 1) / 2) for i in range(S) if Kp[i] >= 2]
        out[f"ils@{K}"] = float(np.mean(ils)) if ils else math.nan
        if distinct is not None:
            out[f"distinct_{field}@{K}"] = float(np.mean([distinct[i][c] for i in range(S)])) if S else math.nan
        x = [0] * n_pool
        for i in range(S):
            for r in lv[i][:K]:
                x[r] += 1
        out[f"coverage@{K}"] = sum(1 for v in x if v) / n_pool
        xs = sorted(x)
        tot = sum(xs)
        out[f"gini@{K}"] = sum((2 * j - n_pool - 1) * v for j, v in enumerate(xs, 1)) / (n_pool * tot) if tot else math.nan
        out[f"list_length@{K}"] = float(np.mean(Kp)) if S else math.nan
    out["impressions"] = S
    return out


def assert_close(got, want, rel=1e-12, tol=None):
    """Same keys; every value within rel (or tol[key]) of want, NaN where want is NaN."""
    assert set(got) == set(want), (sorted(set(got) ^ set(want)))
    for key, w in want.items():
        g = got[key]
        if isinstance(w, float) and math.isnan(w):
            assert math.isnan(g), (key, g)
            continue
        t = (tol or {}).get(key, rel * max(1.0, abs(w)))
        assert abs(g - w) <= t, (key, g, w)
