"""newsrec_b200.pool_eval.evaluate_lists without a GPU: the metric assembly (list_metrics) on hand-built lists with known
answers and against the plain restatement of tests/list_eval_ref.py, the refusals raised before any device work and the
--lists command line."""
import math
import os

import numpy as np
import pytest

import list_eval_ref as R
from newsrec_b200 import NewsrecError
from newsrec_b200 import pool_eval as P


def _csr(positives):
    offsets = np.zeros(len(positives) + 1, np.int64)
    offsets[1:] = np.cumsum([len(p) for p in positives])
    rows = np.array([r for p in positives for r in sorted(p)], np.int64)
    return rows, offsets


def _inv(c):
    return 1.0 / math.log2(c + 2)


def test_hand_built_lists():
    # a capped run's lines: shortened, one empty; positives listed, absent, and one line without any listed
    lists = np.array([[3, 1, 4, -1], [0, 2, -1, -1], [5, -1, -1, -1], [-1, -1, -1, -1]])
    positives = [[1, 5], [0], [2], [3]]
    rows, offsets = _csr(positives)
    ks = (1, 2, 4)
    pair_sum = np.array([[0.0, 0.2, 1.5], [0.0, 0.25, 0.25], [0.0, 0.0, 0.0], [0.0, 0.0, 0.0]])
    distinct = np.array([[1, 2, 2], [1, 1, 1], [1, 1, 1], [0, 0, 0]])
    m = P.list_metrics(lists, rows, offsets, pair_sum, distinct, 6, ks, "category")
    assert m["impressions"] == 4
    assert m["recall@1"] == 0.25 and m["recall@2"] == 0.375 and m["recall@4"] == 0.375
    assert m["ndcg@1"] == 0.25
    assert m["ndcg@2"] == pytest.approx((_inv(1) / (1 + _inv(1)) + 1) / 4, abs=1e-15)
    assert m["mrr@4"] == 0.375                                        # 1/2, 1, 0, 0
    assert math.isnan(m["ils@1"]) and m["ils@2"] == pytest.approx(0.225) and m["ils@4"] == pytest.approx(0.375)
    assert m["list_length@1"] == 0.75 and m["list_length@2"] == 1.25 and m["list_length@4"] == 1.5
    assert m["distinct_category@2"] == 1.0 and m["distinct_category@4"] == 1.0
    assert m["coverage@1"] == 0.5 and m["coverage@4"] == 1.0
    assert m["gini@4"] == 0.0                                         # every news listed once: equal exposure
    assert all(isinstance(v, np.float64) for key, v in m.items() if key != "impressions")
    R.assert_close(m, R.metrics(lists, positives, 6, ks, pair_sum, distinct))
    # ILS with lists of 0, 1 and 2 live entries: only the last qualifies
    m = P.list_metrics(np.array([[-1, -1], [4, -1], [1, 2]]), *_csr([[1], [1], [1]]), np.array([[0.0], [0.0], [0.6]]), None, 5,
                       (2,))
    assert m["ils@2"] == pytest.approx(0.6) and "distinct_category@2" not in m and m["list_length@2"] == 1.0
    assert m["recall@2"] == pytest.approx(1 / 3) and m["mrr@2"] == pytest.approx(1 / 3)


def test_gini_and_coverage():
    n = 5
    one = np.full((7, 1), 2)                                          # one news takes every exposure
    m = P.list_metrics(one, *_csr([[2]] * 7), np.zeros((7, 1)), None, n, (1,))
    assert m["gini@1"] == pytest.approx((n - 1) / n, abs=1e-15) and m["coverage@1"] == 1 / n and m["recall@1"] == 1.0
    assert P.gini([3, 3, 3, 3]) == 0.0 and math.isnan(P.gini([0, 0, 0]))
    assert P.gini([0, 0, 0, 10]) == pytest.approx(3 / 4, abs=1e-15)
    empty = P.list_metrics(np.zeros((0, 3), np.int64), np.zeros(0, np.int64), np.zeros(1, np.int64), np.zeros((0, 2)),
                           np.zeros((0, 2)), 4, (1, 3))
    assert empty["impressions"] == 0 and empty["coverage@3"] == 0.0
    assert all(math.isnan(empty[key]) for key in ("recall@1", "mrr@3", "ils@3", "gini@3", "list_length@1"))


@pytest.mark.parametrize("seed", range(5))
def test_random_lists_agree_with_the_restatement(seed):
    rng = np.random.default_rng(seed)
    n, k, S = 40, 12, 60
    ks = (1, 3, 5, 12)
    lists = np.full((S, k), -1, np.int64)
    positives = []
    for i in range(S):
        L = int(rng.integers(0, k + 1))
        lists[i, :L] = rng.choice(n, L, replace=False)
        lists[i, L:][rng.random(k - L) < 0.3] = 7                    # entries after the first -1 are ignored
        if L < k:
            lists[i, L] = -1
        positives.append(sorted(set(rng.choice(n, int(rng.integers(1, 5)), replace=False).tolist())))
    news = rng.standard_normal((n, 9)).astype(np.float32)
    news[3] = 0
    cats = rng.integers(-3, 4, n)
    ps, dc = R.list_stats(news, lists, ks, cats)
    got = P.list_metrics(lists, *_csr(positives), ps, dc, n, ks, "subcategory")
    R.assert_close(got, R.metrics(lists, positives, n, ks, ps, dc, "subcategory"))


class _Cfg:
    num_clicked_news_a_user = 4


def _fake(name):
    return type(name, (), {"config": _Cfg})()


def _split(d, labelled=True, category=True):
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\ttitle\nN1\t1\t[1]\nN2\t2\t[2]\n" if category else "id\ttitle\nN1\t[1]\nN2\t[2]\n")
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write("1\tU1\tt\tN1\tN2-1 N1-0\n" if labelled else "1\tU1\tt\tN1\tN2 N1\n")


def test_refusals_come_before_the_device(tmp_path):
    # the fake models have no encoders: reaching the device work would raise AttributeError, not these
    d = str(tmp_path)
    _split(d)
    nrms = _fake("NRMS")
    for kw, why in ((dict(k=0), "k="), (dict(k=129), "k="), (dict(k=True), "k="),
                    (dict(ks=()), "ks="), (dict(ks=(0,)), "ks="), (dict(ks=(11,)), "ks="), (dict(ks=(2.0,)), "ks="),
                    (dict(ks=(True,)), "ks="), (dict(k=20, ks=tuple(range(1, 10))), "at most 8"),
                    (dict(max_per_category=0), "max_per_category"), (dict(diversify_by="topic"), "diversify_by"),
                    (dict(mmr_lambda=1.5), "mmr_lambda"), (dict(mmr_lambda=float("nan")), "mmr_lambda"),
                    (dict(mmr_depth=40), "needs mmr_lambda"), (dict(mmr_lambda=0.5, mmr_depth=5), "mmr_depth"),
                    (dict(mmr_lambda=0.5, max_per_category=2), "do not combine")):
        with pytest.raises(NewsrecError, match=why):
            P.evaluate_lists(nrms, d, **kw)
    for name, why in (("HiFiArk", "similarity attention"), ("DKN", "DNN click predictor")):
        with pytest.raises(NewsrecError, match="evaluate_lists: .*" + why):
            P.evaluate_lists(_fake(name), d)
    assert P.check_lists_request(nrms, d, 10) == (5, 10)
    assert P.check_lists_request(nrms, d, 20, (20, 3, 3)) == (3, 20)
    assert P.check_lists_request(nrms, d, 3) == (3,)
    with pytest.raises(ValueError, match="chunk_impressions"):
        P.evaluate_lists(nrms, d, chunk_impressions=0)
    _split(d, category=False)
    with pytest.raises(NewsrecError, match="no subcategory column"):
        P.evaluate_lists(nrms, d, max_per_category=1, diversify_by="subcategory")
    P.check_lists_request(nrms, d, 10, mmr_lambda=0.5)                # no column is needed without a cap
    _split(d, labelled=False)
    with pytest.raises(NewsrecError, match="evaluate_lists: .*unlabelled"):
        P.evaluate_lists(nrms, d)
    os.remove(os.path.join(d, "behaviors.tsv"))
    with pytest.raises(FileNotFoundError, match="behaviors.tsv"):
        P.evaluate_lists(nrms, d)


def test_cli_lists():
    a = P.parse_args(["--lists"])
    assert (a.lists, a.k, a.ks, a.max_per_category, a.mmr_lambda, a.mmr_depth, a.diversify_by) == \
        (True, 10, (5, 10), None, None, None, "category")
    a = P.parse_args(["--lists", "--k", "30", "--ks", "30,1,7", "--mmr-lambda", "0.5", "--mmr-depth", "64"])
    assert (a.k, a.ks, a.mmr_lambda, a.mmr_depth) == (30, (1, 7, 30), 0.5, 64)
    a = P.parse_args(["--lists", "--k", "3", "--max-per-category", "1", "--diversify-by", "subcategory", "--keep-clicked"])
    assert (a.k, a.ks, a.max_per_category, a.diversify_by, a.keep_clicked) == (3, (3,), 1, "subcategory", True)
    a = P.parse_args([])                                              # without --lists: as before
    assert not a.lists and a.ks == (5, 10, 20, 50, 100) and a.directory == "./data/val"
    for bad in (["--k", "10"], ["--max-per-category", "2"], ["--mmr-lambda", "0.5"], ["--mmr-depth", "40"],
                ["--diversify-by", "category"],
                ["--lists", "--ks", "11"], ["--lists", "--k", "5", "--ks", "1,6"], ["--lists", "--k", "0"],
                ["--lists", "--k", "129"], ["--lists", "--ks", "0"], ["--lists", "--k", "20", "--ks", "1,2,3,4,5,6,7,8,9"],
                ["--lists", "--max-per-category", "2", "--mmr-lambda", "0.5"], ["--lists", "--max-per-category", "0"],
                ["--lists", "--mmr-lambda", "2"], ["--lists", "--mmr-depth", "40"],
                ["--lists", "--mmr-lambda", "0.5", "--mmr-depth", "5"], ["--lists", "--diversify-by", "topic"]):
        with pytest.raises(SystemExit):
            P.parse_args(bad)
