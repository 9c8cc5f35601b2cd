"""newsrec_b200.pool_eval and ops.target_parts without a GPU: the metrics from hand-worked ranks, the positives of each
impression, the CSR that splits a query of more than 32 targets, the refusals raised before any device work and the CLI."""
import math
import os

import numpy as np
import pytest

from newsrec_b200 import NewsrecError
from newsrec_b200 import pool_eval as P
from newsrec_b200.ops import target_parts


def _inv(c):
    return 1.0 / math.log2(c + 2)


def test_metrics_from_hand_worked_ranks():
    # impression 0: rows 3 (score 1, rank 0) and 7 (score 2, rank 2): 7 comes first, so c_7 = 2 + 0 and c_3 = 0 + 1.
    # impression 1: rows 5 and 9 tie at 0.5, both of rank 4: the lower row first, c_5 = 4 and c_9 = 5.
    # impression 2: one positive of rank 0.
    rows = np.array([3, 7, 5, 9, 11])
    rank = np.array([0, 2, 4, 4, 0])
    score = np.array([1.0, 2.0, 0.5, 0.5, -3.0], np.float32)
    offsets = np.array([0, 2, 4, 5])
    c = P.positions(rank, score, rows, offsets)
    assert c.tolist() == [1, 2, 4, 5, 0]
    m = P.metrics(c, offsets, (1, 2, 5, 1000))
    assert m["impressions"] == 3
    assert m["recall@1"] == pytest.approx((0 + 0 + 1) / 3)
    assert m["recall@2"] == pytest.approx((0.5 + 0 + 1) / 3)
    assert m["recall@5"] == pytest.approx((1 + 0.5 + 1) / 3)
    assert m["recall@1000"] == 1.0                                  # K larger than the pool
    idcg2 = 1 + _inv(1)
    assert m["ndcg@1"] == pytest.approx((0 + 0 + 1) / 3)
    assert m["ndcg@2"] == pytest.approx((_inv(1) / idcg2 + 0 + 1) / 3)
    assert m["ndcg@5"] == pytest.approx(((_inv(1) + _inv(2)) / idcg2 + _inv(4) / idcg2 + 1) / 3)
    assert m["ndcg@1000"] == pytest.approx(((_inv(1) + _inv(2)) / idcg2 + (_inv(4) + _inv(5)) / idcg2 + 1) / 3)
    assert m["mrr"] == pytest.approx((1 / 2 + 1 / 5 + 1) / 3)
    assert all(isinstance(v, np.float64) for k, v in m.items() if k != "impressions")
    empty = P.metrics(np.zeros(0, np.int64), np.zeros(1, np.int64), (5,))
    assert empty["impressions"] == 0 and np.isnan(empty["recall@5"]) and np.isnan(empty["mrr"])


def test_positives_skip_impressions_without_a_click_and_count_a_duplicate_once():
    cand = np.array([4, 2, 2, 9, 1, 1, 6, 3, 8])
    labels = np.array([0, 1, 1, 1, 0, 0, 0, 1, 0], np.uint8)
    seg_offsets = np.array([0, 4, 6, 6, 9])                        # impression 1 has no click, 2 no candidate
    imp, rows, offsets = P.positives(cand, labels, seg_offsets)
    assert imp.tolist() == [0, 3]
    assert rows.tolist() == [2, 9, 3] and offsets.tolist() == [0, 2, 3]
    imp, rows, offsets = P.positives(cand, np.zeros(9, np.uint8), seg_offsets)
    assert imp.size == 0 and rows.size == 0 and offsets.tolist() == [0]


def test_target_parts_split_a_query_of_more_than_32_targets():
    tr = np.arange(100, 170)
    to = np.array([0, 3, 3, 70])                                   # 3 targets, none, 67 targets
    xr, xo = np.array([5, 6, 7]), np.array([0, 1, 1, 3])
    query, offsets, er, eo = target_parts(tr, to, xr, xo)
    assert query.tolist() == [0, 2, 2, 2]
    assert offsets.tolist() == [0, 3, 35, 67, 70]                  # consecutive: the caller's target order
    parts = [er[eo[i]:eo[i + 1]].tolist() for i in range(4)]
    assert parts[0] == [5]
    for p, (a, b) in zip(parts[1:], [(3, 35), (35, 67), (67, 70)]):
        others = [int(x) for x in tr[3:70] if not tr[a] <= x < tr[b - 1] + 1]
        assert p[:2] == [6, 7] and sorted(p[2:]) == others
        assert len(p) == 2 + 67 - (b - a)
    query, offsets, er, eo = target_parts(tr[:32], np.array([0, 32]))
    assert query.tolist() == [0] and offsets.tolist() == [0, 32] and er.size == 0 and eo.tolist() == [0, 0]
    query, offsets, er, eo = target_parts(tr[:33], np.array([0, 33]))
    assert offsets.tolist() == [0, 32, 33] and [er[eo[i]:eo[i + 1]].tolist() for i in range(2)] == [[132], tr[:32].tolist()]
    query, offsets, er, eo = target_parts(np.zeros(0), np.array([0, 0, 0]))
    assert query.size == 0 and offsets.tolist() == [0] and eo.tolist() == [0]


class _Cfg:
    num_clicked_news_a_user = 4


def _fake(name):
    return type(name, (), {"config": _Cfg})()


def _split(d, labelled=True):
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write("id\ttitle\nN1\t[1]\nN2\t[2]\n")
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write("1\tU1\tt\tN1\tN2-1 N1-0\n" if labelled else "1\tU1\tt\tN1\tN2 N1\n")


def test_refusals_come_before_the_device(tmp_path):
    d = str(tmp_path)
    _split(d)
    for name, why in (("HiFiArk", "similarity attention"), ("DKN", "DNN click predictor")):
        with pytest.raises(NewsrecError, match=why):
            P.evaluate_pool(_fake(name), d)
    for ks in ((), (0,), (5, -1), (2.5,), (True,)):
        with pytest.raises(NewsrecError, match="ks="):
            P.evaluate_pool(_fake("NRMS"), d, ks)
    P.check_request(_fake("NRMS"), d, (5, 10))
    _split(d, labelled=False)
    with pytest.raises(NewsrecError, match="unlabelled"):
        P.evaluate_pool(_fake("NRMS"), d)
    os.remove(os.path.join(d, "news_parsed.tsv"))
    with pytest.raises(FileNotFoundError, match="news_parsed.tsv"):
        P.evaluate_pool(_fake("LSTUR"), d)


def test_cli_arguments():
    a = P.parse_args(["--directory", "x", "--ks", "1,7,20", "--checkpoint", "c.pth", "--keep-clicked",
                      "--chunk-impressions", "3", "--set", "batch_size=2", "--user2int", "u.tsv"])
    assert (a.directory, a.ks, a.checkpoint, a.keep_clicked, a.chunk_impressions, a.set, a.user2int) == \
        ("x", (1, 7, 20), "c.pth", True, 3, ["batch_size=2"], "u.tsv")
    a = P.parse_args([])
    assert a.ks == (5, 10, 20, 50, 100) and not a.keep_clicked and a.checkpoint is None and a.checkpoint_dir is None
    assert a.directory == "./data/val" and a.chunk_impressions == P.DEFAULT_CHUNK
    for bad in (["--ks", "0"], ["--ks", "5,x"], ["--ks", ""], ["--ks", "5,,10"], ["--chunk-impressions", "0"],
                ["--checkpoint", "a", "--checkpoint-dir", "b"]):
        with pytest.raises(SystemExit):
            P.parse_args(bad)
