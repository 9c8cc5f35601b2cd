"""Hi-Fi Ark and DKN through recommend / evaluate_pool without a GPU: a model that exposes pool_user_vector passes the request
checks (one that does not is still refused), top_k_scores / pool_ranks refuse bad dnn operands before the device, and the
benchmarks' --scorer options parse."""
import argparse
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _split(tmp_path):
    d = str(tmp_path)
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write("id\tcategory\tsubcategory\ttitle\nN1\t1\t2\t[1, 2]\n")
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write("1\tU1\tt\tN1\tN1-1\n")
    return d


class HiFiArk:
    def pool_user_vector(self, clicked):
        return clicked


class DKN(HiFiArk):
    pass


class _Bare:
    pass


@pytest.mark.parametrize("cls", [HiFiArk, DKN])
def test_a_model_with_pool_user_vector_passes_the_checks(cls, tmp_path):
    from newsrec_b200.pool_eval import check_request as pool_check
    from newsrec_b200.recommend import check_request
    d = _split(tmp_path)
    check_request(cls(), d, 10)
    check_request(cls(), d, 10, max_per_category=2)
    check_request(cls(), d, 10, mmr_lambda=0.5)
    pool_check(cls(), d, (5, 10))


@pytest.mark.parametrize("name", ["HiFiArk", "DKN"])
def test_a_model_without_pool_user_vector_is_still_refused(name, tmp_path):
    from newsrec_b200 import NewsrecError
    from newsrec_b200.pool_eval import check_request as pool_check
    from newsrec_b200.recommend import check_request
    d = _split(tmp_path)
    model = type(name, (_Bare,), {})()
    with pytest.raises(NewsrecError, match=f"{name} is not supported"):
        check_request(model, d, 10)
    with pytest.raises(NewsrecError, match=f"{name} is not supported"):
        pool_check(model, d, (5,))


def test_bad_dnn_operands_are_refused_before_the_device(monkeypatch):
    from newsrec_b200 import NewsrecError, ops

    def boom():
        raise AssertionError("the device was touched")
    monkeypatch.setattr(ops, "require_cuda", boom)
    F, hid = 8, 4
    news = torch.zeros(10, F)
    dnn = (torch.zeros(hid, 2 * F), torch.zeros(hid), torch.zeros(1, hid), torch.zeros(1))
    for users, d in ((torch.zeros(3, 2, F + 1), dnn), (torch.zeros(3, 2, 2, F), dnn), (torch.zeros(3, F), dnn[:3]),
                     (torch.zeros(3, F), (torch.zeros(hid, F),) + dnn[1:]), (torch.zeros(3, F), dnn[:1] + (torch.zeros(5),) + dnn[2:]),
                     (torch.zeros(3, F), dnn[:3] + (torch.zeros(2),))):
        with pytest.raises(NewsrecError):
            ops.top_k_scores(users, news, 5, dnn=d)
        with pytest.raises(NewsrecError):
            ops.pool_ranks(users, news, torch.zeros(0, dtype=torch.int64), torch.zeros(users.shape[0] + 1, dtype=torch.int64),
                           dnn=d)


@pytest.mark.parametrize("scorer", ["dot", "hifiark", "dkn"])
def test_bench_scorer_options_parse(scorer):
    import archive_pool_bench
    ap = argparse.ArgumentParser()
    archive_pool_bench.add_args(ap)
    a = ap.parse_args(["--scorer", scorer, "--baseline-users", "100", "--sample-users", "8"])
    assert (a.scorer, a.baseline_users, a.sample_users) == (scorer, 100, 8)
    assert ap.parse_args([]).scorer == "dot"
    with pytest.raises(SystemExit):
        ap.parse_args(["--scorer", "nrms"])
