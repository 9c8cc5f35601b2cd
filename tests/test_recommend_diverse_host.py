"""Diversified recommendation without a GPU: check_request's refusals of a bad cap, an unknown field and a news_parsed.tsv
without the field's column, all raised before any device work; the CLI's --max-per-category and --diversify-by; and the
ctypes row of nr_topk_dot_capped."""
import os

import pytest

from newsrec_b200 import SIGNATURES, NewsrecError
from newsrec_b200 import recommend as R

HEADER = "id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n"


class _Cfg:
    num_clicked_news_a_user = 4


def _fake(name):
    return type(name, (), {"config": _Cfg})()


def _split(d, header=HEADER):
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write("1\tU1\tt\tN1\tN2-1\n")
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write(header)


def test_bad_caps_and_fields_are_refused_before_the_device(tmp_path, monkeypatch):
    d = str(tmp_path)
    _split(d)
    import newsrec_b200.evaluate as E

    def no_device(*a, **k):
        raise AssertionError("device work before the refusal")
    monkeypatch.setattr(R, "news_matrix", no_device)
    monkeypatch.setattr(E, "news_matrix", no_device)
    out = os.path.join(d, "out.tsv")
    for m in (0, -1, 2.5, True, "2"):
        with pytest.raises(NewsrecError, match="max_per_category="):
            R.check_request(_fake("NRMS"), d, 10, m)
        with pytest.raises(NewsrecError, match="max_per_category="):
            R.recommend(_fake("NRMS"), d, out, 10, max_per_category=m)
    for field in ("title", "Category", "", None):
        with pytest.raises(NewsrecError, match="diversify_by="):
            R.recommend(_fake("NRMS"), d, out, 10, max_per_category=2, diversify_by=field)
    for m in (1, 2, 128, 10 ** 6, None):
        for field in ("category", "subcategory"):
            R.check_request(_fake("NRMS"), d, 10, m, field)
    assert not os.path.exists(out)


def test_a_missing_column_is_refused_only_when_a_cap_asks_for_it(tmp_path):
    d = str(tmp_path)
    _split(d, "id\tcategory\ttitle\tabstract\n")
    R.check_request(_fake("NRMS"), d, 10, 2, "category")
    R.check_request(_fake("NRMS"), d, 10)                    # no cap: the column is not read
    R.check_request(_fake("NRMS"), d, 10, None, "subcategory")
    with pytest.raises(NewsrecError, match="no subcategory column"):
        R.check_request(_fake("NRMS"), d, 10, 2, "subcategory")
    with pytest.raises(NewsrecError, match="no subcategory column"):
        R.recommend(_fake("NAML"), d, os.path.join(d, "out.tsv"), 10, max_per_category=1, diversify_by="subcategory")
    _split(d, "id\ttitle\n")
    with pytest.raises(NewsrecError, match="no category column"):
        R.check_request(_fake("NRMS"), d, 10, 3)
    with pytest.raises(NewsrecError, match="HiFiArk is not supported"):  # the family refusal still comes first
        R.check_request(_fake("HiFiArk"), d, 10, 3)


def test_cli_diversify_flags():
    a = R.parse_args(["--max-per-category", "2"])
    assert a.max_per_category == 2 and a.diversify_by == "category"
    a = R.parse_args(["--max-per-category", "1", "--diversify-by", "subcategory", "--k", "100"])
    assert (a.max_per_category, a.diversify_by, a.k) == (1, "subcategory", 100)
    a = R.parse_args([])
    assert a.max_per_category is None and a.diversify_by == "category"
    for bad in (["--max-per-category", "0"], ["--max-per-category", "-1"], ["--max-per-category", "2.5"],
                ["--diversify-by", "title"], ["--max-per-category", "2", "--diversify-by", "Category"]):
        with pytest.raises(SystemExit):
            R.parse_args(bad)


def test_capped_entry_point_signature():
    import ctypes as C
    res, args = SIGNATURES["nr_topk_dot_capped"]
    plain_res, plain = SIGNATURES["nr_topk_dot"]
    assert res is plain_res is C.c_int
    # nr_topk_dot's arguments with const int* categories and int max_per_category after the exclusions
    assert args == plain[:10] + [C.c_void_p, C.c_int] + plain[10:]
