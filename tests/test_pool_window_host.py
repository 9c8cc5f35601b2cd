"""Time windows without a GPU: newsrec_b200.window's time parsing, first_shown, time order and ranges against brute-force
loops, the row mappings, and every refusal of max_age_hours in recommend, evaluate_pool, evaluate_lists and their command
lines, raised before a device is needed."""
import math
import os
from datetime import datetime, timedelta

import numpy as np
import pandas as pd
import pytest

from newsrec_b200 import NewsrecError, window
from newsrec_b200 import pool_eval as P
from newsrec_b200 import recommend as R

HEADER = "id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n"


def _secs(text):
    return int((datetime.strptime(text, window.TIME_FORMAT) - datetime(1970, 1, 1)).total_seconds())


def test_times_parse_to_naive_seconds_with_the_12_am_and_pm_edges():
    cases = ["11/15/2019 8:55:22 AM", "11/15/2019 12:00:00 AM", "11/15/2019 12:00:00 PM", "11/15/2019 12:59:59 AM",
             "11/15/2019 11:59:59 PM", "1/2/2019 1:02:03 PM", "02/29/2020 07:07:07 AM"]
    got = window.parse_times(cases)
    assert got.dtype == np.int64 and got.tolist() == [_secs(c) for c in cases]
    assert got[1] == got[0] - (8 * 3600 + 55 * 60 + 22) and got[2] - got[1] == 12 * 3600 and got[3] - got[1] == 3599
    for bad in ["11/15/2019 13:00:00 PM", "2019-11-15 08:00:00", "11/15/2019 8:55:22", "", "t", float("nan")]:
        with pytest.raises(NewsrecError):
            window.parse_times(["11/15/2019 8:55:22 AM", bad])


def _random_split(rng, n_news=40, n_rows=60):
    ids = [f"N{i}" for i in range(n_news)]
    t0 = _secs("11/09/2019 12:00:00 AM")
    times = t0 + 3600 * rng.integers(0, 24 * 6, n_rows) + rng.integers(0, 2, n_rows) * 1800
    imps = []
    for _ in range(n_rows):
        c = rng.choice(ids[:n_news - 5], int(rng.integers(0, 6)), replace=False)  # the last 5 news are never listed
        imps.append(" ".join(f"{x}-{int(rng.integers(0, 2))}" if rng.random() < 0.7 else str(x) for x in c))
    beh = pd.DataFrame({"time": [(datetime(1970, 1, 1) + timedelta(seconds=int(t))).strftime("%m/%d/%Y %I:%M:%S %p") for t in times],
                        "clicked_news": [" ".join(rng.choice(ids, 3)) for _ in range(n_rows)],  # histories never count
                        "impressions": imps})
    pool_ids = ids + ids[:3]  # an id on several pool rows: each gets the id's value
    return beh, times.astype(np.int64), pool_ids


def _brute_first(beh, times, pool_ids):
    first = {}
    for t, imp in zip(times, beh["impressions"]):
        for x in str(imp).split():
            nid = x.split("-")[0]
            first[nid] = min(first.get(nid, t), t)
    shown = np.array([x in first for x in pool_ids])
    return np.array([first.get(x, 0) for x in pool_ids], np.int64), shown


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_first_shown_order_and_ranges_against_brute_force(seed):
    rng = np.random.default_rng(seed)
    beh, times, pool_ids = _random_split(rng)
    assert (window.parse_times(beh["time"]) == times).all()
    first, shown = window.first_shown(beh, times, pool_ids)
    bf, bs = _brute_first(beh, times, pool_ids)
    assert (shown == bs).all() and (first[shown] == bf[bs]).all() and not shown[-8:-3].any()
    pw = window.PoolWindow(first, shown)
    keys = [(0 if s else -1, f if s else 0, r) for r, (f, s) in enumerate(zip(first, shown))]
    assert pw.perm.tolist() == sorted(range(len(keys)), key=lambda r: keys[r])
    assert (pw.perm[pw.inv] == np.arange(len(first))).all()
    W = 24 * 3600.0
    req = np.concatenate([times, first[shown] + W, first[shown], first[shown] - 1])  # both ends exactly, and just past
    for H in (24.0, 0.5, 1e-9, math.inf):
        W = H * 3600.0
        lo, hi = pw.ranges(req, W)
        for t, a, b in zip(req, lo, hi):
            want = {r for r in range(len(first)) if shown[r] and t - W <= first[r] <= t}
            assert set(pw.perm[a:b].tolist()) == want, (t, H)


def test_row_mappings_round_trip_and_keep_minus_one():
    pw = window.PoolWindow(np.array([5, 3, 0, 3, 9]), np.array([True, True, False, True, True]))
    assert pw.perm.tolist() == [2, 1, 3, 0, 4]
    rows = np.array([[4, 0, -1], [2, -1, -1]])
    pos = pw.to_time_order(rows)
    assert pos.tolist() == [[4, 3, -1], [0, -1, -1]]
    assert (pw.to_rows(pos) == rows).all()
    gather, offs = window.csr_take(np.array([0, 2, 2, 5]), np.array([2, 0, 1]))
    assert gather.tolist() == [2, 3, 4, 0, 1] and offs.tolist() == [0, 3, 5, 5]


class _Cfg:
    num_clicked_news_a_user = 5


def _fake(name):
    return type(name, (), {"config": _Cfg})()


def _split(d, time="11/15/2019 8:55:22 AM"):
    with open(os.path.join(d, "behaviors.tsv"), "w") as f:
        f.write(f"1\tU1\t{time}\tN1\tN2-1 N1-0\n")
    with open(os.path.join(d, "news_parsed.tsv"), "w") as f:
        f.write(HEADER)


@pytest.mark.parametrize("H", [0, -1.0, float("nan"), "24", True, [24]])
def test_keyword_refusals(tmp_path, H):
    d = str(tmp_path)
    _split(d)
    with pytest.raises(NewsrecError, match="max_age_hours"):
        R.recommend(_fake("NRMS"), d, str(tmp_path / "o.tsv"), max_age_hours=H)
    with pytest.raises(NewsrecError, match="max_age_hours"):
        P.evaluate_pool(_fake("NRMS"), d, max_age_hours=H)
    with pytest.raises(NewsrecError, match="max_age_hours"):
        P.evaluate_lists(_fake("NRMS"), d, max_age_hours=H)
    assert not os.path.exists(tmp_path / "o.tsv")


def test_an_unparseable_time_is_refused_before_any_device_work(tmp_path):
    d = str(tmp_path)
    _split(d, time="2019-11-15T08:55:22")
    with pytest.raises(NewsrecError, match="time"):
        R.recommend(_fake("NRMS"), d, str(tmp_path / "o.tsv"), max_age_hours=24)
    with pytest.raises(NewsrecError, match="time"):
        P.evaluate_pool(_fake("NRMS"), d, max_age_hours=24)
    with pytest.raises(NewsrecError, match="time"):
        P.evaluate_lists(_fake("NRMS"), d, max_age_hours=24)
    # a split whose times parse: the checks return W in seconds
    _split(d)
    assert R.check_request(_fake("NRMS"), d, 10, max_age_hours=math.inf)[0] == math.inf
    assert P.check_request(_fake("NRMS"), d, (5,), max_age_hours=1.5)[0] == 5400.0


@pytest.mark.parametrize("bad", ["0", "-3", "nan", "x"])
def test_command_line_refusals(bad, capsys):
    for parse, extra in ((R.parse_args, []), (P.parse_args, []), (P.parse_args, ["--lists"])):
        with pytest.raises(SystemExit):
            parse(extra + ["--max-age-hours", bad])
        assert "max-age-hours" in capsys.readouterr().err
    assert R.parse_args(["--max-age-hours", "inf"]).max_age_hours == math.inf
    assert P.parse_args(["--lists", "--max-age-hours", "48"]).max_age_hours == 48.0
    assert P.parse_args([]).max_age_hours is None
