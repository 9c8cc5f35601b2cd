"""Training negatives, CPU side: the NumPy restatement of the device draw (oracle/negsample_oracle.py) and the resampling
feed's host tables against what the reference's own parse_behaviors made of the golden raw behaviours
(tests/golden/negsample/), the restated balancing loop against that output, the build-time errors, and the launcher's
--resample-negatives flag."""
import json
import os
import random
import subprocess
import sys
from collections import Counter

import numpy as np
import pandas as pd
import pytest

from feed_util import ROOT, family_config
from negsample_oracle import draw, negative_order, reference_balance
from newsrec_b200.evaluate import read_behaviors, read_news
from newsrec_b200.feed import DeviceFeed, resample_tables

FIXTURE = os.path.join(ROOT, "tests", "golden", "negsample")
SRC = os.path.join(ROOT, "news-recommendation_b200", "src")
H, K = 50, 2  # the reference NRMS config the fixture was minted with


def _index(directory=FIXTURE):
    ids, _ = read_news(directory, ["title"])
    index = {x: i for i, x in enumerate(ids)}
    index["PADDED_NEWS"] = len(ids)
    return ids, index


def _tables(directory=FIXTURE):
    ids, index = _index(directory)
    return ids, index, resample_tables(directory, index, H, K, os.path.join(directory, "user2int.tsv"))


def _reference_rows():
    """behaviors_parsed.tsv as the reference wrote it (an empty history is an empty field under pandas 3)."""
    return pd.read_table(os.path.join(FIXTURE, "behaviors_parsed.tsv"), keep_default_na=False)


def test_fixture_has_the_edge_cases():
    beh = read_behaviors(FIXTURE)
    P = np.asarray([sum(x.endswith("-1") for x in s.split()) for s in beh["impressions"]])
    N = np.asarray([sum(x.endswith("-0") for x in s.split()) for s in beh["impressions"]])
    hist = np.asarray([len(s.split()) for s in beh["clicked_news"]])
    assert (P == 0).any() and ((N < K) & (P > 0)).any() and (P > N // K).any() and ((P > 1) & (N // K >= P)).any()
    assert (hist == 0).any() and (hist == H).any() and (hist > H).any()
    assert beh["user"].duplicated().any()


@pytest.mark.parametrize("seed,epoch", [(0, 0), (7, 3), (2 ** 63 + 5, 11)])
def test_oracle_draw_has_the_reference_structure(seed, epoch):
    """Per impression the reference's rows and positives in order; every row's K negatives are the impression's
    negatives, and no negative (candidate position) serves two rows of one impression."""
    ids, index, t = _tables()
    ref = _reference_rows()
    row_offsets, cand = draw(t.cand_rows, t.labels, t.imp_offsets, K, seed, epoch)
    np.testing.assert_array_equal(row_offsets, t.row_offsets)
    assert len(ref) == row_offsets[-1] == len(t.behaviors)
    ref_cands = [[index[x] for x in s.split()] for s in ref["candidate_news"]]
    for i in range(len(t.imp_offsets) - 1):
        c = t.cand_rows[t.imp_offsets[i]:t.imp_offsets[i + 1]]
        lab = t.labels[t.imp_offsets[i]:t.imp_offsets[i + 1]]
        negs = Counter(c[lab == 0].tolist())
        mine, theirs = Counter(), Counter()
        for r in range(row_offsets[i], row_offsets[i + 1]):
            assert cand[r, 0] == ref_cands[r][0]  # the same positive, file order
            mine.update(cand[r, 1:].tolist())
            theirs.update(ref_cands[r][1:])
        assert not mine - negs and not theirs - negs  # drawn from the impression's negatives, none twice
        assert sum(mine.values()) == sum(theirs.values())
        n = int((lab == 0).sum())
        order = negative_order(seed, epoch, i, n)
        assert sorted(order.tolist()) == list(range(n))


def test_history_user_and_length_columns_equal_the_reference_rows():
    ids, index, t = _tables()
    ref = _reference_rows()
    pad = index["PADDED_NEWS"]
    for r, (user, hist, clicked) in enumerate(zip(ref["user"].tolist(), ref["clicked_news"].tolist(), ref["clicked"].tolist())):
        h = hist.split()[:H]
        np.testing.assert_array_equal(t.behaviors[r, :H], [pad] * (H - len(h)) + [index[x] for x in h])
        assert t.records[r, :2].tolist() == [int(user), len(h)]
        assert t.records[r, 2:].tolist() == [int(x) for x in clicked.split()] == [1] + [0] * K
    assert not t.behaviors[:, H:].any()  # the candidate columns are the draw's


def test_restated_balancing_loop_reproduces_the_reference_output():
    beh = read_behaviors(FIXTURE)
    pairs = reference_balance([s.split() for s in beh["impressions"]], K, random.Random(20261018))
    ref = _reference_rows()
    flat = [p for rows in pairs for p in rows]
    assert [" ".join(x.split("-")[0] for x in p) for p in flat] == ref["candidate_news"].tolist()
    assert [" ".join(x.split("-")[1] for x in p) for p in flat] == ref["clicked"].tolist()


def test_oracle_draw_is_fixed_by_seed_and_epoch():
    _, _, t = _tables()
    a = draw(t.cand_rows, t.labels, t.imp_offsets, K, 5, 2)[1]
    np.testing.assert_array_equal(a, draw(t.cand_rows, t.labels, t.imp_offsets, K, 5, 2)[1])
    assert not np.array_equal(a, draw(t.cand_rows, t.labels, t.imp_offsets, K, 5, 3)[1])
    assert not np.array_equal(a, draw(t.cand_rows, t.labels, t.imp_offsets, K, 6, 2)[1])
    # every input is hashed at full width: impressions 2^32 apart, epochs 2^32 apart
    assert negative_order(1, 0, 3, 50).tolist() != negative_order(1, 0, 3 + 2 ** 32, 50).tolist()
    assert negative_order(1, 4, 3, 50).tolist() != negative_order(1, 4 + 2 ** 32, 3, 50).tolist()


def _write_raw(tmp_path, rows, users=("U1", "U2")):
    src = open(os.path.join(FIXTURE, "news_parsed.tsv")).read()
    (tmp_path / "news_parsed.tsv").write_text(src)
    (tmp_path / "behaviors.tsv").write_text("".join(f"{n + 1}\t{u}\t11/1/2019 9:00:00 AM\t{h}\t{imp}\n" for n, (u, h, imp) in enumerate(rows)))
    (tmp_path / "user2int.tsv").write_text("user\tint\n" + "".join(f"{u}\t{i + 1}\n" for i, u in enumerate(users)))
    return str(tmp_path)


def test_parsing_errors(tmp_path):
    ok = ("U1", "N100 N101", "N102-1 N103-0 N104-0")
    d = _write_raw(tmp_path, [ok, ("U2", "N105", "N102-1 N103-2 N104-0")])
    with pytest.raises(ValueError, match="label"):
        _tables(d)
    d = _write_raw(tmp_path, [ok, ("U2", "N105", "N102-1 N999-0 N104-0")])
    with pytest.raises(KeyError):
        _tables(d)
    d = _write_raw(tmp_path, [ok, ("U2", "N105 N998", "N102-1 N103-0 N104-0")])
    with pytest.raises(KeyError):
        _tables(d)
    d = _write_raw(tmp_path, [ok, ("U9", "N105", "N102-1 N103-0 N104-0")])
    with pytest.raises(ValueError, match="U9"):
        _tables(d)
    d = _write_raw(tmp_path, [ok])
    assert len(_tables(d)[2].behaviors) == 1


def test_resampling_feed_needs_a_cuda_device():
    import newsrec_b200
    with pytest.raises(newsrec_b200.NewsrecError):
        DeviceFeed(os.path.join(FIXTURE, "behaviors_parsed.tsv"), os.path.join(FIXTURE, "news_parsed.tsv"), family_config("NRMS"),
                   device="cpu", resample_negatives=True, seed=3)


FAKE_TRAIN = '''
import json, os
from torch.utils.data import DataLoader
class BaseDataset:
    pass
def evaluate(*a, **k):
    return 0.5, 0.4, 0.3, 0.2
def train():
    ds = BaseDataset
    with open(os.environ["FAKE_OUT"], "w") as f:
        json.dump({"dataset": getattr(ds, "func", ds).__name__, "keywords": getattr(ds, "keywords", {}),
                   "loader": DataLoader.__qualname__}, f)
'''


def _launch(tmp_path, flags):
    (tmp_path / "train.py").write_text(FAKE_TRAIN)
    out = tmp_path / "out.json"
    env = dict(os.environ, PYTHONPATH=SRC, CUDA_VISIBLE_DEVICES="", FAKE_OUT=str(out), NEWSREC_FLAT_GRADS="0")
    cmd = [sys.executable, "-m", "newsrec_b200.launch", "--reference-src", str(tmp_path), "--no-dropin"] + flags
    return subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300), out


def test_launcher_refuses_resampling_without_the_device_feed(tmp_path):
    r, out = _launch(tmp_path, ["--resample-negatives"])
    assert r.returncode == 2 and "--resample-negatives needs --device-feed" in r.stderr
    assert not out.exists()


def test_launcher_resampling_feed_takes_the_seed(tmp_path):
    r, out = _launch(tmp_path, ["--device-feed", "--resample-negatives", "--seed", "17"])
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(out.read_text())
    assert got == {"dataset": "DeviceFeed", "keywords": {"resample_negatives": True, "seed": 17},
                   "loader": "make_feed_dataloader.<locals>.factory"}
