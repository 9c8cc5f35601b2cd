"""Device feed, CPU side: DeviceFeed's host tables and the restated loader (oracle/feed_oracle.py) against batches the
reference's own BaseDataset + default_collate made of the golden fixture (tests/golden/feed.npz), the build-time errors,
the epoch row order, and the launcher's --device-feed opt-in."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
from torch.utils.data import default_collate

from feed_oracle import FeedOracle
from feed_util import BEHAVIORS, FAMILIES, NEWS, ROOT, collated_arrays, family_config, golden, golden_arrays
from newsrec_b200.feed import DeviceFeed, epoch_rows

SRC = os.path.join(ROOT, "news-recommendation_b200", "src")


def _check_equal(got, want):
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype == np.int64, k
        np.testing.assert_array_equal(got[k], want[k], err_msg=k)


@pytest.mark.parametrize("fam", FAMILIES)
def test_host_tables_equal_the_reference_batches(fam):
    g, cfg = golden(), family_config(fam)
    want = golden_arrays(g, fam)
    order = g[f"{fam}.order"]
    feed = DeviceFeed(BEHAVIORS, NEWS, cfg, device="cpu")
    H, C = cfg.num_clicked_news_a_user, feed.C
    assert feed.behaviors.shape == (len(feed), H + C) and feed.behaviors.dtype == np.int32
    # the tables read the way the gather kernel reads them: news rows of the batch rows, slot-major here
    rows = feed.behaviors[order]
    got = {}
    for attr, table in feed.news_tables.items():
        assert table.dtype == np.int32 and not table[feed.pad_row].any()
        blk = table[rows].astype(np.int64)  # (B, H + C, L)
        blk = blk if table.shape[1] > 1 or attr not in ("category", "subcategory") else blk[..., 0]
        got[f"clicked_news.{attr}"] = np.moveaxis(blk[:, :H], 1, 0)
        got[f"candidate_news.{attr}"] = np.moveaxis(blk[:, H:], 1, 0)
    rec = feed.records[order].astype(np.int64)
    got["clicked"] = rec[:, 2:].T
    for i, name in enumerate(("user", "clicked_news_length")):
        if name in cfg.dataset_attributes["record"]:
            got[name] = rec[:, i]
    _check_equal(got, want)
    # and item by item, collated as the reference's DataLoader does
    _check_equal(collated_arrays(default_collate([feed[int(i)] for i in order]), cfg), want)


@pytest.mark.parametrize("fam", FAMILIES)
def test_restated_loader_equals_the_reference_batches(fam):
    g, cfg = golden(), family_config(fam)
    ds = FeedOracle(BEHAVIORS, NEWS, cfg)
    batch = default_collate([ds[int(i)] for i in g[f"{fam}.order"]])
    _check_equal(collated_arrays(batch, cfg), golden_arrays(g, fam))


def test_fixture_has_the_edge_cases():
    g = golden()
    lengths = g["LSTUR.clicked_news_length"]
    assert 0 in lengths and (lengths == 50).sum() >= 2  # empty, exactly 50 and truncated 60 / 51
    feed = DeviceFeed(BEHAVIORS, NEWS, family_config("DKN"), device="cpu")
    assert (feed.news_tables["title_entities"][:-1] != 0).any()
    import pandas as pd
    beh = pd.read_table(BEHAVIORS)
    hist = beh["clicked_news"].tolist()
    assert " " in hist and any(len(h.split()) == 50 for h in hist) and any(len(h.split()) == 60 for h in hist)
    assert any(len(set(h.split())) < len(h.split()) for h in hist if len(h.split()) < 10)
    assert beh["user"].duplicated().any()


def _write(tmp_path, news_rows, beh_rows):
    n, b = tmp_path / "news_parsed.tsv", tmp_path / "behaviors_parsed.tsv"
    n.write_text("id\tcategory\tsubcategory\ttitle\tabstract\ttitle_entities\tabstract_entities\n" + "".join(news_rows))
    b.write_text("user\tclicked_news\tcandidate_news\tclicked\n" + "".join(beh_rows))
    return str(b), str(n)


def _news(i, T=20, TA=50):
    return f"N{i}\t1\t2\t{[i] * T}\t{[i] * TA}\t{[0] * T}\t{[0] * TA}\n"


def test_unknown_news_id_raises_keyerror(tmp_path):
    b, n = _write(tmp_path, [_news(1), _news(2)], ["1\tN1 N9\tN1 N2\t1 0\n"])
    with pytest.raises(KeyError):
        DeviceFeed(b, n, family_config("NRMS"), device="cpu")
    b, n = _write(tmp_path, [_news(1), _news(2)], ["1\tN1\tN1 N7\t1 0\n"])
    with pytest.raises(KeyError):
        DeviceFeed(b, n, family_config("NRMS"), device="cpu")


def test_varying_candidate_count_raises(tmp_path):
    b, n = _write(tmp_path, [_news(1), _news(2)], ["1\tN1\tN1 N2\t1 0\n", "2\tN2\tN1 N2 N1\t1 0 0\n"])
    with pytest.raises(ValueError, match="candidates"):
        DeviceFeed(b, n, family_config("NRMS"), device="cpu")


def test_list_column_of_another_length_raises(tmp_path):
    b, n = _write(tmp_path, [_news(1), _news(2)], ["1\tN1\tN1 N2\t1 0\n"])
    with pytest.raises(ValueError, match="title"):
        DeviceFeed(b, n, family_config("NRMS", num_words_title=19), device="cpu")
    with pytest.raises(ValueError, match="abstract"):
        DeviceFeed(b, n, family_config("NAML", num_words_abstract=51), device="cpu")
    b, n = _write(tmp_path, [_news(1), _news(2, T=21)], ["1\tN1\tN1 N2\t1 0\n"])
    with pytest.raises(ValueError):
        DeviceFeed(b, n, family_config("NRMS"), device="cpu")


def test_loader_needs_a_cuda_device():
    import newsrec_b200
    feed = DeviceFeed(BEHAVIORS, NEWS, family_config("NRMS"), device="cpu")
    with pytest.raises(newsrec_b200.NewsrecError):
        feed.loader(4)


@pytest.mark.parametrize("n,B", [(20000, 512), (12, 5), (1000, 7)])
def test_epoch_rows_visit_each_row_once(n, B):
    rows = epoch_rows(n, B, shuffle=True, drop_last=True, seed=3, epoch=0)
    assert len(rows) == n // B * B and len(set(rows.tolist())) == len(rows) and 0 <= int(rows.min()) and int(rows.max()) < n
    again = epoch_rows(n, B, shuffle=True, drop_last=True, seed=3, epoch=0)
    assert rows.tolist() == again.tolist()  # the seed and epoch fix the order
    nxt = epoch_rows(n, B, shuffle=True, drop_last=True, seed=3, epoch=1)
    assert nxt.tolist() != rows.tolist()  # a re-created loader draws a new permutation
    assert len(epoch_rows(n, B, shuffle=False, drop_last=False)) == n


def test_epoch_rows_of_two_ranks_are_disjoint():
    r0 = epoch_rows(1000, 16, shuffle=True, drop_last=True, rank=0, world=2, seed=5, epoch=2)
    r1 = epoch_rows(1000, 16, shuffle=True, drop_last=True, rank=1, world=2, seed=5, epoch=2)
    assert len(r0) == len(r1) == 500 // 16 * 16
    assert not set(r0.tolist()) & set(r1.tolist())


def test_feed_dataloader_factory_advances_the_epoch(monkeypatch):
    from newsrec_b200 import launch
    calls = []
    monkeypatch.setattr(DeviceFeed, "loader", lambda self, *a, **k: calls.append((a, k)) or "feed-loader")
    feed = DeviceFeed(BEHAVIORS, NEWS, family_config("NRMS"), device="cpu")
    factory = launch.make_feed_dataloader(lambda ds, *a, **k: ("base", ds), rank=1, world=2, seed=9)
    for _ in range(2):
        assert factory(feed, batch_size=4, shuffle=True, num_workers=4, drop_last=True, pin_memory=True) == "feed-loader"
    assert [k["epoch"] for _, k in calls] == [0, 1]
    assert calls[0] == ((4,), dict(shuffle=True, drop_last=True, rank=1, world=2, seed=9, epoch=0))
    assert factory([1, 2], batch_size=2) == ("base", [1, 2])


FAKE_TRAIN = '''
import json, os
from torch.utils.data import DataLoader
class BaseDataset:
    pass
def evaluate(*a, **k):
    return 0.5, 0.4, 0.3, 0.2
def train():
    with open(os.environ["FAKE_OUT"], "w") as f:
        json.dump({"dataset": BaseDataset.__module__ + "." + BaseDataset.__name__,
                   "loader": DataLoader.__qualname__, "loader_module": DataLoader.__module__}, f)
'''


@pytest.mark.parametrize("flag", [False, True])
def test_launcher_device_feed_flag_patches_the_trainer(tmp_path, flag):
    (tmp_path / "train.py").write_text(FAKE_TRAIN)
    out = tmp_path / "out.json"
    env = dict(os.environ, PYTHONPATH=SRC, CUDA_VISIBLE_DEVICES="", FAKE_OUT=str(out), NEWSREC_FLAT_GRADS="0")
    cmd = [sys.executable, "-m", "newsrec_b200.launch", "--reference-src", str(tmp_path), "--no-dropin"] + (["--device-feed"] if flag else [])
    r = subprocess.run(cmd, cwd=str(tmp_path), env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(out.read_text())
    if flag:
        assert got["dataset"] == "newsrec_b200.feed.DeviceFeed"
        assert got["loader"] == "make_feed_dataloader.<locals>.factory"
    else:  # exactly today's patch: the reference's dataset, the sharded DataLoader factory
        assert got["dataset"] == "train.BaseDataset"
        assert got["loader"] == "make_sharded_dataloader.<locals>.factory"
