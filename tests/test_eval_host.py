"""Device evaluator, CPU side: the NumPy metric oracle against the live reference's values (tests/golden/eval_metrics.npz,
oracle/make_golden_metrics.py), the host tables of newsrec_b200.evaluate on a tiny validation directory, and the
launcher's opt-in."""
import os
import types

import numpy as np
import pytest

import ranking_metrics as R


def test_oracle_reproduces_the_reference_metrics(golden_dir):
    g = np.load(os.path.join(golden_dir, "eval_metrics.npz"))
    got = R.impression_metrics(g["scores"], g["labels"], g["offsets"])
    ref, cross = g["ref"], g["cross_tie"]
    assert cross.any() and (~cross).any()
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    fin = ~np.isnan(ref)
    diff = np.abs(np.where(fin, got - ref, 0.0))
    assert diff[~cross].max() <= 1e-12
    assert diff[cross, 0].max() <= 1e-12  # MRR / nDCG there depend on NumPy's unstable sort
    np.testing.assert_array_equal(R.cross_label_ties(g["scores"], g["labels"], g["offsets"]), cross)
    assert (np.diff(g["offsets"]) > 512).any()  # a segment longer than the kernel's shared-memory chunk


def test_oracle_edges():
    nan = np.isnan
    assert all(nan(R.single_impression([0.1, np.nan], [1, 0])))
    assert all(nan(R.single_impression([0.1, 0.2], [0, 0])))
    auc, mrr, n5, n10 = R.single_impression([0.3, -1.0, 2.0], [1, 1, 1])  # no negative: AUC undefined, the rest defined
    assert nan(auc) and abs(mrr - (1 + 1 / 2 + 1 / 3) / 3) < 1e-15 and n5 == 1.0 and n10 == 1.0
    # ties across labels: the later candidate ranks first
    assert R.single_impression([0.5, 0.5], [1, 0])[1] == 0.5
    assert R.single_impression([0.5, 0.5], [0, 1])[1] == 1.0
    assert R.single_impression([0.5, 0.5], [0, 1])[0] == 0.5
    assert R.single_impression([-0.0, 0.0], [0, 1])[1] == 1.0  # -0 == +0


H = 4


def _write_dir(tmp_path):
    news = ["N1", "N2", "N3", "N4", "N5", "N6"]
    with open(tmp_path / "news_parsed.tsv", "w") as f:
        f.write("id\ttitle\n")
        for i, n in enumerate(news):
            f.write(f"{n}\t{[i + 1, 0, 0]}\n")
    rows = [
        ("U1", "N1 N2 N3 N4 N5 N6", "N1-1 N2-0 N3-0"),  # history longer than H: first H ids
        ("U2", "N1 N2 N3 N4 N5 N6", "N4-0 N5-1"),       # same history, other user: first row wins
        ("U9", "", "N6-1 N1-1"),                       # empty history, unknown user, no negative
        ("U2", "N2", "N3-0 N2-0"),                     # no positive
        ("U1", "N1 N2 N3 N4 N5 N6", "N2-1"),           # duplicate (user, history)
        ("U3", "N5 N1", "N1-0 N2-1"),
    ]
    with open(tmp_path / "behaviors.tsv", "w") as f:
        for i, (u, h, imp) in enumerate(rows):
            f.write(f"{i + 1}\t{u}\t11/15/2019 8:55:22 AM\t{h}\t{imp}\n")
    with open(tmp_path / "user2int.tsv", "w") as f:
        f.write("user\tint\nU1\t1\nU2\t2\nU3\t3\n")
    index = {n: i for i, n in enumerate(news)}
    index["PADDED_NEWS"] = len(news)
    return index


def test_build_tables(tmp_path):
    from newsrec_b200.evaluate import build_tables
    index = _write_dir(tmp_path)
    u2i = str(tmp_path / "user2int.tsv")
    t = build_tables(str(tmp_path), index, H, user2int_path=u2i)
    P = index["PADDED_NEWS"]
    # distinct history strings in order of first appearance: "N1..N6" (U1), " " (U9), "N2" (U2), "N5 N1" (U3)
    np.testing.assert_array_equal(t.user, [1, 0, 2, 3])
    np.testing.assert_array_equal(t.history, [[0, 1, 2, 3], [P] * 4, [P, P, P, 1], [P, P, 4, 0]])
    np.testing.assert_array_equal(t.history_length, [4, 0, 1, 2])
    np.testing.assert_array_equal(t.seg_user, [0, 0, 1, 2, 0, 3])
    np.testing.assert_array_equal(t.seg_offsets, [0, 3, 5, 7, 9, 10, 12])
    np.testing.assert_array_equal(t.cand, [0, 1, 2, 3, 4, 5, 0, 2, 1, 1, 0, 1])
    np.testing.assert_array_equal(t.labels, [1, 0, 0, 0, 1, 1, 1, 0, 0, 1, 0, 1])
    assert t.labels.dtype == np.uint8 and t.cand.dtype == np.int64
    # max_count = k scores the first k - 1 impressions (the reference breaks on count == max_count before scoring)
    t3 = build_tables(str(tmp_path), index, H, max_count=3, user2int_path=u2i)
    np.testing.assert_array_equal(t3.seg_offsets, [0, 3, 5])
    np.testing.assert_array_equal(t3.seg_user, [0, 0])
    np.testing.assert_array_equal(t3.user, t.user)  # users come from every row, as in the reference
    assert len(build_tables(str(tmp_path), index, H, max_count=1, user2int_path=u2i).seg_user) == 0


def test_build_tables_unknown_news_raises(tmp_path):
    from newsrec_b200.evaluate import build_tables
    index = _write_dir(tmp_path)
    with open(tmp_path / "behaviors.tsv", "a") as f:
        f.write("7\tU1\t11/15/2019 8:55:22 AM\tN1\tN77-1 N1-0\n")
    with pytest.raises(KeyError):
        build_tables(str(tmp_path), index, H, user2int_path=str(tmp_path / "user2int.tsv"))


def test_build_tables_flags_labels_other_than_0_1(tmp_path):
    from newsrec_b200.evaluate import build_tables
    index = _write_dir(tmp_path)
    with open(tmp_path / "behaviors.tsv", "a") as f:
        f.write("7\tU1\t11/15/2019 8:55:22 AM\tN1\tN2-2 N1-0 N3-300\n")
    t = build_tables(str(tmp_path), index, H, user2int_path=str(tmp_path / "user2int.tsv"))
    np.testing.assert_array_equal(t.labels[-3:], [2, 0, 2])  # 300 must not wrap to a valid uint8 label


def test_read_news_columns(tmp_path):
    from newsrec_b200.evaluate import read_news
    _write_dir(tmp_path)
    ids, cols = read_news(str(tmp_path), ["title"])
    assert ids[:2] == ["N1", "N2"] and cols["title"].dtype == np.int64 and cols["title"].shape == (6, 3)


def test_patch_trainer_device_evaluate_opt_in():
    from newsrec_b200 import evaluate as ev
    from newsrec_b200 import launch

    def reference_evaluate(*a, **k):
        return ("reference", a)

    seen = {}

    def fake_device(*a, **k):
        seen["args"] = a
        return ("device", a)

    for opt in (False, True):
        mod = types.SimpleNamespace(DataLoader=object, evaluate=reference_evaluate)
        orig = ev.evaluate
        ev.evaluate = fake_device
        try:
            import torch
            adam = torch.optim.Adam
            launch.patch_trainer(mod, 0, 1, device_evaluate=opt)
            torch.optim.Adam = adam
        finally:
            ev.evaluate = orig
        out = mod.evaluate("model", "./data/val", 4, 200000)
        assert out[0] == ("device" if opt else "reference")
        assert out[1] == ("model", "./data/val", 4, 200000)
        assert mod.evaluate is not reference_evaluate and mod.evaluate is not fake_device  # behind the rank-0 wrapper


def test_launcher_parses_device_evaluate(monkeypatch):
    from newsrec_b200 import launch
    got = {}

    def fake_patch(train, rank, world, seed=0, device_evaluate=False):
        got["device_evaluate"] = device_evaluate
        raise SystemExit(0)

    monkeypatch.setattr(launch, "patch_trainer", fake_patch)
    monkeypatch.setattr(launch, "apply_compat_shims", lambda: None)
    import importlib
    fake_train = types.ModuleType("train")
    monkeypatch.setitem(__import__("sys").modules, "train", fake_train)
    monkeypatch.setattr(importlib, "import_module", lambda name: fake_train)
    monkeypatch.setenv("CUDA_VISIBLE_DEVICES", "")
    monkeypatch.setattr(__import__("sys"), "path", list(__import__("sys").path))
    with pytest.raises(SystemExit):
        launch.main(["--reference-src", "/nonexistent", "--device-evaluate"])
    assert got["device_evaluate"] is True
