"""Test-set predictions, CPU side: the host tables of newsrec_b200.predict on tiny test splits, the rank restatement
(tests/prediction_ref.py) against a brute-force count, and the argument checks of the new entry points, which refuse before
touching a device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import prediction_ref as PR

H = 4
NEWS = ["N1", "N2", "N3", "N4", "N5", "N6"]


def _write_dir(tmp_path, rows):
    with open(tmp_path / "behaviors.tsv", "w") as f:
        for iid, u, h, imp in rows:
            f.write(f"{iid}\t{u}\t11/15/2019 8:55:22 AM\t{h}\t{imp}\n")
    with open(tmp_path / "user2int.tsv", "w") as f:
        f.write("user\tint\nU1\t1\nU2\t2\nU3\t3\n")
    index = {n: i for i, n in enumerate(NEWS)}
    index["PADDED_NEWS"] = len(NEWS)
    return index


def _tables(tmp_path, rows):
    from newsrec_b200.predict import build_prediction_tables
    index = _write_dir(tmp_path, rows)
    return build_prediction_tables(str(tmp_path), index, H, user2int_path=str(tmp_path / "user2int.tsv"))


ROWS = [
    (7, "U1", "N1 N2 N3 N4 N5 N6", "N1 N2 N3"),   # unlabelled tokens, history longer than H
    (3, "U2", "N1 N2 N3 N4 N5 N6", "N4-0 N5-1"),  # labelled tokens; same history under another user: first row wins
    (0, "U9", "", "N6 N1-1"),                     # empty history, unknown user, mixed tokens
    (1099511627776, "U2", "N2", "N3"),            # 2^40, one candidate
    (12, "U3", "N5 N1", "N1-0 N2"),
]


def test_tables_accept_unlabelled_labelled_and_mixed_tokens(tmp_path):
    t = _tables(tmp_path, ROWS)
    P = len(NEWS)
    np.testing.assert_array_equal(t.impression_id, [7, 3, 0, 1 << 40, 12])
    np.testing.assert_array_equal(t.user, [1, 0, 2, 3])
    np.testing.assert_array_equal(t.history, [[0, 1, 2, 3], [P] * 4, [P, P, P, 1], [P, P, 4, 0]])
    np.testing.assert_array_equal(t.history_length, [4, 0, 1, 2])
    np.testing.assert_array_equal(t.seg_user, [0, 0, 1, 2, 3])
    np.testing.assert_array_equal(t.seg_offsets, [0, 3, 5, 7, 8, 10])
    np.testing.assert_array_equal(t.cand, [0, 1, 2, 3, 4, 5, 0, 2, 0, 1])
    assert t.impression_id.dtype == np.int64 and t.cand.dtype == np.int64


def test_tables_share_the_user_half_of_build_tables(tmp_path):
    from newsrec_b200.evaluate import build_tables
    labelled = [(i, u, h, " ".join(x if "-" in x else x + "-0" for x in imp.split())) for i, u, h, imp in ROWS]
    t = _tables(tmp_path, labelled)
    e = build_tables(str(tmp_path), {**{n: i for i, n in enumerate(NEWS)}, "PADDED_NEWS": len(NEWS)}, H,
                     user2int_path=str(tmp_path / "user2int.tsv"))
    for k in ("user", "history", "history_length", "seg_user", "cand", "seg_offsets"):
        np.testing.assert_array_equal(getattr(t, k), getattr(e, k), err_msg=k)


def test_chunk_keeps_only_the_users_it_references(tmp_path):
    t = _tables(tmp_path, ROWS)
    c = t.chunk(2, 5)
    np.testing.assert_array_equal(c.impression_id, [0, 1 << 40, 12])
    np.testing.assert_array_equal(c.user, [0, 2, 3])
    np.testing.assert_array_equal(c.seg_user, [0, 1, 2])
    np.testing.assert_array_equal(c.seg_offsets, [0, 2, 3, 5])
    np.testing.assert_array_equal(c.cand, t.cand[5:])
    np.testing.assert_array_equal(c.history, t.history[1:])
    one = t.chunk(1, 2)
    np.testing.assert_array_equal(one.user, [1])
    np.testing.assert_array_equal(one.seg_user, [0])


def test_unknown_news_raises_key_error(tmp_path):
    with pytest.raises(KeyError):
        _tables(tmp_path, ROWS + [(13, "U1", "N1", "N77 N1")])
    with pytest.raises(KeyError):
        _tables(tmp_path, ROWS + [(13, "U1", "N1 N88", "N1")])


@pytest.mark.parametrize("imp", ["", " "])
def test_empty_impression_raises_with_the_row(tmp_path, imp):
    with pytest.raises(ValueError, match="line 6: impression 13 has no candidate"):
        _tables(tmp_path, ROWS + [(13, "U1", "N1", imp)])


@pytest.mark.parametrize("iid", ["-1", "1.5", "x7", "", "+3", "9223372036854775808"])
def test_impression_id_must_be_a_non_negative_integer(tmp_path, iid):
    with pytest.raises(ValueError, match="line 3: impression id"):
        _tables(tmp_path, ROWS[:2] + [(iid, "U1", "N1", "N2")])


def _brute_ranks(s):
    s = [float(x) for x in s]  # -0.0 == 0.0 in Python comparisons
    return [1 + sum(sj > si for sj in s) + sum(s[j] == si for j in range(i + 1, len(s))) for i, si in enumerate(s)]


def test_oracle_ranks_against_a_brute_force_count():
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 31, 33, 100):
        for kind in range(4):
            if kind == 0:
                s = rng.standard_normal(n).astype(np.float32)
            elif kind == 1:
                s = (rng.integers(-2, 3, n) * 0.5).astype(np.float32)  # heavy ties
            elif kind == 2:
                s = rng.choice(np.array([-0.0, 0.0, 1e-45, -1e-45, 1.0], np.float32), n)  # -0 / +0 and subnormals
            else:
                s = np.zeros(n, np.float32)
            r = PR.single_ranks(s)
            assert list(r) == _brute_ranks(s), (n, kind, s)
            assert sorted(r) == list(range(1, n + 1))
    assert list(PR.single_ranks(np.array([-0.0, 0.0], np.float32))) == [2, 1]   # equal: the later candidate first
    assert list(PR.single_ranks(np.array([0.5, 0.5, 2.0], np.float32))) == [3, 2, 1]
    offs = [0, 2, 5]
    np.testing.assert_array_equal(PR.impression_ranks([1.0, 2.0, 3.0, 3.0, -1.0], offs), [2, 1, 2, 1, 3])


def test_mrr_from_oracle_ranks_is_the_metric_oracle_mrr():
    import ranking_metrics as R
    rng = np.random.default_rng(2)
    lens = rng.integers(1, 60, 300)
    offs = np.concatenate([[0], np.cumsum(lens)])
    s = (rng.integers(-3, 4, offs[-1]) * 0.25).astype(np.float32)
    y = (rng.random(offs[-1]) < 0.3).astype(np.uint8)
    r = PR.impression_ranks(s, offs)
    for a, b in zip(offs[:-1], offs[1:]):
        pos = y[a:b] == 1
        if pos.any():
            assert abs(np.mean(1.0 / r[a:b][pos]) - R.single_impression(s[a:b], y[a:b])[1]) <= 1e-12


def test_text_restatement():
    got = PR.prediction_text([0, 10, 1 << 40], np.array([1, 2, 1, 1]), [0, 1, 3, 4])
    assert got == b"0 [1]\n10 [2,1]\n1099511627776 [1]\n"


@pytest.fixture(scope="module")
def lib():
    import newsrec_b200
    return newsrec_b200.load_library()


def _call(lib, fn, *args):
    n0 = lib.nr_launch_count()
    rc = getattr(lib, fn)(*args)
    return rc, lib.nr_last_error().decode(), lib.nr_launch_count() - n0


def test_entry_points_refuse_bad_arguments_without_a_device(lib):
    p, z = C.c_void_p(16), None
    cases = [
        ("nr_impression_ranks", (z, p, 1, p, p, z), "null operand"),
        ("nr_impression_ranks", (p, z, 1, p, p, z), "null operand"),
        ("nr_impression_ranks", (p, p, 1, z, p, z), "null operand"),
        ("nr_impression_ranks", (p, p, 1, p, z, z), "null operand"),
        ("nr_impression_ranks", (p, p, -1, p, p, z), "n_seg=-1"),
        ("nr_prediction_line_offsets", (z, p, p, 1, p, p, 1 << 20, z), "null operand"),
        ("nr_prediction_line_offsets", (p, z, p, 1, p, p, 1 << 20, z), "null operand"),
        ("nr_prediction_line_offsets", (p, p, z, 1, p, p, 1 << 20, z), "null operand"),
        ("nr_prediction_line_offsets", (p, p, p, 1, z, p, 1 << 20, z), "null operand"),
        ("nr_prediction_line_offsets", (p, p, p, 1, p, z, 1 << 20, z), "null operand"),
        ("nr_prediction_line_offsets", (p, p, p, -1, p, p, 1 << 20, z), "n_seg=-1"),
        ("nr_prediction_line_offsets", (p, p, p, 1 << 31, p, p, 1 << 20, z), "at most 2^31 - 2"),
        ("nr_prediction_text", (z, p, p, 1, p, p, z), "null operand"),
        ("nr_prediction_text", (p, z, p, 1, p, p, z), "null operand"),
        ("nr_prediction_text", (p, p, z, 1, p, p, z), "null operand"),
        ("nr_prediction_text", (p, p, p, 1, z, p, z), "null operand"),
        ("nr_prediction_text", (p, p, p, 1, p, z, z), "null operand"),
        ("nr_prediction_text", (p, p, p, -1, p, p, z), "n_seg=-1"),
    ]
    for fn, args, what in cases:
        rc, msg, launched = _call(lib, fn, *args)
        assert rc == -1 and what in msg and fn in msg and launched == 0, (fn, args, rc, msg, launched)
    assert lib.nr_prediction_line_offsets_workspace(-1) == -1 and "n_seg=-1" in lib.nr_last_error().decode()


def test_cli_parses_and_finds_the_latest_checkpoint(tmp_path):
    from newsrec_b200.predict import latest_checkpoint
    assert latest_checkpoint(str(tmp_path / "missing")) is None
    assert latest_checkpoint(str(tmp_path)) is None
    for n in (9, 100, 12):
        (tmp_path / f"ckpt-{n}.pth").write_bytes(b"")
    assert latest_checkpoint(str(tmp_path)) == os.path.join(str(tmp_path), "ckpt-100.pth")


def test_checkpoint_with_a_numpy_early_stop_value_loads_weights_only(tmp_path):
    import torch
    from newsrec_b200.predict import load_checkpoint
    path = str(tmp_path / "ckpt-3.pth")
    torch.save({"model_state_dict": {"w": torch.arange(3.0)}, "optimizer_state_dict": {}, "step": 3,
                "early_stop_value": -np.float64(0.71)}, path)
    got = load_checkpoint(path, "cpu")
    assert torch.equal(got["model_state_dict"]["w"], torch.arange(3.0)) and got["early_stop_value"] == -0.71


def test_cli_without_a_checkpoint_exits(tmp_path, monkeypatch):
    from newsrec_b200 import predict
    monkeypatch.setattr(sys, "path", list(sys.path))
    with pytest.raises(SystemExit, match="no checkpoint file found"):
        predict.main(["--directory", str(tmp_path), "--checkpoint-dir", str(tmp_path / "none")])
